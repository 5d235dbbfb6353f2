"""Record the results of the reference's own code that tests/test_cpu_trainer_pin.py and
tests/test_oracle_pin.py::test_oracle_matches_live_reference compare against (`golden_util.reference_result`): runs those
tests once with the reference importable and writes tests/golden/reference_results.npz.

    HG_REFERENCE=/path/to/reference python tests/golden/make_golden_trainer.py
"""
import os
import sys

import pytest

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, TESTS)

import golden_util  # noqa: E402

if __name__ == "__main__":
    golden_util.RECORDING = {}
    rc = pytest.main([os.path.join(TESTS, "test_cpu_trainer_pin.py"),
                      os.path.join(TESTS, "test_oracle_pin.py") + "::test_oracle_matches_live_reference", "-q", "-p", "no:cacheprovider"])
    if rc != 0:
        sys.exit(rc)
    golden_util.save_reference_results()
