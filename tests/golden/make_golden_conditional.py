"""Record the results of the reference's own step functions that tests/test_cpu_trainer_conditional.py compares against: runs
that file once with the reference importable and writes tests/golden/conditional_phases.npz.

    HG_REFERENCE=/path/to/reference python tests/golden/make_golden_conditional.py
"""
import os
import sys

import pytest

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, TESTS)

import test_cpu_trainer_conditional as pin  # noqa: E402

if __name__ == "__main__":
    pin.RECORDING = {}
    rc = pytest.main([os.path.join(TESTS, "test_cpu_trainer_conditional.py"), "-q", "-p", "no:cacheprovider"])
    if rc != 0:
        sys.exit(rc)
    pin.save_results()
