"""The train-mode schedule of the generator does not move: every `abi.call` of a train() forward + backward -- entry point,
scalar arguments, which pointers are NULL, in order -- equals the sequence recorded before eval-mode gradients, the
`last_back` gradient and the per-parameter weight-gradient gating were added (tests/golden/make_train_launch_sequence.py)."""
import importlib
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_train_launch_sequence as recipe  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", sorted(recipe.CASES))
def test_train_mode_launch_sequence_is_the_recorded_one(pkg, case):
    with open(os.path.join(HERE, "golden", "train_launch_sequence.json")) as f:
        gold = json.load(f)
    want = [gold["calls"][i] for i in gold["cases"][case]]
    got = recipe.record_case(pkg, *recipe.CASES[case])
    # the one change of signature since the recording: hg_render_composite_bwd gained `last_back` before the stream
    # argument, which train mode must pass as 0
    bwd = "hg_render_composite_bwd("
    for i, c in enumerate(got):
        if c.startswith(bwd):
            args = c[len(bwd):-1].split(",")
            assert args[-2] == "0", c
            got[i] = bwd + ",".join(args[:-2] + args[-1:]) + ")"
    assert any(c.startswith(bwd) for c in got) and len(want) > 300
    first = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), None)
    assert first is None, (first, got[first], want[first])
    assert len(got) == len(want)
