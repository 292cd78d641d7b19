"""PIN of the oracle at the reference's NON-DEFAULT run-time settings.

A user changes the six globals of util/settings.cpp:80-88 between frames with ROS dynamic reconfigure
(cfg/LSDParams.cfg:13-34, IOWrapper/ROS/rosReconfigure.h:81-91).  tests/test_ref_pin.py holds the C restatement to the
reference-compiled library at the defaults only; this module runs the same case functions under each setting of
tests/pin_cases.SETS, one at a time, and under one combined ROS-like set, and checks every observation against tests/golden/ref_pin_globals_320x240.npz
(recorded from oracle/_ref/liblsd_ref.so by python -m tests.golden.make_golden_ref_pin_globals).  Each set runs only the cases
that read its setting: the depth-map cases for the mapping settings, the SE3 cases for the tracking ones, the track + map loop
for all of them.

Non-vacuity: every set changes at least one recorded observation against the default record, and the two minUseGrad values
are thresholds some pixels of frame 0 sit exactly on, so `<` and `<=` give different point sets there."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import pin_cases as pin

PAIRS = pin.SETTINGS_PAIRS
_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_GLOBALS)
    return _gold


@pytest.mark.parametrize("set_name,case", PAIRS, ids=[f"{s}-{c}" for s, c in PAIRS])
def test_matches_reference_compiled_under_settings(seq_small, frames_small, set_name, case):
    pin.run_under_settings(set_name, case, _load(), seq_small, frames_small)


@pytest.mark.parametrize("set_name", list(pin.SETS))
def test_each_set_changes_the_recorded_outputs(set_name):
    """the record of every set differs from the default record somewhere: the setting reached the reference's code"""
    g, d = _load(), np.load(pin.GOLD)
    keys = [k for k in g.files if k.startswith(set_name + "/")]
    assert keys
    differ = [k for k in keys if not np.array_equal(g[k], d[k[len(set_name) + 1:]])]
    assert differ, f"{set_name}: every observation equals the default record"


def test_min_use_grad_values_are_ties_on_frame0(seq_small, frames_small):
    """Frame 0 has pixels whose maxGradients equal each minUseGrad value exactly, so the pins above separate `<` from `<=`."""
    po.set_globals(False)
    mg = po.Frame(0, frames_small[0][0], seq_small.K).maxGradients(0)[2:-2]      # the defined interior, see frame_builders
    for s, (g, _) in pin.SETS.items():
        if "minUseGrad" in g:
            assert int((mg == np.float32(g["minUseGrad"])).sum()) > 0, s
