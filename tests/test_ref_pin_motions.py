"""PIN of the oracle under camera motions other than the default (tests/motions.py).

Every other pin runs the synthetic stream's default twist: mostly sideways, so every epipolar line the depth map searches is close
to horizontal and points the same way, the epipole lies far outside the image, and propagation never lands two sources at
inconsistent depths on one pixel.  This module runs the case functions of tests/pin_cases.py that read the geometry under the
vertical, forward, backward and roll motions, plus two cases the default stream cannot reach:
  * wide_baseline: keyframe 0 on ground truth, one updateKeyframe with frame 40 (forward, backward) -- depth ratios outside
    doLineStereo's rescale gate, sample points outside the image;
  * propagation_collisions: a random map propagated to frame 8 (forward, backward) without and with a tracking mask, and once
    more with every validity_counter at 200 -- occluded sources skipped, targets replaced by nearer sources, merged validity
    capped (DepthMap.cpp:588-631).
Every observation is checked against tests/golden/ref_pin_motions_320x240.npz, recorded from oracle/_ref/liblsd_ref.so by
python -m tests.golden.make_golden_ref_pin_motions.

Non-vacuity: the C restatement's branch counters (oracle/lsd_oracle.h, LSDO_BR_*) show that each (motion, case) reaches the
branches listed for it in REACHES at least that many times, and each motion's record differs from the default record."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import motions
from tests import pin_cases as pin

PAIRS = pin.MOTION_PAIRS

# (motion, case) -> {branch: at least this many runs} on the C restatement (pyoracle.BRANCHES), about half the measured count.
# prepare_for_stereo and se3_single_evaluation run no depth-map pass: they read the motion through the frames and poses only.
REACHES = {
    ("vertical", "prepare_for_stereo"): dict(),
    ("vertical", "depthmap_update_sequence"):
        dict(depth_y=10000, clip_right=40, clip_bottom=1000, subpixel_pre=4000, subpixel_post=5000),
    ("vertical", "depthmap_random_init_every_branch"):
        dict(depth_y=20000, epl_crop=10, clip_right=100, clip_bottom=1000, subpixel_pre=6000, subpixel_post=10000),
    ("vertical", "depthmap_individual_passes"):
        dict(depth_y=10000, clip_right=10, clip_bottom=100, subpixel_pre=5000, subpixel_post=5000),
    ("vertical", "create_keyframe_and_finalize"):
        dict(depth_y=20000, epl_crop=20, clip_left=40, clip_right=10, clip_top=400, clip_bottom=500, subpixel_pre=10000,
             subpixel_post=10000, prop_merge=60),
    ("vertical", "se3_single_evaluation"): dict(),
    ("vertical", "se3_track_scalar"): dict(depth_y=10000, clip_right=50, clip_bottom=1000, subpixel_pre=3000, subpixel_post=6000),
    ("vertical", "bench_loop_with_keyframe_changes"):
        dict(depth_y=30000, epl_crop=1000, clip_right=100, clip_bottom=3000, subpixel_pre=10000, subpixel_post=20000,
             prop_merge=200),
    ("forward", "prepare_for_stereo"): dict(),
    ("forward", "depthmap_update_sequence"):
        dict(depth_x=6000, depth_y=4000, firstx_gate=60, subpixel_pre=5000, subpixel_post=5000),
    ("forward", "depthmap_random_init_every_branch"):
        dict(depth_x=10000, depth_y=10000, firstx_gate=100, epl_crop=20, subpixel_pre=7000, subpixel_post=10000),
    ("forward", "depthmap_individual_passes"):
        dict(depth_x=6000, depth_y=3000, firstx_gate=8, subpixel_pre=4000, subpixel_post=4000),
    ("forward", "create_keyframe_and_finalize"):
        dict(depth_x=10000, depth_y=9000, firstx_gate=100, epl_crop=1000, clip_left=300, clip_right=100, clip_top=300,
             clip_bottom=200, subpixel_pre=10000, subpixel_post=10000, prop_merge=1000),
    ("forward", "se3_single_evaluation"): dict(),
    ("forward", "se3_track_scalar"): dict(depth_x=6000, depth_y=4000, firstx_gate=60, subpixel_pre=4000, subpixel_post=5000),
    ("forward", "bench_loop_with_keyframe_changes"):
        dict(depth_x=20000, depth_y=10000, firstx_gate=300, epl_crop=6000, subpixel_pre=10000, subpixel_post=20000,
             prop_merge=3000),
    ("forward", "wide_baseline"):
        dict(depth_x=6000, depth_y=4000, firstx_gate=50, rescale_gate=20, subpixel_pre=5000, subpixel_post=5000),
    ("forward", "propagation_collisions"): dict(prop_skip=800, prop_invalidate=600, prop_merge=5000, prop_merge_cap=1000),
    ("backward", "prepare_for_stereo"): dict(),
    ("backward", "depthmap_update_sequence"):
        dict(depth_x=6000, depth_y=3000, clip_left=100, clip_right=300, clip_top=400, clip_bottom=400, subpixel_pre=4000,
             subpixel_post=4000),
    ("backward", "depthmap_random_init_every_branch"):
        dict(depth_x=10000, depth_y=7000, rescale_gate=1, near_clamp=20, epl_crop=30, clip_left=1000, clip_right=1000,
             clip_top=1000, clip_bottom=1000, subpixel_pre=5000, subpixel_post=9000),
    ("backward", "depthmap_individual_passes"):
        dict(depth_x=5000, depth_y=3000, clip_left=100, clip_right=100, clip_top=100, clip_bottom=200, subpixel_pre=4000,
             subpixel_post=4000),
    ("backward", "create_keyframe_and_finalize"):
        dict(depth_x=10000, depth_y=7000, clip_left=300, clip_right=500, clip_top=400, clip_bottom=600, subpixel_pre=10000,
             subpixel_post=10000),
    ("backward", "se3_single_evaluation"): dict(),
    ("backward", "se3_track_scalar"):
        dict(depth_x=6000, depth_y=3000, clip_left=200, clip_right=300, clip_top=500, clip_bottom=600, subpixel_pre=4000,
             subpixel_post=5000),
    ("backward", "bench_loop_with_keyframe_changes"):
        dict(depth_x=10000, depth_y=10000, near_clamp=1, epl_crop=10, clip_left=600, clip_right=1000, clip_top=1000,
             clip_bottom=1000, subpixel_pre=10000, subpixel_post=10000),
    ("backward", "wide_baseline"):
        dict(depth_x=1000, depth_y=700, rescale_gate=5000, clip_right=100, clip_top=40, clip_bottom=90, subpixel_pre=1000,
             subpixel_post=1000),
    ("backward", "propagation_collisions"): dict(prop_skip=400, prop_invalidate=300, prop_merge=2000, prop_merge_cap=800),
    ("roll", "prepare_for_stereo"): dict(),
    ("roll", "depthmap_update_sequence"):
        dict(depth_x=10000, clip_right=200, clip_bottom=200, subpixel_pre=5000, subpixel_post=5000),
    ("roll", "depthmap_random_init_every_branch"):
        dict(depth_x=20000, epl_crop=20, clip_right=800, clip_bottom=600, subpixel_pre=6000, subpixel_post=9000),
    ("roll", "depthmap_individual_passes"):
        dict(depth_x=10000, clip_right=100, clip_bottom=100, subpixel_pre=4000, subpixel_post=5000),
    ("roll", "create_keyframe_and_finalize"):
        dict(depth_x=20000, epl_crop=400, clip_left=100, clip_right=100, clip_top=200, clip_bottom=100, subpixel_pre=10000,
             subpixel_post=10000, prop_merge=100),
    ("roll", "se3_single_evaluation"): dict(),
    ("roll", "se3_track_scalar"): dict(depth_x=10000, clip_right=400, clip_bottom=300, subpixel_pre=6000, subpixel_post=5000),
    ("roll", "bench_loop_with_keyframe_changes"):
        dict(depth_x=30000, depth_y=1000, epl_crop=2000, clip_right=1000, clip_bottom=1000, subpixel_pre=10000,
             subpixel_post=10000, prop_merge=400),
}

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_MOTIONS)
    return _gold


@pytest.mark.parametrize("motion,case", PAIRS, ids=[f"{m}-{c}" for m, c in PAIRS])
def test_matches_reference_compiled_under_motion(motion, case):
    po.branch_counts_reset()
    pin.run_under_motion(motion, case, _load())
    got = po.branch_counts()
    low = {b: (got[b], n) for b, n in REACHES[(motion, case)].items() if got[b] < n}
    assert not low, f"{motion}/{case}: branches reached fewer times than stated (got, stated): {low}"


@pytest.mark.parametrize("motion", list(motions.MOTIONS))
def test_each_motion_changes_the_recorded_outputs(motion):
    """the record of every motion differs from the default record somewhere: the motion reached the reference's code"""
    g, d = _load(), np.load(pin.GOLD)
    keys = [k for k in g.files if k.startswith(motion + "/") and k[len(motion) + 1:] in d.files]
    assert keys
    differ = [k for k in keys if not np.array_equal(g[k], d[k[len(motion) + 1:]])]
    assert differ, f"{motion}: every observation equals the default record"


# the branches no case of tests/test_ref_pin.py reaches under the default motion (DESIGN.md section 5, Camera motion).  The left
# and top clips of the search segment are not among them: create_keyframe_and_finalize reaches both with the frames it maps on
# the new keyframe.
UNREACHED_BY_DEFAULT = ("depth_y", "firstx_gate", "rescale_gate", "near_clamp", "prop_skip", "prop_invalidate", "prop_merge_cap")


def test_the_motions_reach_what_the_default_does_not():
    """every branch the default cases leave unreached is stated to run in at least one (motion, case), and so are the left and
    top clips under each motion"""
    assert set(REACHES) == set(PAIRS)
    reached = {b for want in REACHES.values() for b, n in want.items() if n > 0}
    assert set(UNREACHED_BY_DEFAULT) <= reached, set(UNREACHED_BY_DEFAULT) - reached
    for m in motions.MOTIONS:
        per_motion = {b for (mm, _), want in REACHES.items() if mm == m for b in want}
        assert {"clip_left", "clip_top"} <= per_motion, m


def test_default_cases_leave_those_branches_unreached(seq_small, frames_small):
    """the claim behind UNREACHED_BY_DEFAULT, on the C restatement: the depth-map cases of tests/test_ref_pin.py under the default
    motion never run those branches"""
    po.set_globals(False)
    po.branch_counts_reset()
    for c in pin.GEOMETRY:
        fn, fl, _ = pin.CASES[c]
        fn(pin.Pin(c), fl, seq_small, frames_small)
    got = po.branch_counts()
    assert all(got[b] == 0 for b in UNREACHED_BY_DEFAULT), {b: got[b] for b in UNREACHED_BY_DEFAULT}
    # reached by tests/test_ref_pin_photometry.py (exposure changes) and the allowNegativeIdepths=0 set of the settings pin
    unreached = pin.UNREACHED_BY_DEFAULT_PHOTOMETRIC
    assert all(got[b] == 0 for b in unreached), {b: got[b] for b in unreached}
    assert got["depth_x"] > 100000 and got["clip_left"] > 0 and got["clip_top"] > 0
