"""PIN of the oracle under camera motions other than the default (tests/motions.py).

Every other pin runs the synthetic stream's default twist: mostly sideways, so every epipolar line the depth map searches is close
to horizontal and points the same way, the epipole lies far outside the image, and propagation never lands two sources at
inconsistent depths on one pixel.  This module runs the case functions of tests/test_ref_pin.py that read the geometry under the
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
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import motions
from tests import test_ref_pin as pin

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin_motions_320x240.npz")

WIDE_BASELINE_FRAME = 40
PROPAGATION_FRAME = 8


def wide_baseline(p, fl, seq, frames):
    """updateKeyframe with one frame far from the keyframe, on ground-truth depth and poses"""
    s = pin.Side(seq, frames, fl, "gt")
    k = WIDE_BASELINE_FRAME
    s.add_frame(k, pin._gt_qts(seq, k))
    s.dm.updateKeyframe([s.fr[k]])
    assert p.hyp(f"updateKeyframe[{k}]", s.dm.current()) > 10000


def propagation_collisions(p, fl, seq, frames):
    """propagateDepth of a random map: its sources disagree about depth, so under a motion along the optical axis many land on one
    pixel at inconsistent depths (DepthMap.cpp:588-601); validity 200 makes every merge exceed the cap of :626"""
    k = PROPAGATION_FRAME
    mask = (np.random.default_rng(8).random((seq.h // 2, seq.w // 2)) > 0.15).astype(np.uint8)
    for what, m, validity in (("no mask", None, None), ("mask", mask, None), ("validity 200", None, 200)):
        s = pin.Side(seq, frames, fl, "random")
        if validity is not None:
            cur = s.dm.current().copy()
            cur["validity_counter"][cur["isValid"] != 0] = validity
            s.dm.set_current(cur)
        s.add_frame(k, pin._gt_qts(seq, k), mask=m)
        s.dm.propagateDepth(s.fr[k])
        assert p.hyp(f"propagateDepth[{k}] {what}", s.dm.current()) > 5000


# the case functions of tests/test_ref_pin.py that read the camera motion
GEOMETRY = ("prepare_for_stereo", "depthmap_update_sequence", "depthmap_random_init_every_branch", "depthmap_individual_passes",
            "create_keyframe_and_finalize", "se3_single_evaluation", "se3_track_scalar", "bench_loop_with_keyframe_changes")
# case -> (function, C-restatement flavour, reference-compiled flavour), as test_ref_pin.CASES
CASES = {c: pin.CASES[c] for c in GEOMETRY}
CASES["wide_baseline"] = (wide_baseline, False, "ref")
CASES["propagation_collisions"] = (propagation_collisions, False, "ref")
ONLY = {"wide_baseline": ("forward", "backward"), "propagation_collisions": ("forward", "backward")}
PAIRS = [(m, c) for m in motions.MOTIONS for c in CASES if m in ONLY.get(c, (m,))]

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


_streams: dict = {}


def stream(motion):
    if motion not in _streams:
        seq = motions.sequence(motion)
        _streams[motion] = (seq, motions.Frames(seq))
    return _streams[motion]


def _run(motion, case, gold):
    """runs one case under one motion on the C restatement (gold = the record) or on the reference-compiled library
    (gold = None); returns the case's Pin"""
    fn, fl, ref_fl = CASES[case]
    fl = ref_fl if gold is None else fl
    seq, frames = stream(motion)
    p = pin.Pin(f"{motion}/{case}", gold)
    try:
        fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record():
    """every (motion, case) on the reference-compiled library (needs oracle/_ref): the arrays of the golden file"""
    out = {}
    for m, c in PAIRS:
        out.update(_run(m, c, None).rec)
    return out


_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(GOLD)
    return _gold


@pytest.mark.parametrize("motion,case", PAIRS, ids=[f"{m}-{c}" for m, c in PAIRS])
def test_matches_reference_compiled_under_motion(motion, case):
    po.branch_counts_reset()
    _run(motion, case, _load())
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
    for c in GEOMETRY:
        fn, fl, _ = pin.CASES[c]
        fn(pin.Pin(c), fl, seq_small, frames_small)
    got = po.branch_counts()
    assert all(got[b] == 0 for b in UNREACHED_BY_DEFAULT), {b: got[b] for b in UNREACHED_BY_DEFAULT}
    assert got["depth_x"] > 100000 and got["clip_left"] > 0 and got["clip_top"] > 0
