"""PIN of the oracle's Sim3 tracker and permaRef path on keyframes the mapper finished, under every camera motion.

The other pins give the Sim3 tracker ground-truth depth: one variance at a level, scales between keyframes of about 1.  A
restatement that read the reference point's variance `s` where the reference reads the frame pixel's `sv`
(Sim3Tracker.cpp:527-542, 762-835) would compute the same numbers there.  Here oracle/cpu_stream.py's loop maps 16 frames of each
stream (the default twist and the motions of tests/motions.py) with a keyframe every 5 frames, and the cases of
tests/pin_cases.py run on its finished keyframes 0, 5 and 10 (semi-dense, variances over orders of magnitude, rescaled by
createKeyFrame):
  * sim3_eval_mapped: one calcSim3Buffers + calcSim3WeightsAndResidual + calcSim3LGS per ordered pair, level 4..1, perturbed
    and not, two affine estimates, and once under var_weight = 2.5, huber_d = 1.5;
  * sim3_track_mapped: trackFrameSim3 per ordered pair over levels 4..1 and 3..2;
  * perma_mapped: Frame::setPermaRef of each keyframe, checkPermaRefOverlap at seeded random poses and at ground truth,
    trackFrameOnPermaref of frame 12 from ground truth and from identity;
  * adversarial_map (default, forward): the active keyframe's map edited to the value edges of Frame::setDepth, with the three
    calls above on it.
Every observation is checked against tests/golden/ref_pin_sim3_320x240.npz, recorded from oracle/_ref/liblsd_ref.so by
python -m tests.golden.make_golden_ref_pin_sim3: bit for bit, except poses read back from Sophus' non-unit quaternion (1e-12).

Non-vacuity: the C restatement's counters (oracle/lsd_oracle.h, LSDO_S3_*) reach the minima of REACHES in each (motion, case);
the reference point's variance and the frame pixel's differ on most warped points; the keyframes are rescaled."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import motions
from tests import pin_cases as pin

PAIRS = pin.SIM3_PAIRS

# (motion, case) -> {counter: at least this many} on the C restatement (pyoracle.SIM3_BRANCHES), about half the measured count.
# ldlt7_pivot: every 7x7 solve of trackFrameSim3 on these keyframes permutes (ldlt7_pivot == ldlt7_solve in each case), so the
# reference's pivoted LDLT and the device's unpivoted first solve always eliminate in different orders.
REACHES = {
    ("default", "sim3_eval_mapped"):
        dict(sim3_outside=5000, sim3_no_depth=10000, sim3_usage_clamp=90000, sim3_affine_clamp=100000, sim3_huber=40000),
    ("default", "sim3_track_mapped"):
        dict(sim3_outside=9000, sim3_no_depth=10000, sim3_usage_clamp=100000, sim3_affine_clamp=90000, sim3_huber=6000,
             ldlt7_pivot=90),
    ("default", "perma_mapped"): dict(perma_outside=500, perma_usage_clamp=500),
    ("default", "adversarial_map"):
        dict(sim3_outside=2000, sim3_no_depth=20000, sim3_usage_clamp=100000, sim3_affine_clamp=90000, sim3_huber=50000,
             ldlt7_pivot=10, perma_outside=200, perma_usage_clamp=200),
    ("vertical", "sim3_eval_mapped"):
        dict(sim3_outside=5000, sim3_no_depth=10000, sim3_usage_clamp=90000, sim3_affine_clamp=100000, sim3_huber=40000),
    ("vertical", "sim3_track_mapped"):
        dict(sim3_outside=8000, sim3_no_depth=10000, sim3_usage_clamp=100000, sim3_affine_clamp=100000, sim3_huber=9000,
             ldlt7_pivot=90),
    ("vertical", "perma_mapped"): dict(perma_outside=500, perma_usage_clamp=500),
    ("forward", "sim3_eval_mapped"):
        dict(sim3_outside=6000, sim3_no_depth=10000, sim3_usage_clamp=90000, sim3_affine_clamp=100000, sim3_huber=40000),
    ("forward", "sim3_track_mapped"):
        dict(sim3_outside=10000, sim3_no_depth=10000, sim3_usage_clamp=100000, sim3_affine_clamp=100000, sim3_huber=10000,
             ldlt7_pivot=90),
    ("forward", "perma_mapped"): dict(perma_outside=500, perma_usage_clamp=400),
    ("forward", "adversarial_map"):
        dict(sim3_outside=900, sim3_no_depth=20000, sim3_usage_clamp=100000, sim3_affine_clamp=100000, sim3_huber=50000,
             ldlt7_pivot=10, perma_outside=200, perma_usage_clamp=200),
    ("backward", "sim3_eval_mapped"):
        dict(sim3_outside=10000, sim3_no_depth=10000, sim3_usage_clamp=80000, sim3_affine_clamp=100000, sim3_huber=30000),
    ("backward", "sim3_track_mapped"):
        dict(sim3_outside=10000, sim3_no_depth=10000, sim3_usage_clamp=100000, sim3_affine_clamp=100000, sim3_huber=9000,
             ldlt7_pivot=90),
    ("backward", "perma_mapped"): dict(perma_outside=500, perma_usage_clamp=700),
    ("roll", "sim3_eval_mapped"):
        dict(sim3_outside=7000, sim3_no_depth=10000, sim3_usage_clamp=90000, sim3_affine_clamp=100000, sim3_huber=40000),
    ("roll", "sim3_track_mapped"):
        dict(sim3_outside=10000, sim3_no_depth=10000, sim3_usage_clamp=100000, sim3_affine_clamp=100000, sim3_huber=9000,
             ldlt7_pivot=80),
    ("roll", "perma_mapped"): dict(perma_outside=500, perma_usage_clamp=400),
}

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_SIM3)
    return _gold


@pytest.mark.parametrize("motion,case", PAIRS, ids=[f"{m}-{c}" for m, c in PAIRS])
def test_sim3_and_perma_match_reference_compiled(motion, case):
    po.sim3_branch_counts_reset()
    pin.run_sim3(motion, case, _load())
    got = po.sim3_branch_counts()
    low = {b: (got[b], n) for b, n in REACHES[(motion, case)].items() if got[b] < n}
    assert not low, f"{motion}/{case}: counters below their stated minimum (got, stated): {low}"


def test_every_counter_is_reached():
    """every counter of pyoracle.SIM3_BRANCHES has a stated minimum somewhere, and the usage clamp and the frame pixels without
    depth have one under forward and under backward"""
    assert set(REACHES) == set(PAIRS)
    reached = {b for want in REACHES.values() for b, n in want.items() if n > 0}
    assert set(po.SIM3_BRANCHES) - {"ldlt7_solve"} <= reached, set(po.SIM3_BRANCHES) - reached
    for m in ("forward", "backward"):
        for b in ("sim3_usage_clamp", "sim3_no_depth", "perma_usage_clamp"):
            assert any(REACHES[(m, c)].get(b, 0) > 0 for c in pin.SIM3_CASES if (m, c) in REACHES), (m, b)


def _var_mismatch(m, ref, fr, lvl):
    """(warped points, of them on a frame pixel with depth whose variance differs from the reference point's) of calcSim3Buffers'
    warp (Sim3Tracker.cpp:478-541) from keyframe ref onto keyframe fr at the chained pose, restated in numpy"""
    pos, _, colvar, _ = m.of[ref].point_cloud(lvl)
    rot, t, roll = np.zeros(9, np.float32), np.zeros(3, np.float32), np.zeros(4, np.float32)
    fp = C.POINTER(C.c_float)
    q = np.ascontiguousarray(m.ref_to_frame(ref, fr, perturb=False))
    po.lib(False).lsdo_sim3_pose_constants(po._dp(q), rot.ctypes.data_as(fp), t.ctypes.data_as(fp), roll.ctypes.data_as(fp))
    W = pos @ rot.reshape(3, 3).T + t
    K = m.of[fr].K(lvl)[0]
    w, h = m.of[fr].size(lvl)
    u, v = W[:, 0] / W[:, 2] * K[0, 0] + K[0, 2], W[:, 1] / W[:, 2] * K[1, 1] + K[1, 2]
    inside = (u > 1) & (v > 1) & (u < w - 2) & (v < h - 2)
    idx = (u[inside] + 0.5).astype(np.int64) + w * (v[inside] + 0.5).astype(np.int64)
    sv = m.of[fr].idepthVar(lvl).ravel()[idx]
    return int(inside.sum()), int(((sv > 0) & (sv != colvar[inside, 1])).sum())


@pytest.mark.parametrize("motion", pin.SIM3_MOTIONS)
def test_mapped_keyframes_tell_the_two_variances_apart(motion):
    """on every ordered pair and level, most warped points land on a frame pixel with depth whose variance is not the reference
    point's own (so swapping `s` and `sv` changes the sums), and the keyframes were rescaled by createKeyFrame"""
    po.set_globals(False)
    seq, frames = motions.stream(motion)
    m = pin.mapped(False, seq, frames)
    for ref, fr in m.pairs():
        for lvl in (4, 3, 2, 1):
            n, differ = _var_mismatch(m, ref, fr, lvl)
            assert n > 10 and differ > 0.5 * n, (ref, fr, lvl, n, differ)
    scales = [q[7] for q in m.c2w.values()]
    assert max(scales) / min(scales) > 1.2, scales
    var = m.of[m.kfs[0]].idepthVar(0)
    assert np.unique(var[var > 0]).size > 100


@pytest.mark.parametrize("motion", list(motions.MOTIONS))
def test_each_motion_changes_the_recorded_outputs(motion):
    """the record of each motion differs from the default's: the motion reached the reference's Sim3 and permaRef code"""
    g = _load()
    keys = [k for k in g.files if k.startswith(f"{motion}/sim3_track_mapped/")]
    assert keys
    assert any(not np.array_equal(g[k], g[f"{motions.DEFAULT}/" + k.split("/", 1)[1]]) for k in keys), motion


@pytest.mark.parametrize("motion,ref,fr,lo,hi", sorted(pin.POSE_SENSITIVE_DEPTH_RESIDUAL))
def test_pose_sensitive_depth_residuals_are_ill_conditioned(motion, ref, fr, lo, hi):
    """the calls whose lastDepthResidual the device tests hold only to the reference tolerance: moving the final translation by
    pin.SENSITIVE_TRANSLATION (well inside the pose tolerance) moves that residual by more than 2e-3, with no term changing its
    pixel or depth status -- so a 4.5e-3 gap between two poses 7e-6 apart is the residual's conditioning, not a kernel fault"""
    po.set_globals(False)
    seq, frames = motions.stream(motion)
    dmax, cmax = pin.depth_residual_sensitivity(pin.mapped(False, seq, frames), ref, fr, lo, hi)
    assert dmax > 2e-3 and cmax == 0, (dmax, cmax)
