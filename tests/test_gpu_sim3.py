"""GPU parity of the batched Sim3 tracker (SURVEY 8f row 1): Sim3Tracker::trackFrameSim3 and its three hot loops
(Tracking/Sim3Tracker.cpp:149-382, 414-607, 748-856, 992-1047) against the oracle, through the C ABI."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4          # north_star: SE3/Sim3 pose parity <= 1e-4 relative
SUM_TOL = 2e-4           # float sums over up to 77k points in a different (tree) order


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _setup(oracle, w=640, h=480, kfs=((0, 1.0), (6, 1.0), (12, 1.05))):
    seq = synth.Sequence(w, h, seed=1234)
    ctx = abi.Context(w, h, seq.K, max_frames=8)
    of = {}
    for k, sc in kfs:
        img, z = seq.render(k)
        z = (z * sc).astype(np.float32)
        ctx.upload(k, img)
        ctx.set_depth_gt(k, z)
        f = oracle.Frame(k, img, seq.K)
        f.setDepthFromGroundTruth(z)
        of[k] = f
    return seq, ctx, abi.Sim3Tracker(ctx), of


def _init(seq, frame, ref, dt=(0.01, -0.005, 0.004), scale=1.02):
    q = np.concatenate([seq.frame_to_ref_qt(frame, ref), [scale]])
    q[4:7] += dt
    return q


def _sim3_err(a, b):
    a, b = np.asarray(a), np.asarray(b)
    dt = np.linalg.norm(a[4:7] - b[4:7]) / max(np.linalg.norm(b[4:7]), 1e-12)
    ang = 2 * np.arccos(min(1.0, abs(float(np.dot(a[:4], b[:4])))))
    return dt, ang, abs(a[7] - b[7]) / b[7]


def _check_eval(got, want):
    """one Sim3 evaluation: the counts exactly, the normal equations and the residual and affine sums to SUM_TOL"""
    assert got.warpedSize == want.warpedSize
    assert (got.numTermsD, got.numTermsP, got.num_constraints) == (want.numTermsD, want.numTermsP, want.num_constraints)
    A, Aw = np.array(got.A), np.array(want.A)
    assert np.abs(A - Aw).max() <= SUM_TOL * np.abs(Aw).max()
    bb, bw = np.array(got.b), np.array(want.b)
    assert np.abs(bb - bw).max() <= SUM_TOL * np.abs(bw).max() + 1e-3 * np.abs(Aw).max() ** 0.5
    for f in ("sumResD", "sumResP", "mean", "meanD", "meanP", "pointUsage", "affine_a_lastIt"):
        assert abs(getattr(got, f) - getattr(want, f)) <= SUM_TOL * abs(getattr(want, f)), f
    assert abs(got.affine_b_lastIt - want.affine_b_lastIt) <= 2e-2


def test_sim3_eval_matches_oracle(oracle):
    seq, ctx, trk, of = _setup(oracle)
    for (ref, fr), lvl, a, b in (((0, 6), 4, 1.0, 0.0), ((0, 6), 2, 1.0, 0.0), ((6, 0), 1, 0.97, 1.5), ((0, 12), 3, 1.0, 0.0)):
        r2f = np.zeros(8)
        oracle.lib().lsdo_sim3d_inverse(_d(_init(seq, fr, ref)), _d(r2f))
        got = trk.eval(ref, fr, lvl, r2f, a, b)
        want = oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b)
        assert want.warpedSize > 100
        _check_eval(got, want)
    ctx.close()


def _check_track(got, want, res_tol=2e-2):
    assert got.diverged == want.diverged
    assert list(got.numCalcResidualCalls) == list(want.numCalcResidualCalls)
    assert list(got.numCalcWarpUpdateCalls) == list(want.numCalcWarpUpdateCalls)
    dt, ang, ds = _sim3_err(got.frameToRef_qts, want.frameToRef_qts)
    assert dt <= POSE_TOL and ang <= POSE_TOL and ds <= POSE_TOL, (dt, ang, ds)
    H, Hw = np.array(got.lastSim3Hessian), np.array(want.lastSim3Hessian)
    assert np.abs(H - Hw).max() <= 1e-3 * np.abs(Hw).max()
    for f in ("lastResidual", "lastDepthResidual", "lastPhotometricResidual"):
        assert abs(getattr(got, f) - getattr(want, f)) <= res_tol * abs(getattr(want, f)) + 1e-7, f
    assert abs(got.pointUsage - want.pointUsage) <= 1e-3 * want.pointUsage
    assert abs(got.affineEstimation_a - want.affineEstimation_a) <= 0.25 * res_tol
    assert abs(got.affineEstimation_b - want.affineEstimation_b) <= 25 * res_tol


def _oracle_track(oracle, ref, fr, init, lo=4, hi=1):
    """-> (the reference's arithmetic, the same with the five affine-lighting sums accumulated in double).
    calcSim3Buffers adds ~60k terms of ~1.6e4 into fp32 sums of ~1e9 (ulp 64): a_lastIt / b_lastIt carry that noise, it is
    fed back through every accepted step and moves the final residuals by up to ~6e-3 relative -- the kernel's tree sums
    do not have it.  Pose, scale, Hessian and iteration counts are checked against the reference arithmetic; the residuals
    tightly against the exact-sum twin and loosely against the reference arithmetic."""
    want = oracle.sim3_track(ref, fr, init, lo, hi)
    oracle.set_globals(exactAffineSums=1)
    try:
        exact = oracle.sim3_track(ref, fr, init, lo, hi)
    finally:
        oracle.set_globals()
    return want, exact


def test_track_frame_sim3_matches_oracle(oracle):
    seq, ctx, trk, of = _setup(oracle)
    for ref, fr in ((0, 6), (6, 0)):
        init = _init(seq, fr, ref)
        est = trk.trackFrameSim3(ref, fr, init, 4, 1)
        want, exact = _oracle_track(oracle, of[ref], of[fr], init)
        assert not want.diverged and abs(want.frameToRef_qts[7] - 1) < 5e-3
        _check_track(trk.last, want)
        _check_track(trk.last, exact, res_tol=5e-4)
        assert np.array_equal(est, np.array(trk.last.frameToRef_qts))
        assert np.allclose(trk.lastSim3Hessian, trk.lastSim3Hessian.T, rtol=1e-5)
    ctx.close()


def test_track_frame_sim3_scale_and_level_range(oracle):
    """keyframe 12 carries a 1.05x larger map; also the (3, 2) level range of SlamSystem::testConstraint's coarse check"""
    seq, ctx, trk, of = _setup(oracle)
    init = np.concatenate([seq.frame_to_ref_qt(12, 0), [1.0]])
    trk.trackFrameSim3(0, 12, init, 4, 1)
    want, exact = _oracle_track(oracle, of[0], of[12], init)
    assert abs(want.frameToRef_qts[7] - 1 / 1.05) < 5e-3
    _check_track(trk.last, want)
    _check_track(trk.last, exact, res_tol=5e-4)
    trk.trackFrameSim3(0, 12, init, 3, 2)
    want, exact = _oracle_track(oracle, of[0], of[12], init, 3, 2)
    assert want.numCalcResidualCalls[4] == 0 and want.numCalcResidualCalls[1] == 0
    _check_track(trk.last, want)
    _check_track(trk.last, exact, res_tol=5e-4)
    ctx.close()


def test_track_frame_sim3_batch(oracle):
    """all ordered pairs in one launch == the same problems one by one (bit-identical) == the oracle"""
    seq, ctx, trk, of = _setup(oracle)
    pairs = [(a, b) for a in of for b in of if a != b]
    inits = np.array([_init(seq, fr, ref) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    for (ref, fr), init, r in zip(pairs, inits, res):
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        assert bytes(trk.last) == bytes(r)
        _check_track(r, oracle.sim3_track(of[ref], of[fr], init, 4, 1))
    ctx.close()


def test_track_frame_sim3_early_returns(oracle):
    seq, ctx, trk, of = _setup(oracle)
    far = np.array([0, 0, 0, 1, 50.0, 0, 0, 1.0])
    trk.trackFrameSim3(0, 6, far, 4, 1)
    want = oracle.sim3_track(of[0], of[6], far, 4, 1)
    assert want.diverged and trk.diverged
    assert np.allclose(trk.last.frameToRef_qts, [0, 0, 0, 1, 0, 0, 0, 1]) and not trk.lastSim3Hessian.any()
    with pytest.raises(abi.LsdGpuError):
        img, _ = seq.render(3)
        ctx.upload(3, img)                       # no depth on frame 3
        trk.trackFrameSim3(0, 3, far, 4, 1)
    ctx.close()


def test_cluster_sizes_agree(oracle, monkeypatch):
    """the per-problem cluster size only changes how the level is split: decisions and iteration counts are identical,
    sums differ by float re-association only"""
    seq, ctx, trk, of = _setup(oracle)
    init = _init(seq, 6, 0)
    out = {}
    for cs in (1, 2, 4, 8):
        monkeypatch.setenv("LSDGPU_SIM3_CLUSTER", str(cs))
        trk.trackFrameSim3(0, 6, init, 4, 1)
        out[cs] = trk.last
    for cs in (1, 2, 4):
        assert list(out[cs].numCalcResidualCalls) == list(out[8].numCalcResidualCalls)
        dt, ang, ds = _sim3_err(out[cs].frameToRef_qts, out[8].frameToRef_qts)
        assert max(dt, ang, ds) < POSE_TOL
    ctx.close()
