"""Shared helpers for the parity tests: drive the oracle and the CUDA path through the same call sequence, and compare what
each kind of call returns (one check per kind of result, with the tolerances of BASELINE.json's north_star)."""
import contextlib

import numpy as np

from oracle.pyoracle import _dp
from oracle.replay import pose_err  # noqa: F401  (re-exported: the tests' pose comparison)

IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)

EVAL_RTOL = 2e-4         # one SE3 evaluation: the sums differ by summation order only (sequential on the CPU, a tree on the GPU)
SUM_TOL = 2e-4           # one Sim3 evaluation: float sums over up to 77k points in a different (tree) order
POSE_TOL = 1e-4          # north_star: SE3/Sim3 pose parity <= 1e-4 relative
PERMA_ANG_TOL = 2e-6     # trackFrameOnPermaref: rotation angle in rad (translation: POSE_TOL)
OVERLAP_RTOL, OVERLAP_ATOL = 2e-5, 1e-6                # checkPermaRefOverlap
SE3_EVAL_FIELDS = ("lsError", "meanWeightedRes", "meanUnweightedRes", "pointUsage", "affine_a_lastIt", "affine_b_lastIt",
                   "meanRes", "sxx", "syy", "sx", "sy", "sw")
CLOUD_FILTERS = [None, {"minNearSupport": 1}, {"minNearSupport": 9}, {"scaledDepthVarTH": 0.01, "absDepthVarTH": 0.02},
                 {"scaledDepthVarTH": 100.0, "absDepthVarTH": 100.0}]


def hyp_equal_report(a: np.ndarray, b: np.ndarray):
    """Compare two hypothesis fields (structured arrays).  Fields other than the flags only count where valid."""
    rep = {}
    va, vb = a["isValid"] > 0, b["isValid"] > 0
    rep["valid_mismatch"] = int((va != vb).sum())
    rep["blacklist_mismatch"] = int((a["blacklisted"] != b["blacklisted"]).sum())
    both = va & vb
    for f in ("idepth", "idepth_var", "idepth_smoothed", "idepth_var_smoothed", "nextStereoFrameMinID"):
        x, y = a[f][both], b[f][both]
        rep[f + "_bitdiff"] = int((x.view(np.uint32) != y.view(np.uint32)).sum())
        den = np.maximum(np.abs(x), 1e-12)
        rep[f + "_maxrel"] = float(np.max(np.abs(x - y) / den)) if x.size else 0.0
    rep["validity_mismatch"] = int((a["validity_counter"][both] != b["validity_counter"][both]).sum())
    rep["n_valid"] = int(both.sum())
    return rep


def rot_angle(qt):
    return 2 * np.arccos(min(1.0, abs(float(qt[3]))))


# ---- Sim3 / SE3 pose arithmetic of the oracle -----------------------------------------------------------------------------
def _pose_op(oracle, fn, n, *args):
    out = np.zeros(n, np.float64)
    arrs = [np.ascontiguousarray(a, np.float64) for a in args]
    getattr(oracle.lib(), fn)(*[_dp(a) for a in arrs], _dp(out))
    return out


def se3_inverse(oracle, qt):
    return _pose_op(oracle, "lsdo_se3d_inverse", 7, qt)


def sim3_inverse(oracle, qts):
    return _pose_op(oracle, "lsdo_sim3d_inverse", 8, qts)


def sim3_mul(oracle, a, b):
    return _pose_op(oracle, "lsdo_sim3d_mul", 8, a, b)


def sim3_init(seq, frame, ref, dt=(0.01, -0.005, 0.004), scale=1.02):
    """the ground-truth frame-to-reference Sim3 with its translation and scale perturbed"""
    q = np.concatenate([seq.frame_to_ref_qt(frame, ref), [scale]])
    q[4:7] += dt
    return q


def sim3_err(a, b):
    """(relative translation error, rotation angle error in rad, relative scale error) between two (q,t,s) poses"""
    a, b = np.asarray(a), np.asarray(b)
    dt = np.linalg.norm(a[4:7] - b[4:7]) / max(np.linalg.norm(b[4:7]), 1e-12)
    ang = 2 * np.arccos(min(1.0, abs(float(np.dot(a[:4], b[:4])))))
    return dt, ang, abs(a[7] - b[7]) / b[7]


# ---- both sides in one state ------------------------------------------------------------------------------------------------
class Pair:
    """The same state on both sides: oracle objects + a GPU context, driven through identical calls."""

    def __init__(self, ctx, oracle, seq, frames, init="gt"):
        from lsd_slam_b200 import abi
        self.ctx, self.o, self.seq, self.frames = ctx, oracle, seq, frames
        img0, d0 = frames[0]
        self.okf = oracle.Frame(0, img0, seq.K)
        self.odm = oracle.DepthMap(seq.w, seq.h, seq.K)
        self.gdm = abi.DepthMap(ctx)
        ctx.upload(0, img0)
        if init == "gt":
            self.okf.setDepthFromGroundTruth(d0)
            self.odm.initializeFromGTDepth(self.okf)
            ctx.set_depth_gt(0, d0)
            self.gdm.initializeFromGTDepth(0)
        else:
            self.odm.initializeRandomly(self.okf)            # glibc rand() on the host (DepthMap.cpp:898)
            self.gdm.setHypotheses(0, self.odm.current().copy(), reactivated=False, do_set_depth=True)
        self.oframes = {0: self.okf}

    def add_frame(self, k, pose_qt=None, itr=0.0):
        """upload frame k on both sides with the SAME pose (ground truth unless given)"""
        img, _ = self.frames[k]
        of = self.o.Frame(k, img, self.seq.K)
        qts = np.concatenate([self.seq.frame_to_ref_qt(k) if pose_qt is None else pose_qt, [1.0]])
        of.set_thisToParent(qts, self.okf)
        self.ctx.upload(k, img)
        self.ctx.set_pose(k, qts, 0, itr)
        # an untracked oracle frame has initialTrackedResidual == 0: keep itr = 0 on the GPU side too
        self.oframes[k] = of
        return of

    def sync_counters(self):
        t, m = self.o.lib().lsdo_frame_numFramesTrackedOnThis(self.okf.ptr), self.o.lib().lsdo_frame_numMappedOnThis(self.okf.ptr)
        self.ctx.set_counters(0, t, m)

    def compare(self, exact=True, rtol=1e-3, max_flag_mismatch=0):
        a, b = self.gdm.current(), self.odm.current()
        rep = hyp_equal_report(a, b)
        assert rep["valid_mismatch"] <= max_flag_mismatch, rep
        assert rep["blacklist_mismatch"] <= max_flag_mismatch, rep
        assert rep["validity_mismatch"] <= max_flag_mismatch, rep
        for f in ("idepth", "idepth_var", "idepth_smoothed", "idepth_var_smoothed", "nextStereoFrameMinID"):
            if exact:
                assert rep[f + "_bitdiff"] == 0, rep
            else:
                assert rep[f + "_maxrel"] <= rtol or rep[f + "_bitdiff"] <= max_flag_mismatch, rep
        return rep


def tracked_pair(ctx, oracle, seq, frames, ks, init="gt"):
    """frames tracked BY THE ORACLE; the oracle's pose, residual and good-mask are pushed to the GPU side so that
    both depth maps see identical inputs"""
    p = Pair(ctx, oracle, seq, frames, init)
    last = IDENT
    for k in ks:
        img, _ = frames[k]
        of = oracle.Frame(k, img, seq.K)
        r = oracle.se3_track(p.okf, of, last)
        last = np.array(r.frameToRef_qt)
        p.oframes[k] = of
        ctx.upload(k, img)
        ctx.set_pose(k, of.thisToParent(), 0, r.initialTrackedResidual)
    return p


def new_depth(p):
    """the keyframe's depth was read since its last update (importFrame, SlamSystem.cpp:907-912), on both sides"""
    p.o.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
    p.ctx.L.lsdgpu_ref_import(p.ctx.ptr, 0)
    p.sync_counters()


def kf_depth_equal(ctx, okf, fid):
    """Frame::setDepth's pyramids (what the tracker reads) bit for bit"""
    from lsd_slam_b200 import abi
    for lvl in range(5):
        assert np.array_equal(ctx.download(fid, abi.BUF_IDEPTH, lvl).view(np.uint32), okf.idepth(lvl).view(np.uint32)), lvl
        assert np.array_equal(ctx.download(fid, abi.BUF_IDEPTH_VAR, lvl).view(np.uint32), okf.idepthVar(lvl).view(np.uint32)), lvl


@contextlib.contextmanager
def under(oracle, g, w, h, K, max_frames=12):
    """a context created with the settings g, and the oracle switched to them; both back at the defaults afterwards"""
    from lsd_slam_b200 import abi
    oracle.set_globals(**g)
    ctx = abi.Context(w, h, K, max_frames=max_frames, **g)
    try:
        yield ctx
    finally:
        ctx.close()
        oracle.set_globals()


# ---- SE3 tracker --------------------------------------------------------------------------------------------------------------
def check_se3_eval(g, o, affine_b_noise=0.0):
    """one SE3 evaluation: the counts exactly, the normal equations and the statistics to EVAL_RTOL, affine b (a difference of
    fp32 sums that cancel) to 5e-3 grey levels plus the caller's `affine_b_noise`.  Where the oracle's statistics are not finite
    (no or one warped point): NaN in the same fields, the finite ones to EVAL_RTOL, and the counts."""
    if not all(np.isfinite(getattr(o, f)) for f in SE3_EVAL_FIELDS):
        assert g.warpedSize == o.warpedSize and g.goodCount == o.goodCount and g.badCount == o.badCount
        for f in SE3_EVAL_FIELDS:
            a, b = getattr(g, f), getattr(o, f)
            assert np.isnan(a) == np.isnan(b) and (np.isnan(b) or abs(a - b) <= EVAL_RTOL * abs(b) + 1e-6), (f, a, b)
        return
    A_g, A_o = np.array(g.A).reshape(6, 6), np.array(o.A).reshape(6, 6)
    scale = np.sqrt(np.outer(np.diag(A_o), np.diag(A_o)))
    assert np.abs(A_g - A_o).max() <= EVAL_RTOL * scale.max()
    assert np.all(np.abs(A_g - A_o) <= EVAL_RTOL * scale + 1e-12)
    b_g, b_o = np.array(g.b), np.array(o.b)
    assert np.all(np.abs(b_g - b_o) <= EVAL_RTOL * np.sqrt(np.diag(A_o)) * np.sqrt(max(o.lsError, 1e-12)) + 1e-9)
    assert g.warpedSize == o.warpedSize
    assert g.goodCount == o.goodCount and g.badCount == o.badCount
    for f in ("lsError", "meanWeightedRes", "meanUnweightedRes", "pointUsage", "affine_a_lastIt", "sxx", "syy", "sx", "sy", "sw"):
        assert abs(getattr(g, f) - getattr(o, f)) <= EVAL_RTOL * abs(getattr(o, f)) + 1e-7, f
    assert abs(g.affine_b_lastIt - o.affine_b_lastIt) <= 5e-3 + affine_b_noise, (g.affine_b_lastIt, o.affine_b_lastIt, affine_b_noise)
    assert abs(g.meanRes - o.meanRes) <= 1e-4 + EVAL_RTOL * abs(o.meanRes)


def check_se3_track(ctx, trk, fid, pose_g, r, of, diverges=False, noise=(0.0, 0.0), usage_noise=0.0):
    """SE3Tracker::trackFrame of frame `fid` on keyframe 0 (trk, its returned pose_g) against the oracle's result r on the oracle
    frame `of`: the pose to POSE_TOL plus the caller's (translation, rotation) `noise` (the point usage to 1e-4 plus its
    `usage_noise`), the outcome flags and the LM call
    counters exactly, and -- when the reference did not diverge, as `diverges` states -- the residual, point usage, good / bad
    counts, affine estimate, the frame's pose record and the keyframe's counter, and the good-mask"""
    from lsd_slam_b200 import abi
    pose_o = np.array(r.frameToRef_qt)
    dt, ang = pose_err(pose_g, pose_o)
    assert dt <= POSE_TOL + noise[0], (dt, noise[0], pose_g, pose_o)
    assert ang <= POSE_TOL * max(rot_angle(pose_o), 1e-2) + 1e-7 + noise[1], (ang, noise[1])
    assert trk.trackingWasGood == bool(r.trackingWasGood) and trk.diverged == bool(r.diverged)
    assert bool(r.diverged) == diverges
    assert list(trk.last.numCalcResidualCalls) == list(r.numCalcResidualCalls)
    assert list(trk.last.numCalcWarpUpdateCalls) == list(r.numCalcWarpUpdateCalls)
    if r.diverged:
        return
    assert abs(trk.lastResidual - r.lastResidual) <= 1e-3 * abs(r.lastResidual) + 1e-6
    assert abs(trk.pointUsage - r.pointUsage) <= 1e-4 + usage_noise
    assert abs(trk.lastGoodCount - r.lastGoodCount) <= 2 and abs(trk.lastBadCount - r.lastBadCount) <= 2
    assert abs(trk.affineEstimation_a - r.affineEstimation_a) <= 1e-3 and abs(trk.affineEstimation_b - r.affineEstimation_b) <= 5e-2
    _, pid, itr = ctx.get_pose(fid)
    assert pid == 0 and abs(itr - r.initialTrackedResidual) <= 1e-3 * abs(r.initialTrackedResidual) + 1e-6
    assert ctx.get_counters(0)[0] == int(bool(r.trackingWasGood))     # numFramesTrackedOnThis++ if good (SE3Tracker.cpp:479-480)
    assert (ctx.download(fid, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < 1e-3


# ---- Sim3 tracker -------------------------------------------------------------------------------------------------------------
def check_sim3_eval(got, want):
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


def check_sim3_track(got, want, res_tol=2e-2, depth_res_tol=None, pose_noise=0.0):
    """Sim3Tracker::trackFrameSim3: outcome and LM call counters exactly, pose and scale to POSE_TOL, the Hessian, the residuals
    to `res_tol` (lastDepthResidual to `depth_res_tol` where the caller gives one) and the affine estimate in proportion; the
    pose may also differ by the caller's `pose_noise`"""
    assert got.diverged == want.diverged
    assert list(got.numCalcResidualCalls) == list(want.numCalcResidualCalls)
    assert list(got.numCalcWarpUpdateCalls) == list(want.numCalcWarpUpdateCalls)
    dt, ang, ds = sim3_err(got.frameToRef_qts, want.frameToRef_qts)
    assert dt <= POSE_TOL + pose_noise and ang <= POSE_TOL + pose_noise and ds <= POSE_TOL + pose_noise, (dt, ang, ds, pose_noise)
    H, Hw = np.array(got.lastSim3Hessian), np.array(want.lastSim3Hessian)
    assert np.abs(H - Hw).max() <= 1e-3 * np.abs(Hw).max()
    for f in ("lastResidual", "lastDepthResidual", "lastPhotometricResidual"):
        tol = depth_res_tol if f == "lastDepthResidual" and depth_res_tol is not None else res_tol
        assert abs(getattr(got, f) - getattr(want, f)) <= tol * abs(getattr(want, f)) + 1e-7, f
    assert abs(got.pointUsage - want.pointUsage) <= 1e-3 * want.pointUsage
    assert abs(got.affineEstimation_a - want.affineEstimation_a) <= 0.25 * res_tol
    assert abs(got.affineEstimation_b - want.affineEstimation_b) <= 25 * res_tol


def oracle_sim3_track(oracle, ref, fr, init, lo=4, hi=1, g=None):
    """-> (the reference's arithmetic, the same with the five affine-lighting sums accumulated in double), under the settings g
    (default: the defaults).
    calcSim3Buffers adds ~60k terms of ~1.6e4 into fp32 sums of ~1e9 (ulp 64): a_lastIt / b_lastIt carry that noise, it is
    fed back through every accepted step and moves the final residuals by up to ~6e-3 relative -- the kernel's tree sums
    do not have it.  Pose, scale, Hessian and iteration counts are checked against the reference arithmetic; the residuals
    tightly against the exact-sum twin and loosely against the reference arithmetic."""
    g = g or {}
    want = oracle.sim3_track(ref, fr, init, lo, hi)
    oracle.set_globals(exactAffineSums=1, **g)
    try:
        exact = oracle.sim3_track(ref, fr, init, lo, hi)
    finally:
        oracle.set_globals(**g)
    return want, exact


def oracle_sim3_exact(oracle, ref, fr, init, lo=4, hi=1, g=None):
    """the same trackFrameSim3 with EVERY sum of the Sim3 tracker accumulated in double from the same fp32 terms (the affine
    sums, the residual sums, LGS4 / LGS6 A and b: lsdo_globals.exactSim3Sums), under the settings g.  oracle_sim3_track's twin
    makes only the affine sums exact; on some calls the sequential fp32 sums of the normal equations move the reference's pose
    much further (DESIGN.md section 5, Cameras), and the device's tree sums follow the exact values"""
    g = g or {}
    oracle.set_globals(exactSim3Sums=1, **g)
    try:
        return oracle.sim3_track(ref, fr, init, lo, hi)
    finally:
        oracle.set_globals(**g)


# ---- permaRef -----------------------------------------------------------------------------------------------------------------
def check_perma_track(g, o, noise=(0.0, 0.0)):
    """one trackFrameOnPermaref result against the oracle's: the outcome; unless diverged the pose (to POSE_TOL and PERMA_ANG_TOL
    plus the caller's (translation, rotation) `noise`), the LM call counters, the residual, trackingWasGood and the point usage.
    -> whether the oracle's tracking was good"""
    assert bool(g.diverged) == bool(o.diverged)
    if o.diverged:
        return False
    dt, ang = pose_err(np.array(g.frameToRef_qt), np.array(o.frameToRef_qt))
    assert dt <= POSE_TOL + noise[0] and ang <= PERMA_ANG_TOL + noise[1], (dt, ang, noise)
    assert list(g.numCalcResidualCalls) == list(o.numCalcResidualCalls)
    assert list(g.numCalcWarpUpdateCalls) == list(o.numCalcWarpUpdateCalls)
    assert abs(g.lastResidual - o.lastResidual) <= 1e-3 * abs(o.lastResidual) + 1e-6
    assert bool(g.trackingWasGood) == bool(o.trackingWasGood)
    assert abs(g.pointUsage - o.pointUsage) <= 1e-4
    return bool(o.trackingWasGood)


def check_perma_overlap(se3, oracle, prs, rng):
    """checkPermaRefOverlap of five random poses around each keyframe of prs (id -> oracle PermaRef) in one batch.
    -> the oracle's overlaps"""
    ids, poses = [], []
    for k in prs:
        for _ in range(5):
            ids.append(k)
            poses.append(_pose_op(oracle, "lsdo_se3d_exp", 7, rng.normal(0, [0.2, 0.2, 0.3, 0.05, 0.05, 0.05])))
    got = se3.checkPermaRefOverlap(ids, np.array(poses))
    want = np.array([prs[k].overlap(q) for k, q in zip(ids, poses)], np.float32)
    assert np.allclose(got, want, rtol=OVERLAP_RTOL, atol=OVERLAP_ATOL), np.abs(got - want).max()
    return want


def perma_noise(oracle, pr, frame, init):
    """the reference's own summation noise in one trackFrameOnPermaref: (translation, rotation) pose_err between its sequential
    fp32 sums and the same tracking with exact sums (lsdo_globals.exactTrackingSums).  On mapped keyframes under camera motion
    it reaches 8e-6 rad, four times PERMA_ANG_TOL"""
    a = pr.track(frame, init)
    oracle.set_globals(exactTrackingSums=1)
    try:
        b = pr.track(frame, init)
    finally:
        oracle.set_globals()
    return pose_err(np.array(a.frameToRef_qt), np.array(b.frameToRef_qt))


# ---- closed loops replayed on the oracle (oracle/replay.py) ----------------------------------------------------------------
def assert_step_ok(r):
    """one replayed step: the pose within 1e-4 plus the reference's own summation noise, the depth map bit for bit"""
    assert r["pose_rel"] <= 1e-4 + r["ref_noise_rel"], (r["frame"], r["pose_rel"], r["ref_noise_rel"])
    assert r["rot_rad"] <= 1e-6 + r["ref_noise_rot"], (r["frame"], r["rot_rad"])
    assert r["map_ok"], (r["frame"], r["map"])


# ---- stream groups ------------------------------------------------------------------------------------------------------------
def observe(gs, fid, qts):
    """what one stream's step left behind, as bytes: the tracking result, the frame's pose record and counters, its good-mask,
    the new keyframe's thisToParent (qts, or None) and the depth map"""
    from lsd_slam_b200 import abi
    ctx = gs.ctx
    pose, parent, itr = ctx.get_pose(fid)
    return {"result": bytes(gs.tracker.last), "pose": pose.tobytes(), "parent": parent, "itr": np.float32(itr).tobytes(),
            "new_kf_qts": None if qts is None else np.asarray(qts).tobytes(),
            "counters": (ctx.get_counters(fid), ctx.get_counters(gs.kf_id)),
            "mask": ctx.download(fid, abi.BUF_GOODMASK).tobytes(),
            "depth": gs.map.current().tobytes()}


def assert_same(a, b):
    """two logs of `observe` records (per step, per stream) are equal"""
    assert len(a) == len(b)
    for k, (sa, sb) in enumerate(zip(a, b), start=1):
        for s, (oa, ob) in enumerate(zip(sa, sb)):
            for key in oa:
                assert oa[key] == ob[key], f"step {k}, stream {s}: {key} differs"


# ---- point cloud ----------------------------------------------------------------------------------------------------------------
def _level_cam(ctx, level):
    """Frame::fx(level) etc. as ROSOutput3DWrapper.cpp:85-88 puts them into the message (Frame.cpp:403-459)"""
    fx, fy, cx, cy = np.float32(ctx.K[0, 0]), np.float32(ctx.K[1, 1]), np.float32(ctx.K[0, 2]), np.float32(ctx.K[1, 2])
    cx0, cy0 = cx, cy
    for lv in range(1, level + 1):
        fx, fy = np.float32(np.float64(fx) * 0.5), np.float32(np.float64(fy) * 0.5)
        cx = np.float32((np.float64(cx0) + 0.5) / (1 << lv) - 0.5)
        cy = np.float32((np.float64(cy0) + 0.5) / (1 << lv) - 0.5)
    return float(fx), float(fy), float(cx), float(cy)


def oracle_cloud(ctx, kf_ids, c2w, level, filt, layout):
    """the CPU viewer oracle's cloud of the context's keyframes: (points as uint32 rows of 4, (total, shown) per keyframe)"""
    from lsd_slam_b200 import abi
    from oracle import cloud
    cam = _level_cam(ctx, level)
    outs, counts = [], []
    for i, kf in enumerate(kf_ids):
        pc = ctx.pack_pointcloud(kf, level).reshape(ctx.h >> level, ctx.w >> level)
        vert, ply, total, shown = cloud.keyframe(pc.view(cloud.INPUT_POINT_DENSE), cam, c2w[i], filt)
        outs.append(vert if layout == abi.CLOUD_VERTEX else ply)
        counts.append((total, shown))
    return np.concatenate(outs).view(np.uint32).reshape(-1, 4), np.array(counts, np.int32).reshape(-1, 2)


def same_cloud(gpu, ref):
    """byte-identical, except that NaN equals NaN.  -> the number of NaN values"""
    g, r = np.ascontiguousarray(gpu).view(np.uint32).reshape(-1, 4), np.asarray(ref).reshape(-1, 4)
    assert g.shape == r.shape
    gn, rn = np.isnan(g.view(np.float32)), np.isnan(r.view(np.float32))
    assert (gn == rn).all()
    assert (g[~gn] == r[~rn]).all()
    return int(gn.sum())
