"""The hot path at frame sizes off the 4:3 grid the other suites use, against the oracle.

Every width and height that is a multiple of 16 is legal (SlamSystem.cpp:55).  The other GPU tests only run widths that are
multiples of 32, so every 32-wide tile of the staging, fill and regularisation kernels is full.  Here:
  * 336x240 and 208x352 (portrait): w % 32 == 16, the last column of tiles is half full on every level;
  * 64x48: level 4 is 4x3, most of the tracker's virtual CTAs get no chunk;
  * 16x16: the smallest legal frame, level 4 is 1x1 (no interior pixel).
At 64x48 and 16x16 the reference's own tracker diverges on every frame: level 4 has no pixel that can warp inside
(SE3Tracker.cpp:324-329), so trackFrame is compared on that outcome and the mapping sequence runs on ground-truth poses."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import IDENT
from oracle.replay import run_with_replay
from tests.test_gpu_cloud import FILTERS, _oracle, _same
from tests.test_gpu_depth import Pair
from tests.test_gpu_group import _assert_same, _run
from tests.test_gpu_track import _cmp_eval
from tests.util import pose_err, rot_angle

pytestmark = pytest.mark.gpu

SHAPES = [(336, 240), (208, 352), (64, 48), (16, 16)]
TRACKABLE = {(336, 240), (208, 352)}          # the reference's tracker converges at these sizes
N_FRAMES = 12
KF_EVERY = 5
SHAPE_IDS = [f"{w}x{h}" for w, h in SHAPES]

_cache = {}


def _seq(w, h):
    if (w, h) not in _cache:
        seq = synth.Sequence(w, h, seed=1234)
        _cache[(w, h)] = (seq, [seq.render(k) for k in range(N_FRAMES)])
    return _cache[(w, h)]


@pytest.fixture(params=SHAPES, ids=SHAPE_IDS)
def shape(request):
    return request.param


@pytest.fixture()
def setup(shape):
    seq, frames = _seq(*shape)
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=8)
    yield seq, frames, ctx
    ctx.close()


def test_frame_staging_bit_exact(setup, oracle):
    seq, frames, ctx = setup
    img, d = frames[2]
    d = d.copy()
    d[: max(1, seq.h // 8), : max(1, seq.w // 8)] = np.nan          # invalid GT depth cells (Frame.cpp:270)
    ctx.upload(2, img)
    ctx.set_depth_gt(2, d)
    of = oracle.Frame(2, img, seq.K)
    of.setDepthFromGroundTruth(d)
    for lvl in range(5):
        assert np.array_equal(ctx.download(2, abi.BUF_IMAGE, lvl), of.image(lvl)), lvl
        g, o = ctx.download(2, abi.BUF_GRADIENTS, lvl), of.gradients(lvl)
        for c, name in enumerate("xyz"):
            assert np.array_equal(g[..., c], o[..., c]), (lvl, name)
        assert np.array_equal(ctx.download(2, abi.BUF_IDEPTH, lvl), of.idepth(lvl)), lvl
        assert np.array_equal(ctx.download(2, abi.BUF_IDEPTH_VAR, lvl), of.idepthVar(lvl)), lvl
    assert np.array_equal(ctx.download(2, abi.BUF_MAXGRAD, 0), of.maxGradients(0))


EVAL_FIELDS = ("lsError", "meanWeightedRes", "meanUnweightedRes", "pointUsage", "affine_a_lastIt", "affine_b_lastIt", "meanRes",
               "sxx", "syy", "sx", "sy", "sw")


def _cmp_eval_any(g, o):
    """_cmp_eval, or -- where the oracle's statistics are NaN (no or one warped point) -- NaN in the same fields and the counts"""
    if all(np.isfinite(getattr(o, f)) for f in EVAL_FIELDS):
        _cmp_eval(g, o)
        return
    assert g.warpedSize == o.warpedSize and g.goodCount == o.goodCount and g.badCount == o.badCount
    for f in EVAL_FIELDS:
        a, b = getattr(g, f), getattr(o, f)
        assert np.isnan(a) == np.isnan(b) and (np.isnan(b) or abs(a - b) <= 2e-4 * abs(b) + 1e-6), (f, a, b)


def test_single_evaluation_per_level(setup, oracle):
    seq, frames, ctx = setup
    ctx.upload(0, frames[0][0])
    ctx.set_depth_gt(0, frames[0][1])
    ctx.upload(3, frames[3][0])
    okf = oracle.Frame(0, frames[0][0], seq.K)
    okf.setDepthFromGroundTruth(frames[0][1])
    of = oracle.Frame(3, frames[3][0], seq.K)
    trk = abi.SE3Tracker(ctx)
    inv = np.zeros(7)
    oracle.lib().lsdo_se3d_inverse(oracle._dp(seq.frame_to_ref_qt(3)), oracle._dp(inv))
    for level in (4, 3, 2, 1):
        for pose, a, b in ((IDENT.astype(np.float32), 1.0, 0.0), (inv.astype(np.float32), 0.98, 1.5)):
            g = trk.eval(0, 3, level, pose, a, b, write_mask=level == 1)
            o = oracle.se3_eval(okf, of, level, pose, a, b, write_mask=level == 1)
            _cmp_eval_any(g, o)
            if level == 1:
                assert (ctx.download(3, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < 1e-3


@pytest.mark.parametrize("mode", [0, 1])
def test_track_frame(setup, oracle, mode):
    seq, frames, ctx = setup
    ctx.upload(0, frames[0][0])
    ctx.set_depth_gt(0, frames[0][1])
    ctx.upload(2, frames[2][0])
    trk = abi.SE3Tracker(ctx, mode=mode)
    pose_g = trk.trackFrame(0, 2, IDENT)
    res = []
    for exact in (0, 1):                         # the reference, and the same tracking with exact sums (its own summation noise)
        oracle.set_globals(exactTrackingSums=exact)
        try:
            okf = oracle.Frame(0, frames[0][0], seq.K)
            okf.setDepthFromGroundTruth(frames[0][1])
            of = oracle.Frame(2, frames[2][0], seq.K)
            res.append((oracle.se3_track(okf, of, IDENT), of))
        finally:
            oracle.set_globals()
    (r, of), (rx, _) = res
    pose_o = np.array(r.frameToRef_qt)
    noise_t, noise_r = pose_err(pose_o, np.array(rx.frameToRef_qt))
    dt, ang = pose_err(pose_g, pose_o)
    assert dt <= 1e-4 + noise_t, (dt, noise_t)
    assert ang <= 1e-4 * max(rot_angle(pose_o), 1e-2) + 1e-7 + noise_r, ang
    assert trk.diverged == bool(r.diverged) and trk.trackingWasGood == bool(r.trackingWasGood)
    assert r.diverged == ((seq.w, seq.h) not in TRACKABLE)
    assert list(trk.last.numCalcResidualCalls) == list(r.numCalcResidualCalls)
    assert list(trk.last.numCalcWarpUpdateCalls) == list(r.numCalcWarpUpdateCalls)
    if not r.diverged:
        assert (ctx.download(2, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < 1e-3


def test_stream_replayed_on_the_oracle(shape, oracle):
    """observe, fill and regularise, propagate, the createKeyFrame rescale and setDepth with its pyramid: every step's depth map
    bit for bit, with two keyframe changes"""
    seq, frames = _seq(*shape)
    if shape not in TRACKABLE:
        pytest.skip("the reference diverges on every frame at this size: test_mapping_on_ground_truth_poses maps it")
    reps = run_with_replay(seq, frames, N_FRAMES, kf_every=KF_EVERY)
    assert len(reps) == N_FRAMES - 1 and sum(r["kf_change"] for r in reps) == 2
    for r in reps:
        assert r["pose_rel"] <= 1e-4 + r["ref_noise_rel"], (r["frame"], r["pose_rel"], r["ref_noise_rel"])
        assert r["rot_rad"] <= 1e-6 + r["ref_noise_rot"], (r["frame"], r["rot_rad"])
        assert r["mask_mismatch"] <= 1e-3 * (seq.w // 2) * (seq.h // 2), (r["frame"], r["mask_mismatch"])
        g, o = r["stats"]["good"]
        assert abs(g - o) <= 2, r["frame"]
    assert sum(r["counts_equal"] for r in reps) >= len(reps) - 1           # one decision exactly at a threshold may flip
    bad = [(r["frame"], r["map"]) for r in reps if not r["map_ok"]]
    assert not bad, bad[:2]


def test_mapping_on_ground_truth_poses(setup, oracle):
    """the same mapping sequence as the replay, with the ground-truth pose handed to both sides (every size)"""
    seq, frames, ctx = setup
    p = Pair(ctx, oracle, seq, frames, "gt")
    kf, okf, changes = 0, p.okf, 0
    for k in range(1, N_FRAMES):
        img = frames[k][0]
        of = oracle.Frame(k, img, seq.K)
        qts = np.concatenate([seq.frame_to_ref_qt(k, ref=kf), [1.0]])
        of.set_thisToParent(qts, okf)
        ctx.upload(k, img)
        ctx.set_pose(k, qts, kf, 0.0)
        if k % KF_EVERY == 0:
            p.odm.finalizeKeyFrame()
            p.odm.createKeyFrame(of)
            p.gdm.finalizeKeyFrame()
            p.gdm.createKeyFrame(k)
            kf, okf = k, of
            changes += 1
        else:
            oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(okf.ptr, 0)
            ctx.L.lsdgpu_ref_import(ctx.ptr, kf)
            p.odm.updateKeyframe([of])
            p.gdm.updateKeyframe([k])
        rep = p.compare(exact=True)
        assert np.array_equal(ctx.download(kf, abi.BUF_IDEPTH, 0), okf.idepth(0)), k
        if k != kf:
            ctx.release(k)
        elif k != KF_EVERY:
            ctx.release(k - KF_EVERY)             # the previous keyframe
    assert changes == 2 and rep["n_valid"] > 0
    for lvl in range(5):                      # Frame::setDepth of the last keyframe and its pyramid
        assert np.array_equal(ctx.download(kf, abi.BUF_IDEPTH, lvl), okf.idepth(lvl)), lvl
        assert np.array_equal(ctx.download(kf, abi.BUF_IDEPTH_VAR, lvl), okf.idepthVar(lvl)), lvl


def test_group_of_two_equals_single_calls(shape):
    w, h = shape
    phases = [15, 17]                             # keyframe changes at steps 5 and 3 (test_gpu_group's KF_EVERY = 20)
    single = _run(w, h, phases, 6, lambda k: False)
    group = _run(w, h, phases, 6, lambda k: True)
    assert all(o["diverged"] == (shape not in TRACKABLE) for step in single for o in step)
    _assert_same(group, single)


@pytest.mark.parametrize("layout", [abi.CLOUD_PLY, abi.CLOUD_VERTEX])
def test_cloud_every_level(setup, layout):
    seq, frames, ctx = setup
    c2w = []
    for i in range(2):
        ctx.upload(i, frames[3 * i][0])
        ctx.set_depth_gt(i, frames[3 * i][1])
        c2w.append(np.concatenate([seq.frame_to_ref_qt(3 * i), [1.0]]))
    c2w = np.array([np.concatenate([q[:4] * 1.25, q[4:7]]) for q in c2w], np.float32)
    ctx.cloud_reserve(2)
    levels = [lvl for lvl in range(5) if (seq.w >> lvl) >= 3 and (seq.h >> lvl) >= 3]
    assert levels[-1] >= 2
    for lvl in levels:
        for filt in FILTERS:
            pts, counts = ctx.export_pointcloud([0, 1], c2w, level=lvl, filter=filt, layout=layout)
            ref, ref_counts = _oracle(ctx, [0, 1], c2w, lvl, filt, layout)
            assert (counts == ref_counts).all(), (lvl, filt)
            _same(pts, ref)
        assert counts[:, 0].sum() > 0, lvl


def test_sim3_and_perma_batches_at_336x240(oracle):
    from tests.test_gpu_sim3 import _check_track, _init
    from tests.test_gpu_sim3 import _setup as sim3_setup
    seq, ctx, trk, of = sim3_setup(oracle, 336, 240)
    pairs = [(a, b) for a in of for b in of if a != b]
    inits = np.array([_init(seq, fr, ref) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    for (ref, fr), init, r in zip(pairs, inits, res):
        _check_track(r, oracle.sim3_track(of[ref], of[fr], init, 4, 1))
    ctx.close()

    # permaRef (level 4, 21x15 here): setPermaRef, then trackFrameOnPermaref from the ground truth and from identity
    ctx = abi.Context(336, 240, seq.K, max_frames=8)
    try:
        se3 = abi.SE3Tracker(ctx)
        prs = {}
        for k in (0, 6):
            img, d = seq.render(k)
            ctx.upload(k, img)
            ctx.set_depth_gt(k, d)
            okf = oracle.Frame(k, img, seq.K)
            okf.setDepthFromGroundTruth(d)
            prs[k] = oracle.PermaRef(okf)
            assert se3.setPermaRef(k) == prs[k].n > 100
        img, _ = seq.render(3)
        ctx.upload(3, img)
        of3 = oracle.Frame(3, img, seq.K)
        ids, inits = [], []
        for k in prs:
            gt_inv = np.zeros(7)
            oracle.lib().lsdo_se3d_inverse(oracle._dp(seq.frame_to_ref_qt(3, ref=k)), oracle._dp(gt_inv))
            ids += [k, k]
            inits += [gt_inv, IDENT]
        n_good = 0
        for k, init, g in zip(ids, inits, se3.trackFrameOnPermaref(ids, 3, np.array(inits))):
            o = prs[k].track(of3, init)
            assert bool(g.diverged) == bool(o.diverged)
            if o.diverged:
                continue
            dt, ang = pose_err(np.array(g.frameToRef_qt), np.array(o.frameToRef_qt))
            assert dt <= 1e-4 and ang <= 2e-6, (k, dt, ang)
            assert list(g.numCalcResidualCalls) == list(o.numCalcResidualCalls)
            assert abs(g.lastResidual - o.lastResidual) <= 1e-3 * abs(o.lastResidual) + 1e-6
            assert bool(g.trackingWasGood) == bool(o.trackingWasGood)
            assert abs(g.pointUsage - o.pointUsage) <= 1e-4
            n_good += int(o.trackingWasGood)
        assert n_good >= 2
    finally:
        ctx.close()
