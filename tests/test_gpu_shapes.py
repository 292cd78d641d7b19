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
from oracle.replay import run_with_replay
from tests import device_cases as cases
from tests.util import CLOUD_FILTERS, Pair, assert_same, assert_step_ok, oracle_cloud, same_cloud

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


def test_single_evaluation_per_level(setup, oracle):
    seq, frames, ctx = setup
    cases.se3_eval_each_level(ctx, oracle, seq, frames, mask_tol=1e-3)


@pytest.mark.parametrize("mode", [0, 1])
def test_track_frame(setup, oracle, mode):
    """against the reference, and the same tracking with exact sums (its own summation noise)"""
    seq, frames, ctx = setup
    cases.se3_track(ctx, oracle, seq, frames, mode, 2, sum_noise=True, diverges=(seq.w, seq.h) not in TRACKABLE)


def test_stream_replayed_on_the_oracle(shape, oracle):
    """observe, fill and regularise, propagate, the createKeyFrame rescale and setDepth with its pyramid: every step's depth map
    bit for bit, with two keyframe changes"""
    seq, frames = _seq(*shape)
    if shape not in TRACKABLE:
        pytest.skip("the reference diverges on every frame at this size: test_mapping_on_ground_truth_poses maps it")
    reps = run_with_replay(seq, frames, N_FRAMES, kf_every=KF_EVERY)
    assert len(reps) == N_FRAMES - 1 and sum(r["kf_change"] for r in reps) == 2
    for r in reps:
        assert_step_ok(r)
        assert r["mask_mismatch"] <= 1e-3 * (seq.w // 2) * (seq.h // 2), (r["frame"], r["mask_mismatch"])
        g, o = r["stats"]["good"]
        assert abs(g - o) <= 2, r["frame"]
    assert sum(r["counts_equal"] for r in reps) >= len(reps) - 1           # one decision exactly at a threshold may flip


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
    phases = [15, 17]                             # keyframe changes at steps 5 and 3 (GROUP_KF_EVERY = 20)
    single = cases.run_streams(w, h, phases, 6, lambda k: False)
    group = cases.run_streams(w, h, phases, 6, lambda k: True)
    assert all(o["diverged"] == (shape not in TRACKABLE) for step in single for o in step)
    assert_same(group, single)


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
        for filt in CLOUD_FILTERS:
            pts, counts = ctx.export_pointcloud([0, 1], c2w, level=lvl, filter=filt, layout=layout)
            ref, ref_counts = oracle_cloud(ctx, [0, 1], c2w, lvl, filt, layout)
            assert (counts == ref_counts).all(), (lvl, filt)
            same_cloud(pts, ref)
        assert counts[:, 0].sum() > 0, lvl


def test_sim3_and_perma_batches_at_336x240(oracle):
    seq, ctx, trk, of = cases.sim3_setup(oracle, 336, 240)
    cases.sim3_batch(trk, oracle, seq, of)
    ctx.close()

    # permaRef (level 4, 21x15 here): setPermaRef, then trackFrameOnPermaref from the ground truth and from identity
    ctx = abi.Context(336, 240, seq.K, max_frames=8)
    try:
        se3, prs = cases.perma_setup(ctx, oracle, seq, (0, 6), 100)
        assert cases.perma_batch(ctx, oracle, seq, se3, prs, 3) >= 2
    finally:
        ctx.close()
