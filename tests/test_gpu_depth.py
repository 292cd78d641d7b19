"""GPU parity: DepthMap kernels vs the oracle, pass by pass on identical inputs (bit-exact: integer / flag
fields identical, float fields identical bit patterns) and through whole updateKeyframe / createKeyFrame
sequences (north_star tolerance: inverse depth <= 1e-3 relative per pixel)."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import device_cases as cases
from tests.util import IDENT, Pair, hyp_equal_report, pose_err, sim3_inverse, sim3_mul, tracked_pair

pytestmark = pytest.mark.gpu


def test_observe_update_bit_exact(gpu_ctx_small, oracle, seq_small, frames_small):
    p = tracked_pair(gpu_ctx_small, oracle, seq_small, frames_small, [1, 2])
    p.sync_counters()
    # no good-mask on the GPU side -> drop it on the oracle side too (refPixelWasGoodNoCreate == 0)
    for k in (1, 2):
        oracle.lib().lsdo_frame_clear_refPixelWasGood(p.oframes[k].ptr)
    p.odm.observeDepth([p.oframes[1], p.oframes[2]])
    p.gdm.observeDepth([1, 2])
    rep = p.compare(exact=True)
    assert rep["n_valid"] > 10000


def test_observe_create_from_empty_bit_exact(gpu_ctx_small, oracle, seq_small, frames_small):
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "gt")
    empty = np.zeros((seq_small.h, seq_small.w), oracle.HYP_DTYPE)
    p.odm.set_current(empty)
    p.gdm.setHypotheses(0, empty, do_set_depth=False)
    of = p.add_frame(10)
    oracle.lib().lsdo_frame_clear_refPixelWasGood(of.ptr)
    # both sides: initialTrackedResidual = 0 on the oracle frame (never tracked) -> same on the GPU
    gpu_ctx_small.set_pose(10, of.thisToParent(), 0, 0.0)
    p.odm.observeDepth([of])
    p.gdm.observeDepth([10])
    rep = p.compare(exact=True)
    assert rep["n_valid"] > 3000


def test_random_init_update_sequence_bit_exact(gpu_ctx_small, oracle, seq_small, frames_small):
    """random hypotheses exercise every branch of observeDepthUpdate / doLineStereo (fail, inconsistent, skip)"""
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "random")
    for k in (4, 6, 8, 10):
        of = p.add_frame(k)
        gpu_ctx_small.set_pose(k, of.thisToParent(), 0, 0.0)
        oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        gpu_ctx_small.L.lsdgpu_ref_import(gpu_ctx_small.ptr, 0)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
        p.compare(exact=True)
    # Frame::setDepth output
    assert np.array_equal(gpu_ctx_small.download(0, abi.BUF_IDEPTH, 0), p.okf.idepth(0))
    assert np.array_equal(gpu_ctx_small.download(0, abi.BUF_IDEPTH_VAR, 0), p.okf.idepthVar(0))
    m, n, flag = gpu_ctx_small.depth_stats(0)
    assert n == oracle.lib().lsdo_frame_numPoints(p.okf.ptr) and flag
    assert abs(m - oracle.lib().lsdo_frame_meanIdepth(p.okf.ptr)) <= 1e-4 * abs(m)


def test_fill_holes_and_regularize_bit_exact(gpu_ctx_small, oracle, seq_small, frames_small):
    cases.fill_holes_and_regularize(gpu_ctx_small, oracle, seq_small, frames_small)


def test_integral_buffer_matches_oracle(gpu_ctx_small, oracle, seq_small, frames_small):
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "random")
    p.odm.regularizeFillHoles()
    # the oracle's validityIntegralBuffer was built from the state BEFORE fill-holes
    p.gdm_integral = p.gdm.integral()
    assert np.array_equal(p.gdm_integral, p.odm.integral())


@pytest.mark.parametrize("with_mask", [False, True])
def test_propagate_and_create_keyframe(gpu_ctx_small, oracle, seq_small, frames_small, with_mask):
    cases.propagate_and_create_keyframe(gpu_ctx_small, oracle, seq_small, frames_small, with_mask)


def test_update_keyframe_with_frames_tracked_on_the_previous_keyframe(gpu_ctx_small, oracle, seq_small, frames_small):
    """DepthMap.cpp:1085-1099: frames still queued when the keyframe changes were tracked on the OLD keyframe; they are mapped with
    refToKf = activeKeyFrame->getScaledCamToWorld().inverse() * frame->getScaledCamToWorld() and without their tracking mask
    (:245, :322).  The caller passes that product in lsdgpu_ref_desc; every field of every pixel equals the oracle's.
    (Scene rescaled to mean inverse depth 1 on keyframe 0 -- see the pin's create_keyframe_and_finalize.)"""
    d0 = frames_small[0][1]
    sc = float(np.mean(1.0 / d0[d0 > 0]))
    frames = {k: (frames_small[k][0], (frames_small[k][1] * sc).astype(np.float32)) for k in range(13)}

    def qt(k, ref=0):
        q = seq_small.frame_to_ref_qt(k, ref=ref).copy()
        q[4:7] *= sc
        return q
    p = Pair(gpu_ctx_small, oracle, seq_small, frames, "gt")
    ctx = gpu_ctx_small
    for k in (1, 2, 3):
        of = p.add_frame(k, qt(k))
        oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        ctx.L.lsdgpu_ref_import(ctx.ptr, 0)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
    p.compare(exact=True)
    # frames 4 and 5: TRACKED on keyframe 0 on both sides (so both carry a tracking mask), poses then set to ground truth
    trk = abi.SE3Tracker(ctx, mode=1)
    for k in (4, 5):
        of = p.add_frame(k, qt(k))
        r = oracle.se3_track(p.okf, of, qt(k))
        trk.trackFrame(0, k, qt(k))
        qts = np.concatenate([qt(k), [1.0]])
        of.set_thisToParent(qts, p.okf)
        oracle.lib().lsdo_frame_set_initialTrackedResidual(of.ptr, float(r.initialTrackedResidual))
        ctx.set_pose(k, qts, 0, float(r.initialTrackedResidual))
        assert of.refPixelWasGood(create=False) is not None
    ctx.set_counters(0, oracle.lib().lsdo_frame_numFramesTrackedOnThis(p.okf.ptr), oracle.lib().lsdo_frame_numMappedOnThis(p.okf.ptr))
    # keyframe change to frame 9 (no mask on it: identical inputs -> identical maps, rescale included)
    of9 = p.add_frame(9, qt(9))
    p.odm.finalizeKeyFrame()
    p.gdm.finalizeKeyFrame()
    p.odm.createKeyFrame(of9)
    q9 = p.gdm.createKeyFrame(9)
    assert np.float32(q9[7]).tobytes() == np.float32(of9.thisToParent()[7]).tobytes() and 0.8 < q9[7] < 1.25
    p.compare(exact=True)
    # ids only: refused, with a pointer to the descriptor call
    with pytest.raises(abi.LsdGpuError, match="update_keyframe_refs"):
        p.gdm.updateKeyframe([4])
    w2c9 = sim3_inverse(oracle, of9.thisToParent())              # keyframe 0 is the first frame: its camToWorld is the identity
    items = [(k, sim3_mul(oracle, w2c9, p.oframes[k].thisToParent())) for k in (4, 5)]
    before = p.gdm.current().copy()
    p.odm.updateKeyframe([p.oframes[4], p.oframes[5]])
    p.gdm.updateKeyframe(items)
    rep = p.compare(exact=True)
    after = p.gdm.current()
    both = (before["isValid"] != 0) & (after["isValid"] != 0)
    assert rep["n_valid"] > 10000 and int((before["idepth"][both] != after["idepth"][both]).sum()) > 2000      # they did observe
    # mixed parents in one call; a frame declared tracked_on_kf whose parent is another keyframe is refused
    of12 = oracle.Frame(12, frames[12][0], seq_small.K)
    q12 = np.concatenate([qt(12, ref=9), [1.0]])
    q12[4:7] /= q9[7]
    of12.set_thisToParent(q12, of9)
    ctx.upload(12, frames[12][0])
    ctx.set_pose(12, q12, 9, 0.0)
    p.odm.updateKeyframe([p.oframes[5], of12])
    p.gdm.updateKeyframe([items[1], 12])
    p.compare(exact=True)
    descs = (abi.RefDesc * 1)()
    descs[0].frame_id, descs[0].tracked_on_kf = 4, 1
    assert ctx.L.lsdgpu_depth_update_keyframe_refs(ctx.ptr, descs, 1) != 0


def test_finalize_keyframe(gpu_ctx_small, oracle, seq_small, frames_small):
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "random")
    p.odm.finalizeKeyFrame()
    p.gdm.finalizeKeyFrame()
    p.compare(exact=True)
    assert np.array_equal(gpu_ctx_small.download(0, abi.BUF_IDEPTH, 0), p.okf.idepth(0))


def test_full_loop_parity(gpu_ctx_small, oracle, seq_small, frames_small):
    """track + map loop run independently on both sides (each side consumes ITS OWN poses): inverse depth
    within 1e-3 relative per pixel, poses within 1e-4 (north_star)."""
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "gt")
    trk = abi.SE3Tracker(gpu_ctx_small, mode=1)
    last_o = last_g = IDENT
    for k in range(1, 9):
        img, _ = frames_small[k]
        of = oracle.Frame(k, img, seq_small.K)
        if oracle.lib().lsdo_frame_depthHasBeenUpdatedFlag(p.okf.ptr):
            oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        r = oracle.se3_track(p.okf, of, last_o)
        last_o = np.array(r.frameToRef_qt)
        p.odm.updateKeyframe([of])
        gpu_ctx_small.upload(k, img)
        trk.importFrame(0)
        last_g = trk.trackFrame(0, k, last_g)
        p.gdm.updateKeyframe([k])
        dt, ang = pose_err(last_g, last_o)
        assert dt <= 1e-4 and ang <= 1e-6, (k, dt, ang)
        if k > 2:
            gpu_ctx_small.release(k - 2)
    a, b = p.gdm.current(), p.odm.current()
    va, vb = a["isValid"] > 0, b["isValid"] > 0
    assert (va != vb).mean() <= 1e-3
    both = va & vb
    rel = np.abs(a["idepth_smoothed"][both] - b["idepth_smoothed"][both]) / np.abs(b["idepth_smoothed"][both])
    assert (rel <= 1e-3).mean() >= 0.999, float((rel <= 1e-3).mean())


def test_fused_call_equals_individual_calls(seq_small, frames_small):
    """lsdgpu_track_and_map (one ABI call per frame) == the individual calls, bit for bit"""
    from lsd_slam_b200.stream import GpuStream
    outs = []
    for fused in (True, False):
        ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=8)
        gs = GpuStream(ctx, mode=1, kf_every=4, fused_call=fused)
        gs.init_gt(0, frames_small[0][0], frames_small[0][1])
        for k in range(1, 8):
            gs.step(k, frames_small[k][0])
        outs.append((np.array(gs.poses), gs.map.current().copy(), ctx.download(gs.kf_id, abi.BUF_IDEPTH, 2)))
        ctx.close()
    assert np.array_equal(outs[0][0], outs[1][0])
    assert outs[0][1].tobytes() == outs[1][1].tobytes()
    assert np.array_equal(outs[0][2], outs[1][2])


def test_fused_call_divergence_leaves_map_untouched(seq_small, frames_small):
    """frame path: when tracking diverges nothing of the map may change"""
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=8)
    from lsd_slam_b200.stream import GpuStream
    gs = GpuStream(ctx, mode=1, kf_every=0, fused_call=True)
    gs.init_gt(0, frames_small[0][0], frames_small[0][1])
    gs.step(1, frames_small[1][0])
    before = gs.map.current().copy()
    idepth_before = ctx.download(0, abi.BUF_IDEPTH, 1).copy()
    gs.last_pose = np.array([0, 0.7071067811865476, 0, 0.7071067811865476, 0, 0, 0], np.float64)   # looks away
    with pytest.raises(RuntimeError):
        gs.step(2, frames_small[2][0])
    assert gs.tracker.diverged
    assert gs.map.current().tobytes() == before.tobytes()
    assert np.array_equal(ctx.download(0, abi.BUF_IDEPTH, 1), idepth_before)
    # and the stream continues normally afterwards
    gs.last_pose = np.array(gs.poses[-1])
    gs.n_tracked -= 1
    ctx.release(2)
    p = gs.step(3, frames_small[3][0])
    assert not gs.tracker.diverged and np.isfinite(p).all()
    ctx.close()


def test_reactivated_keyframe_and_multiple_reference_frames(gpu_ctx_small, oracle, seq_small, frames_small):
    """setFromExistingKF semantics (activeKeyFrameIsReactivated: newest reference frame is used, DepthMap.cpp:241,317)
    and a 3-frame reference deque with id gaps (referenceFrameByID, DepthMap.cpp:1103-1104)"""
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "random")
    refs = []
    for k in (3, 5, 8):                      # ids with gaps: byId table has repeated entries
        of = p.add_frame(k)
        gpu_ctx_small.set_pose(k, of.thisToParent(), 0, 0.0)
        refs.append(of)
    # non-reactivated, three references at once
    oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
    gpu_ctx_small.L.lsdgpu_ref_import(gpu_ctx_small.ptr, 0)
    p.odm.updateKeyframe(refs)
    p.gdm.updateKeyframe([3, 5, 8])
    p.compare(exact=True)
    # make some hypotheses point at later frames, then update again
    cur = p.odm.current().copy()
    rng = np.random.default_rng(9)
    cur["nextStereoFrameMinID"] = rng.integers(0, 12, cur.shape).astype(np.float32)
    p.odm.set_current(cur)
    p.gdm.setHypotheses(0, cur, do_set_depth=False)
    p.odm.observeDepth(refs)
    p.gdm.observeDepth([3, 5, 8])
    p.compare(exact=True)


def test_set_from_existing_keyframe_reactivated(gpu_ctx_small, oracle, seq_small, frames_small):
    """DepthMap::setFromExistingKF (DepthMap.cpp:920-962): re-activation data -> hypotheses, regularizeDepthMap(false),
    activeKeyFrameIsReactivated => observeDepth uses the NEWEST reference frame (:241, :317)"""
    img0, d0 = frames_small[0]
    rng = np.random.default_rng(11)
    okf = oracle.Frame(0, img0, seq_small.K)
    mg = okf.maxGradients(0)
    idepth = np.where(mg >= 5, 1.0 / d0 + rng.normal(0, 0.02, d0.shape), 0).astype(np.float32)
    var = np.where(mg >= 5, 0.01, -1.0).astype(np.float32)
    var[rng.random(var.shape) < 0.02] = -2.0                       # blacklisted cells (Frame.cpp:134-137)
    validity = rng.integers(0, 60, d0.shape).astype(np.uint8)
    odm = oracle.DepthMap(seq_small.w, seq_small.h, seq_small.K)
    odm.setFromExistingKF(okf, idepth, var, validity)
    # GPU: the host builds the AoS exactly as DepthMap.cpp:937-959 and asks for the reactivation semantics
    hyp = np.zeros(d0.shape, abi.HYP_DTYPE)
    ok = var > 0
    hyp["isValid"] = ok
    hyp["idepth"] = np.where(ok, idepth, 0); hyp["idepth_var"] = np.where(ok, var, 0)
    hyp["idepth_smoothed"] = np.where(ok, -1, 0); hyp["idepth_var_smoothed"] = np.where(ok, -1, 0)
    hyp["validity_counter"] = np.where(ok, validity, 0)
    hyp["blacklisted"] = np.where(~ok & (var == -2), -2, 0)
    gpu_ctx_small.upload(0, img0)
    gdm = abi.DepthMap(gpu_ctx_small)
    gdm.setHypotheses(0, hyp, reactivated=True, do_set_depth=False)
    a, b = gdm.current(), odm.current()
    rep = hyp_equal_report(a, b)
    assert rep["valid_mismatch"] == 0 and rep["blacklist_mismatch"] == 0 and rep["idepth_smoothed_bitdiff"] == 0, rep
    # two reference frames: the reactivated map must take the newest one for every pixel
    ofs = []
    for k in (4, 7):
        of = oracle.Frame(k, frames_small[k][0], seq_small.K)
        qts = np.concatenate([seq_small.frame_to_ref_qt(k), [1.0]])
        of.set_thisToParent(qts, okf)
        gpu_ctx_small.upload(k, frames_small[k][0])
        gpu_ctx_small.set_pose(k, qts, 0, 0.0)
        ofs.append(of)
    odm.observeDepth(ofs)
    gdm.observeDepth([4, 7])
    rep = hyp_equal_report(gdm.current(), odm.current())
    assert rep["valid_mismatch"] == 0 and rep["idepth_bitdiff"] == 0 and rep["idepth_var_bitdiff"] == 0, rep
    assert rep["nextStereoFrameMinID_bitdiff"] == 0 and rep["validity_mismatch"] == 0, rep
