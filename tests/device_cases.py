"""Device scenarios that the parity tests run under more than one axis (the default stream, non-default run-time settings, other
camera motions, other frame shapes, mapped keyframes).  Each drives the oracle and the CUDA path through one call sequence and
checks the results with tests/util.py; the caller chooses the context, the stream and its own thresholds."""
import numpy as np

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup, sim3_mul_qts
from tests.pin_cases import (AB, MAPPED_FRAMES, MAPPED_KF_EVERY, PERMA_FRAME, POSE_SENSITIVE_DEPTH_RESIDUAL, SIM3_DT, SIM3_SCALE,
                             adversarial_edit, set_depth)
from tests.util import (IDENT, Pair, check_perma_overlap, check_perma_track, check_se3_eval, check_se3_track, check_sim3_eval,
                        check_sim3_track, kf_depth_equal, new_depth, observe, oracle_sim3_exact, oracle_sim3_track, perma_noise,
                        pose_err, se3_inverse, sim3_err, sim3_init, sim3_inverse, sim3_mul, tracked_pair)


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def observe_from_gt(ctx, oracle, seq, frames):
    """observeDepth with two reference frames (line stereo, the minUseGrad gates of the observe pass)"""
    p = Pair(ctx, oracle, seq, frames, "gt")
    ofs = [p.add_frame(k) for k in (1, 2)]
    p.sync_counters()
    p.odm.observeDepth(ofs)
    p.gdm.observeDepth([1, 2])
    assert p.compare(exact=True)["n_valid"] > 3000


def random_init_observe_and_update(ctx, oracle, seq, frames):
    """random hypotheses drive the line stereo through its failure branches (the -2 of a negative inverse depth among them)"""
    p = Pair(ctx, oracle, seq, frames, "random")
    of = p.add_frame(4)
    p.odm.observeDepth([of])
    p.gdm.observeDepth([4])
    p.compare(exact=True)
    for k in (6, 8, 10):
        of = p.add_frame(k)
        new_depth(p)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
        p.compare(exact=True)
    kf_depth_equal(ctx, p.okf, 0)


def _integral(cur):
    v = np.where(cur["isValid"] > 0, cur["validity_counter"], 0).astype(np.int64)
    return v.cumsum(0).cumsum(1).astype(np.int32)


def fill_holes_and_regularize(ctx, oracle, seq, frames):
    """a random map with holes punched and pixels blacklisted, so that every fill-holes branch triggers; then both regularisers"""
    p = Pair(ctx, oracle, seq, frames, "random")
    cur = p.odm.current().copy()
    rng = np.random.default_rng(3)
    cur["isValid"][rng.random(cur.shape) < 0.3] = 0
    cur["blacklisted"][rng.random(cur.shape) < 0.05] = -3
    cur["validity_counter"] = rng.integers(0, 30, cur.shape)
    p.odm.set_current(cur)
    p.gdm.setHypotheses(0, cur, do_set_depth=False)
    p.odm.regularizeFillHoles()
    p.gdm.regularizeFillHoles()
    p.compare(exact=True)
    integral = p.gdm.integral()
    assert np.array_equal(integral, p.odm.integral())
    assert np.array_equal(integral, _integral(p.gdm.current()))
    for occl in (False, True):
        p.odm.regularize(occl, 24)
        p.gdm.regularize(occl, 24)
        p.compare(exact=True)


def update_keyframe_sequence(ctx, oracle, seq, frames):
    """updateKeyframe = observe + the fused fill-holes and regulariser (depth.cuh) + Frame::setDepth, 1 and 2 reference frames"""
    p = Pair(ctx, oracle, seq, frames, "gt")
    for ks in ([1], [2, 3], [5]):
        ofs = [p.add_frame(k) for k in ks]
        new_depth(p)
        p.odm.updateKeyframe(ofs)
        p.gdm.updateKeyframe(ks)
        assert p.compare(exact=True)["n_valid"] > 3000
        kf_depth_equal(ctx, p.okf, 0)


def fill_holes_and_regularize_observed(ctx, oracle, seq, frames):
    """the passes of depthmap_individual_passes, on the map one observeDepth of the stream left"""
    p = Pair(ctx, oracle, seq, frames, "gt")
    ofs = [p.add_frame(k) for k in (2, 3)]
    p.sync_counters()
    p.odm.observeDepth(ofs)
    p.gdm.observeDepth([2, 3])
    assert p.compare(exact=True)["n_valid"] > 10000
    p.odm.regularizeFillHoles()
    p.gdm.regularizeFillHoles()
    p.compare(exact=True)
    assert np.array_equal(p.gdm.integral(), p.odm.integral())
    for occl in (False, True):
        p.odm.regularize(occl, 24)
        p.gdm.regularize(occl, 24)
        p.compare(exact=True)


def propagate_and_create_keyframe_device_mask(ctx, oracle, seq, frames):
    """propagate_and_create_keyframe with the tracking mask, from identical inputs: each frame is tracked on the device and its
    good mask is handed to the oracle, as oracle/replay.py does.  propagate_and_create_keyframe's with-mask variant lets each
    side use its own tracker's mask; the two masks differ on up to 1e-3 of the pixels (test_gpu_track.py), and under the backward
    and roll motions those pixels move the regularised depth of their neighbours after createKeyFrame by up to 1.1e-3, beyond
    the 2e-5 it allows.  With the same mask on both sides every step is bit for bit."""
    p = tracked_pair(ctx, oracle, seq, frames, [2, 5, 9])
    trk = abi.SE3Tracker(ctx, mode=0)
    for k in (2, 5, 9):
        of = p.oframes[k]
        oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        ctx.L.lsdgpu_ref_import(ctx.ptr, 0)
        trk.trackFrame(0, k, IDENT if k == 2 else of.thisToParent()[:7])        # writes the device's mask; the pose is restored
        ctx.set_pose(k, of.thisToParent(), 0, oracle.lib().lsdo_frame_initialTrackedResidual(of.ptr))
        mask = ctx.download(k, abi.BUF_GOODMASK)
        assert mask.mean() > 0.05
        of.refPixelWasGood(create=True)[:] = mask
        p.sync_counters()
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
        p.compare(exact=True)
    before = p.odm.current().copy()
    p.odm.propagateDepth(p.oframes[9])
    p.gdm.propagateDepth(9)
    assert p.compare(exact=True)["n_valid"] > 5000
    p.odm.set_current(before)
    p.gdm.setHypotheses(0, before, do_set_depth=False)
    p.odm.createKeyFrame(p.oframes[9])
    q = p.gdm.createKeyFrame(9)
    assert np.allclose(q[:7], p.oframes[9].thisToParent()[:7], atol=1e-12)
    assert np.float32(q[7]).tobytes() == np.float32(p.oframes[9].thisToParent()[7]).tobytes()
    p.compare(exact=True)
    assert np.array_equal(ctx.download(9, abi.BUF_IDEPTH, 0), p.oframes[9].idepth(0))


def finalize_create_and_refs(ctx, oracle, seq, frames_in):
    """finalizeKeyFrame + createKeyFrame (propagation, rescale) and then update_keyframe_refs with frames tracked on the previous
    keyframe -- the scene at mean inverse depth 1 on keyframe 0, as in the pin's create_keyframe_and_finalize"""
    d0 = frames_in[0][1]
    sc = float(np.mean(1.0 / d0[d0 > 0]))
    frames = {k: (frames_in[k][0], (frames_in[k][1] * sc).astype(np.float32)) for k in range(13)}

    def qt(k):
        q = seq.frame_to_ref_qt(k).copy()
        q[4:7] *= sc
        return q
    p = Pair(ctx, oracle, seq, frames, "gt")
    for k in (1, 2, 3):
        of = p.add_frame(k, qt(k))
        new_depth(p)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
    p.compare(exact=True)
    trk = abi.SE3Tracker(ctx, mode=1)
    for k in (4, 5):                                # tracked on keyframe 0 on both sides, then put at the ground truth
        of = p.add_frame(k, qt(k))
        r = oracle.se3_track(p.okf, of, qt(k))
        trk.trackFrame(0, k, qt(k))
        qts = np.concatenate([qt(k), [1.0]])
        of.set_thisToParent(qts, p.okf)
        oracle.lib().lsdo_frame_set_initialTrackedResidual(of.ptr, float(r.initialTrackedResidual))
        ctx.set_pose(k, qts, 0, float(r.initialTrackedResidual))
    p.sync_counters()
    of9 = p.add_frame(9, qt(9))
    p.odm.finalizeKeyFrame()
    p.gdm.finalizeKeyFrame()
    p.compare(exact=True)
    p.odm.createKeyFrame(of9)
    q9 = p.gdm.createKeyFrame(9)
    assert np.float32(q9[7]).tobytes() == np.float32(of9.thisToParent()[7]).tobytes()
    p.compare(exact=True)
    kf_depth_equal(ctx, of9, 9)
    w2c9 = sim3_inverse(oracle, of9.thisToParent())          # keyframe 0 is the first frame: its camToWorld is the identity
    items = [(k, sim3_mul(oracle, w2c9, p.oframes[k].thisToParent())) for k in (4, 5)]
    before = p.gdm.current().copy()
    p.odm.updateKeyframe([p.oframes[4], p.oframes[5]])
    p.gdm.updateKeyframe(items)
    rep = p.compare(exact=True)
    after = p.gdm.current()
    both = (before["isValid"] != 0) & (after["isValid"] != 0)
    assert rep["n_valid"] > 3000 and int((before["idepth"][both] != after["idepth"][both]).sum()) > 200     # they did observe


def propagate_and_create_keyframe(ctx, oracle, seq, frames, with_mask):
    """three oracle-tracked frames mapped, then propagateDepth alone and the whole createKeyFrame from the same state: bit for bit
    without a tracking mask; with each side's own tracker's mask, to the tolerance those masks' differences leave"""
    p = tracked_pair(ctx, oracle, seq, frames, [2, 5, 9])
    for k in (2, 5, 9):
        oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        ctx.L.lsdgpu_ref_import(ctx.ptr, 0)
        p.sync_counters()
        if not with_mask:
            oracle.lib().lsdo_frame_clear_refPixelWasGood(p.oframes[k].ptr)
        else:
            # give the GPU frame the oracle's good mask by tracking it there as well (mask parity is tested
            # in test_gpu_track); tracking overwrites the pose, so restore the oracle's
            trk = abi.SE3Tracker(ctx, mode=0)
            trk.trackFrame(0, k, IDENT if k == 2 else p.oframes[k].thisToParent()[:7])
            ctx.set_pose(k, p.oframes[k].thisToParent(), 0, oracle.lib().lsdo_frame_initialTrackedResidual(p.oframes[k].ptr))
            ctx.set_counters(0, *[oracle.lib().lsdo_frame_numFramesTrackedOnThis(p.okf.ptr), oracle.lib().lsdo_frame_numMappedOnThis(p.okf.ptr)])
        p.odm.updateKeyframe([p.oframes[k]])
        p.gdm.updateKeyframe([k])
    if not with_mask:
        p.compare(exact=True)
    # propagate only
    before_o = p.odm.current().copy()
    p.odm.propagateDepth(p.oframes[9])
    p.gdm.propagateDepth(9)
    rep = p.compare(exact=not with_mask, rtol=1e-3, max_flag_mismatch=0 if not with_mask else 40)
    assert rep["n_valid"] > 5000
    # restore and run the whole createKeyFrame on both sides
    p.odm.set_current(before_o)
    p.gdm.setHypotheses(0, before_o, do_set_depth=False)
    p.odm.createKeyFrame(p.oframes[9])
    q = p.gdm.createKeyFrame(9)
    qo = p.oframes[9].thisToParent()
    # the rescale factor comes from the reference's sequential fp32 `sumIdepth +=` (DepthMap.cpp:1286-1294): the device reproduces
    # that sum bit for bit (csrc/seqsum.cuh) whenever it sums the same hypotheses -- without the tracking mask the maps are
    # identical before the sum, so everything after it is too
    assert np.allclose(q[:7], qo[:7], atol=1e-12)
    if not with_mask:
        assert np.float32(q[7]).tobytes() == np.float32(qo[7]).tobytes()
        p.compare(exact=True)
    else:
        assert abs(q[7] - qo[7]) <= 2e-5 * qo[7]
        p.compare(exact=False, rtol=2e-5, max_flag_mismatch=40)
    assert ctx.L.lsdgpu_depth_active_keyframe(ctx.ptr) == 9
    idg, ido = ctx.download(9, abi.BUF_IDEPTH, 0), p.oframes[9].idepth(0)
    assert ((idg > 0) != (ido > 0)).sum() <= (0 if not with_mask else 40)
    both = (idg > 0) & (ido > 0)
    if not with_mask:
        assert np.array_equal(idg, ido)
    assert np.max(np.abs(idg[both] - ido[both]) / ido[both]) <= 2e-5


# ---- SE3 tracker --------------------------------------------------------------------------------------------------------------
def se3_setup(ctx, oracle, seq, frames, k):
    """keyframe 0 on ground-truth depth and frame k, on both sides -> the oracle's (keyframe, frame)"""
    img0, d0 = frames[0]
    ctx.upload(0, img0)
    ctx.set_depth_gt(0, d0)
    okf = oracle.Frame(0, img0, seq.K)
    okf.setDepthFromGroundTruth(d0)
    ctx.upload(k, frames[k][0])
    return okf, oracle.Frame(k, frames[k][0], seq.K)


def se3_eval_each_level(ctx, oracle, seq, frames, mask_tol=1e-4, sum_noise=False):
    """one SE3 evaluation of frame 3 on levels 4..1, from identity and from near the truth with an affine guess; the good-mask of
    level 1 to mask_tol.  sum_noise: affine b may also differ by the reference's own summation error, its distance to the same
    sums taken exactly (besides check_se3_eval's 5e-3 grey levels: up to 1e-2 at level 1 with minUseGrad 2.5, where the device
    lands on the exact value)"""
    okf, of = se3_setup(ctx, oracle, seq, frames, 3)
    trk = abi.SE3Tracker(ctx)
    inv = se3_inverse(oracle, seq.frame_to_ref_qt(3))
    g = ctx.get_globals()
    for level in (4, 3, 2, 1):
        for pose, a, b in ((IDENT.astype(np.float32), 1.0, 0.0), (inv.astype(np.float32), 0.98, 1.5)):
            got = trk.eval(0, 3, level, pose, a, b, write_mask=level == 1)
            noise = 0.0
            if sum_noise:
                oracle.set_globals(exactTrackingSums=1, **g)
                exact = oracle.se3_eval(okf, of, level, pose, a, b)
                oracle.set_globals(**g)
            want = oracle.se3_eval(okf, of, level, pose, a, b, write_mask=level == 1)
            if sum_noise:
                noise = abs(want.affine_b_lastIt - exact.affine_b_lastIt)
            check_se3_eval(got, want, affine_b_noise=noise)
            if level == 1:
                assert (ctx.download(3, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < mask_tol


def se3_track(ctx, oracle, seq, frames, mode, k, sum_noise=False, diverges=False, usage_points=0):
    """trackFrame of frame k on keyframe 0 from identity, checked by check_se3_track.  sum_noise: the pose and the point usage may
    also differ by the reference's own summation noise, their distance to the same tracking with exact sums (the point usage also
    by how much it moves between the oracle's final pose and the device's); usage_points: the point usage may also differ by that
    many level-1 points' worth (1 / refNum each)"""
    okf, of = se3_setup(ctx, oracle, seq, frames, k)
    trk = abi.SE3Tracker(ctx, mode=mode)
    pose_g = trk.trackFrame(0, k, IDENT)
    r = oracle.se3_track(okf, of, IDENT)
    noise, usage_noise = (0.0, 0.0), 0.0
    if sum_noise:
        g = ctx.get_globals()
        oracle.set_globals(exactTrackingSums=1, **g)
        try:
            okfx = oracle.Frame(0, frames[0][0], seq.K)
            okfx.setDepthFromGroundTruth(frames[0][1])
            rx = oracle.se3_track(okfx, oracle.Frame(k, frames[k][0], seq.K), IDENT)
        finally:
            oracle.set_globals(**g)
        noise = pose_err(np.array(r.frameToRef_qt), np.array(rx.frameToRef_qt))
        # the point usage at the device's pose against the oracle's, both at the oracle's (a, b): how far it moves over the pose gap
        fk = oracle.Frame(k, frames[k][0], seq.K)
        at = [oracle.se3_eval(okf, fk, 1, se3_inverse(oracle, q).astype(np.float32), r.affineEstimation_a,
                              r.affineEstimation_b).pointUsage for q in (pose_g, np.array(r.frameToRef_qt))]
        usage_noise = abs(r.pointUsage - rx.pointUsage) + abs(at[0] - at[1])
    if usage_points:
        # the reported point usage is that of the LAST evaluated pose, a rejected candidate whenever level 1 ends on a step below
        # stepSizeMin (SE3Tracker.cpp:432-441); that candidate is the final pose plus a step solved from each side's own sums,
        # so a point at the image border can be inside for one side and outside for the other.  Each such point moves the usage
        # by up to 1 / refNum, as it moves the good / bad counts check_se3_track holds to 2.
        usage_noise += usage_points / len(okf.point_cloud(1)[0])
    check_se3_track(ctx, trk, k, pose_g, r, of, diverges=diverges, noise=noise, usage_noise=usage_noise)


# ---- Sim3 tracker -------------------------------------------------------------------------------------------------------------
SIM3_KEYFRAMES = ((0, 1.0), (6, 1.0), (12, 1.05))       # (frame, depth scale): keyframe 12 carries a 1.05x larger map


def gt_keyframes(ctx, oracle, seq, kfs=SIM3_KEYFRAMES):
    """keyframes on scaled ground-truth depth on both sides -> frame id -> oracle Frame"""
    of = {}
    for k, sc in kfs:
        img, z = seq.render(k)
        z = (z * sc).astype(np.float32)
        ctx.upload(k, img)
        ctx.set_depth_gt(k, z)
        of[k] = oracle.Frame(k, img, seq.K)
        of[k].setDepthFromGroundTruth(z)
    return of


def sim3_setup(oracle, w=640, h=480):
    """-> (sequence, context, Sim3Tracker, gt_keyframes) of the seed-1234 stream at w x h"""
    seq = synth.Sequence(w, h, seed=1234)
    ctx = abi.Context(w, h, seq.K, max_frames=8)
    of = gt_keyframes(ctx, oracle, seq)
    return seq, ctx, abi.Sim3Tracker(ctx), of


def sim3_eval(trk, oracle, seq, of):
    """single Sim3 evaluations of the keyframes of gt_keyframes: coarse and fine levels, both directions, an affine guess, and the
    pair with a scale ratio"""
    for (ref, fr), lvl, a, b in (((0, 6), 4, 1.0, 0.0), ((0, 6), 2, 1.0, 0.0), ((6, 0), 1, 0.97, 1.5), ((0, 12), 3, 1.0, 0.0)):
        r2f = sim3_inverse(oracle, sim3_init(seq, fr, ref))
        want = oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b)
        assert want.warpedSize > 100
        check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), want)


def sim3_batch(trk, oracle, seq, of, exact_twin=False):
    """all ordered pairs of keyframes in one launch == the same problems one by one (bit-identical) == the oracle.
    exact_twin (non-default settings): the five affine-lighting sums of calcSim3Buffers carry fp32 noise that feeds back through
    every accepted step (oracle_sim3_track); off the defaults it can flip an LM decision of the reference arithmetic (minUseGrad
    10, pair 12 -> 0) or move its translation by 5e-4 (cameraPixelNoise2 1, pair 0 -> 6), and the device follows the same
    arithmetic with those sums exact.  So: the device against the exact-sum twin always, and against the reference arithmetic
    wherever that agrees with its own exact-sum twin"""
    pairs = [(a, b) for a in of for b in of if a != b]
    inits = np.array([sim3_init(seq, fr, ref) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    g = trk.ctx.get_globals() if exact_twin else None
    for (ref, fr), init, r in zip(pairs, inits, res):
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        assert bytes(trk.last) == bytes(r)
        if not exact_twin:
            check_sim3_track(r, oracle.sim3_track(of[ref], of[fr], init, 4, 1))
            continue
        want, exact = oracle_sim3_track(oracle, of[ref], of[fr], init, g=g)
        check_sim3_track(r, exact)
        if list(want.numCalcResidualCalls) == list(exact.numCalcResidualCalls) and \
                max(sim3_err(want.frameToRef_qts, exact.frameToRef_qts)) <= 5e-5:
            check_sim3_track(r, want)


# ---- permaRef -----------------------------------------------------------------------------------------------------------------
def perma_setup(ctx, oracle, seq, kf_ids, min_points):
    """keyframes on ground-truth depth on both sides, each set as permaRef (more than min_points points) -> (SE3Tracker,
    frame id -> oracle PermaRef)"""
    trk = abi.SE3Tracker(ctx)
    prs = {}
    for k in kf_ids:
        img, d = seq.render(k)
        ctx.upload(k, img)
        ctx.set_depth_gt(k, d)
        okf = oracle.Frame(k, img, seq.K)
        okf.setDepthFromGroundTruth(d)
        prs[k] = oracle.PermaRef(okf)
        assert trk.setPermaRef(k) == prs[k].n > min_points
    return trk, prs


def perma_batch(ctx, oracle, seq, trk, prs, fid):
    """trackFrameOnPermaref of frame fid on every permaRef of prs in one launch, from the ground-truth relative pose and from
    identity -> the number of candidates the oracle tracked well"""
    img, _ = seq.render(fid)
    ctx.upload(fid, img)
    of = oracle.Frame(fid, img, seq.K)
    ids, inits = [], []
    for k in prs:
        gt_inv = se3_inverse(oracle, seq.frame_to_ref_qt(fid, ref=k))
        ids += [k, k]
        inits += [gt_inv, IDENT]
    res = trk.trackFrameOnPermaref(ids, fid, np.array(inits))
    return sum(check_perma_track(g, prs[k].track(of, init)) for k, init, g in zip(ids, inits, res))


# ---- Sim3 and permaRef on keyframes the device's mapper finished ---------------------------------------------------------------
def hyp_of_planes(oracle, idepth, var):
    """hypotheses that Frame::setDepth turns back into these level-0 planes: valid pixels (var > 0) are >= -0.05 there, so
    setDepth keeps them as they are and turns every other pixel into -1 / -1 again"""
    hyp = np.zeros(idepth.shape, oracle.HYP_DTYPE)
    hyp["isValid"] = var > 0
    hyp["idepth"] = hyp["idepth_smoothed"] = idepth
    hyp["idepth_var"] = hyp["idepth_var_smoothed"] = var
    return hyp


def mirror(oracle, ctx, seq, kf, img):
    """an oracle Frame of the same image given the device keyframe's level-0 plane through Frame::setDepth"""
    f = oracle.Frame(kf, img, seq.K)
    set_depth(f, hyp_of_planes(oracle, ctx.download(kf, abi.BUF_IDEPTH, 0), ctx.download(kf, abi.BUF_IDEPTH_VAR, 0)))
    return f


def pyramid_mismatches(ctx, kf, of):
    """(level, plane) pairs whose bits differ between the device keyframe and its oracle Frame"""
    bad = []
    for lvl in range(abi.LEVELS):
        for name, buf, plane in (("idepth", abi.BUF_IDEPTH, of.idepth), ("idepthVar", abi.BUF_IDEPTH_VAR, of.idepthVar)):
            if not np.array_equal(ctx.download(kf, buf, lvl).view(np.uint32), plane(lvl).view(np.uint32)):
                bad.append((lvl, name))
    return bad


class MappedRun:
    """A GpuStream of the seed-1234 sequence of `motion` (tests/motions.py; the default twist by default) with its finished
    keyframes resident and an oracle mirror of each.  `seq`, if given, is run instead; `motion` then only names the run, as the
    key of POSE_SENSITIVE_DEPTH_RESIDUAL.  After every keyframe change it compares the pyramids of every resident keyframe with
    the oracle (`checks`)."""

    def __init__(self, oracle, w, h, motion="default", seq=None):
        from tests import motions
        self.motion = motion
        self.seq = seq = motions.sequence(motion, w, h) if seq is None else seq
        self.ctx = ctx = abi.Context(w, h, seq.K, max_frames=12)
        self.gs = gs = GpuStream(ctx, kf_every=MAPPED_KF_EVERY, keep_keyframes=True)
        self.images = {}
        img, d = seq.render(0)
        self.images[0] = img
        gs.init_gt(0, img, d)
        self.of, self.checks = {}, []
        for k in range(1, MAPPED_FRAMES):
            self.images[k] = seq.render(k)[0]
            change = gs.next_is_keyframe_change()
            gs.step(k, self.images[k])
            if not change:
                continue
            for kf in gs.keyframe_ids[:-1]:           # finished: mirrored once, then re-checked after every later change
                if kf not in self.of:
                    self.of[kf] = mirror(oracle, ctx, seq, kf, self.images[kf])
                self.checks.append((k, kf, pyramid_mismatches(ctx, kf, self.of[kf])))
            active = gs.keyframe_ids[-1]              # the new keyframe as createKeyFrame left it
            self.checks.append((k, active, pyramid_mismatches(ctx, active, mirror(oracle, ctx, seq, active, self.images[active]))))
        self.kfs = gs.keyframe_ids[:-1]
        self.active = gs.keyframe_ids[-1]
        self.active_hyp = gs.map.current()            # the active keyframe's hypotheses (DepthMap::currentDepthMap)

    def frame_to_ref(self, oracle, ref, fr, perturb=True):
        """the relative Sim3 SlamSystem starts from: reference->getScaledCamToWorld().inverse() * frame->getScaledCamToWorld()
        (scale ratio of the two keyframes included), with util.sim3_init's perturbation of translation and scale"""
        c2w = dict(zip(self.gs.keyframe_ids, self.gs.keyframe_cam_to_world))
        q = sim3_mul_qts(sim3_inverse(oracle, c2w[ref]), c2w[fr])
        if perturb:
            q[4:7] += SIM3_DT
            q[7] *= SIM3_SCALE
        return q

    def ref_to_frame(self, oracle, ref, fr, perturb=True):
        return sim3_inverse(oracle, self.frame_to_ref(oracle, ref, fr, perturb))

    def pairs(self):
        return [(a, b) for a in self.kfs for b in self.kfs if a != b]

    def close(self):
        self.ctx.close()


def mapped_mirror_bit_exact(mapped):
    """every resident keyframe's idepth / idepthVar pyramid (levels 0-4) equals the oracle's Frame::setDepth of the same
    level-0 plane, and a finished keyframe stays so through the later map swaps and createKeyFrame calls of the run"""
    assert len(mapped.kfs) >= 3
    assert [kf for _, kf, _ in mapped.checks].count(mapped.kfs[0]) >= 3
    bad = [(k, kf, m) for k, kf, m in mapped.checks if m]
    assert not bad, bad
    ctx = mapped.ctx
    spread = []
    for kf in mapped.kfs:                             # what these tests are about: a semi-dense map, no variance shared by all
        var = ctx.download(kf, abi.BUF_IDEPTH_VAR, 0)
        v = var[var > 0]
        assert 0.2 < v.size / var.size < 0.7 and np.unique(v).size > 100, (kf, v.size / var.size, np.unique(v).size)
        spread.append(v.max() / v.min())
    assert max(spread) > 30, spread
    scales = [q[7] for q in mapped.gs.keyframe_cam_to_world]
    assert max(scales) / min(scales) > 1.2, scales       # createKeyFrame rescales every new keyframe


def mapped_sim3_eval(run, oracle):
    """one Sim3 evaluation per ordered pair, perturbed and not, levels 4..1, two affine estimates"""
    trk = abi.Sim3Tracker(run.ctx)
    n_no_depth = 0
    for ref, fr in run.pairs():
        for perturb in (True, False):
            r2f = run.ref_to_frame(oracle, ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in AB:
                    got = trk.eval(ref, fr, lvl, r2f, a, b)
                    want = oracle.sim3_eval(run.of[ref], run.of[fr], lvl, r2f, a, b)
                    assert want.warpedSize > 10, (ref, fr, lvl)
                    check_sim3_eval(got, want)
                    n_no_depth += want.numTermsD < want.numTermsP      # warped onto frame pixels without depth (sim3.cuh:116-117)
    assert n_no_depth > 0


def mapped_sim3_eval_settings(run, oracle):
    """var_weight and huber_d other than their defaults (1, 3) reach the kernel's weights"""
    trk = abi.Sim3Tracker(run.ctx)
    st = oracle.default_track_settings(main_tracker=False)
    for s in (trk.settings, st):
        s.var_weight, s.huber_d = 2.5, 1.5
    for ref, fr in run.pairs():
        r2f = run.ref_to_frame(oracle, ref, fr)
        for lvl in (4, 3, 2, 1):
            a, b = AB[lvl % 2]
            check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), oracle.sim3_eval(run.of[ref], run.of[fr], lvl, r2f, a, b, settings=st))


def _sum_noise(oracle, ref, fr, init, lo, hi, *results):
    """-> (the all-sums-exact twin of trackFrameSim3, each result's pose distance to it): how far the fp32 summation of each
    oracle result alone moved its pose"""
    tw = oracle_sim3_exact(oracle, ref, fr, init, lo, hi)
    return tw, [max(sim3_err(r.frameToRef_qts, tw.frameToRef_qts)) for r in results]


def mapped_sim3_track(run, oracle, sum_noise=False, lm_flips=()):
    """trackFrameSim3 per ordered pair over levels 4..1 and 3..2 (lastDepthResidual of pin_cases.POSE_SENSITIVE_DEPTH_RESIDUAL
    against the exact-sum twin to the reference tolerance).  sum_noise: the pose may also differ from each oracle result by
    that result's own distance to the all-sums-exact twin, which holds the device to POSE_TOL.  lm_flips (with sum_noise): the
    (motion, reference keyframe, frame keyframe, startLevel, finalLevel) calls where the reference arithmetic takes another LM
    decision than its all-sums-exact twin; there the device is held to the twin alone"""
    trk = abi.Sim3Tracker(run.ctx)
    n_converged = 0
    for ref, fr in run.pairs():
        init = run.frame_to_ref(oracle, ref, fr)
        for lo, hi in ((4, 1), (3, 2)):
            est = trk.trackFrameSim3(ref, fr, init, lo, hi)
            want, exact = oracle_sim3_track(oracle, run.of[ref], run.of[fr], init, lo, hi)
            noise = (0.0, 0.0)
            if sum_noise:
                tw, noise = _sum_noise(oracle, run.of[ref], run.of[fr], init, lo, hi, want, exact)
                check_sim3_track(trk.last, tw)
                if (run.motion, ref, fr, lo, hi) in lm_flips:
                    assert list(want.numCalcResidualCalls) != list(tw.numCalcResidualCalls)
                    assert np.array_equal(est, np.array(trk.last.frameToRef_qts))
                    n_converged += not want.diverged
                    continue
            check_sim3_track(trk.last, want, pose_noise=noise[0])
            sensitive = (run.motion, ref, fr, lo, hi) in POSE_SENSITIVE_DEPTH_RESIDUAL
            check_sim3_track(trk.last, exact, res_tol=5e-4, depth_res_tol=2e-2 if sensitive else None, pose_noise=noise[1])
            assert np.array_equal(est, np.array(trk.last.frameToRef_qts))
            n_converged += not want.diverged
    assert n_converged >= len(run.pairs())


def mapped_sim3_batch(run, oracle, sum_noise=False):
    """every ordered pair in one launch == one by one (bit-identical) == the oracle (sum_noise: as mapped_sim3_track)"""
    trk = abi.Sim3Tracker(run.ctx)
    pairs = run.pairs()
    inits = np.array([run.frame_to_ref(oracle, ref, fr) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    for (ref, fr), init, r in zip(pairs, inits, res):
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        assert bytes(trk.last) == bytes(r)
        want = oracle.sim3_track(run.of[ref], run.of[fr], init, 4, 1)
        noise = (0.0,)
        if sum_noise:
            tw, noise = _sum_noise(oracle, run.of[ref], run.of[fr], init, 4, 1, want)
            check_sim3_track(r, tw)
        check_sim3_track(r, want, pose_noise=noise[0])


def mapped_perma(run, oracle, noise_aware=False):
    """setPermaRef of each finished keyframe, the overlap at random poses, trackFrameOnPermaref of PERMA_FRAME from its
    ground-truth pose (translation in the keyframe's map units: the chain's scale of the keyframe) and from identity.
    noise_aware: the pose tolerance grows by the reference's own summation noise of each tracking (util.perma_noise)"""
    ctx, seq = run.ctx, run.seq
    se3 = abi.SE3Tracker(ctx)
    prs = {}
    for k in run.kfs:
        prs[k] = oracle.PermaRef(run.of[k])
        assert se3.setPermaRef(k) == prs[k].n > 30
    want = check_perma_overlap(se3, oracle, prs, np.random.default_rng(3))
    assert want.min() < 0.9 < want.max()
    img = seq.render(PERMA_FRAME)[0]
    ctx.upload(PERMA_FRAME, img)
    of = oracle.Frame(PERMA_FRAME, img, seq.K)
    scale = dict(zip(run.gs.keyframe_ids, [q[7] for q in run.gs.keyframe_cam_to_world]))
    ids, inits = [], []
    for k in prs:
        gt = seq.frame_to_ref_qt(PERMA_FRAME, ref=k)
        gt[4:7] /= scale[k]
        gt_inv = se3_inverse(oracle, gt)
        for init in (gt_inv, IDENT):
            ids.append(k)
            inits.append(init)
    res = se3.trackFrameOnPermaref(ids, PERMA_FRAME, np.array(inits))
    n_good = 0
    for k, init, g in zip(ids, inits, res):
        noise = perma_noise(oracle, prs[k], of, init) if noise_aware else (0.0, 0.0)
        n_good += check_perma_track(g, prs[k].track(of, init), noise)
    assert n_good >= 2
    ctx.release(PERMA_FRAME)


def mapped_adversarial(run, oracle):
    """the edited map of the active keyframe (pin_cases.adversarial_edit) loaded on both sides (DepthMap setHypotheses +
    Frame::setDepth): pyramids, permaRef and Sim3 on it.  Points with negative idepth lie behind the camera and can warp into
    the image mirrored; the reference has no Wz > 0 test in calcSim3Buffers or checkPermaRefOverlap, and neither have the
    kernels."""
    ctx, seq = run.ctx, run.seq
    kf, other = run.active, run.kfs[-1]
    hyp = adversarial_edit(run.active_hyp, np.random.default_rng(7))
    run.gs.map.setHypotheses(kf, hyp, do_set_depth=True)
    okf = oracle.Frame(kf, run.images[kf], seq.K)
    set_depth(okf, hyp)
    assert not pyramid_mismatches(ctx, kf, okf)
    idepth0, valid0 = okf.idepth(0), okf.idepthVar(0) > 0
    assert ((idepth0 < 0) & valid0).sum() >= 50 and ((idepth0 == 0) & valid0).sum() >= 32
    for lvl in range(1, abi.LEVELS):                  # the cancelled blocks reach every level
        assert ((okf.idepth(lvl) == 0) & (okf.idepthVar(lvl) > 0)).any(), lvl

    se3 = abi.SE3Tracker(ctx)
    pr = oracle.PermaRef(okf)
    assert se3.setPermaRef(kf) == pr.n
    check_perma_overlap(se3, oracle, {kf: pr}, np.random.default_rng(5))

    of = dict(run.of)
    of[kf] = okf
    trk = abi.Sim3Tracker(ctx)
    for ref, fr in ((kf, other), (other, kf)):
        r2f = run.ref_to_frame(oracle, ref, fr)
        for lvl in range(abi.LEVELS):
            for a, b in AB:
                check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b))
        init = run.frame_to_ref(oracle, ref, fr)
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        want, exact = oracle_sim3_track(oracle, of[ref], of[fr], init)
        assert trk.diverged == bool(want.diverged)
        if not want.diverged:
            check_sim3_track(trk.last, want)
            check_sim3_track(trk.last, exact, res_tol=5e-4)


# ---- stream groups ------------------------------------------------------------------------------------------------------------
GROUP_KF_EVERY = 20
_group_frames = {}


def _group_sequence(w, h, s, n, make=None):
    """stream s: its own synthetic sequence (seed 1234 + 1000 s, as scripts/bench_streams.py), or make(w, h) if given"""
    key = (w, h, s, make)
    seq, fr = _group_frames.get(key, (None, []))
    if seq is None:
        seq = make(w, h) if make else synth.Sequence(w, h, seed=1234 + 1000 * s)
    while len(fr) < n:
        fr.append(seq.render(len(fr)))
    _group_frames[key] = (seq, fr)
    return seq, fr


def run_streams(w, h, phases, n_steps, grouped, before_step=None, sequences=None):
    """one GpuStream per phase (keyframe every GROUP_KF_EVERY frames, shifted by its phase), stepped n_steps times.
    sequences: per stream a function (w, h) -> sequence to use instead of its own seeded one.
    grouped(k): step k is one group call (True) or one single call per stream (False).  before_step(k, streams) may change
    the streams' state first.  Returns per step and stream what util.observe saw, whether the step diverged and whether it
    changed keyframe."""
    streams, frames = [], []
    for s, ph in enumerate(phases):
        seq, fr = _group_sequence(w, h, s, n_steps + 1, sequences[s] if sequences else None)
        ctx = abi.Context(w, h, seq.K, max_frames=8)
        gs = GpuStream(ctx, mode=1, kf_every=GROUP_KF_EVERY, kf_phase=ph)
        gs.init_gt(0, fr[0][0], fr[0][1])
        streams.append(gs)
        frames.append(fr)
    group = GpuStreamGroup(streams)
    log = []
    try:
        for k in range(1, n_steps + 1):
            if before_step:
                before_step(k, streams)
            kf = [gs.next_is_keyframe_change() for gs in streams]
            if grouped(k):
                try:
                    group.step([k] * len(streams), images=[f[k][0] for f in frames])
                except RuntimeError:
                    pass
                qts = [group._qts[i].copy() if kf[i] else None for i in range(len(streams))]
            else:
                qts = []
                for i, (gs, f) in enumerate(zip(streams, frames)):
                    try:
                        gs.step(k, f[k][0])
                    except RuntimeError:
                        pass
                    qts.append(gs._qts.copy() if kf[i] else None)
            log.append([dict(observe(gs, k, q), diverged=bool(gs.tracker.diverged), kf=kf[i])
                        for i, (gs, q) in enumerate(zip(streams, qts))])
    finally:
        for gs in streams:
            gs.ctx.close()
    return log
