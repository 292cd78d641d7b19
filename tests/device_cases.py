"""Device scenarios that the parity tests run under more than one axis (the default stream, non-default run-time settings, other
camera motions, other frame shapes, mapped keyframes).  Each drives the oracle and the CUDA path through one call sequence and
checks the results with tests/util.py; the caller chooses the context, the stream and its own thresholds."""
import numpy as np

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from tests.util import (IDENT, Pair, check_perma_track, check_se3_eval, check_se3_track, check_sim3_eval, check_sim3_track,
                        kf_depth_equal, new_depth, observe, oracle_sim3_track, pose_err, se3_inverse, sim3_err, sim3_init,
                        sim3_inverse, sim3_mul, tracked_pair)


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


def se3_track(ctx, oracle, seq, frames, mode, k, sum_noise=False, diverges=False):
    """trackFrame of frame k on keyframe 0 from identity, checked by check_se3_track.  sum_noise: the pose may also differ by the
    reference's own summation noise, its distance to the same tracking with exact sums"""
    okf, of = se3_setup(ctx, oracle, seq, frames, k)
    trk = abi.SE3Tracker(ctx, mode=mode)
    pose_g = trk.trackFrame(0, k, IDENT)
    r = oracle.se3_track(okf, of, IDENT)
    noise = (0.0, 0.0)
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
    check_se3_track(ctx, trk, k, pose_g, r, of, diverges=diverges, noise=noise)


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


# ---- stream groups ------------------------------------------------------------------------------------------------------------
GROUP_KF_EVERY = 20
_group_frames = {}


def _group_sequence(w, h, s, n):
    """stream s: its own synthetic sequence (seed 1234 + 1000 s, as scripts/bench_streams.py)"""
    key = (w, h, s)
    seq, fr = _group_frames.get(key, (None, []))
    if seq is None:
        seq = synth.Sequence(w, h, seed=1234 + 1000 * s)
    while len(fr) < n:
        fr.append(seq.render(len(fr)))
    _group_frames[key] = (seq, fr)
    return seq, fr


def run_streams(w, h, phases, n_steps, grouped, before_step=None):
    """one GpuStream per phase (keyframe every GROUP_KF_EVERY frames, shifted by its phase), stepped n_steps times.
    grouped(k): step k is one group call (True) or one single call per stream (False).  before_step(k, streams) may change
    the streams' state first.  Returns per step and stream what util.observe saw, whether the step diverged and whether it
    changed keyframe."""
    streams, frames = [], []
    for s, ph in enumerate(phases):
        seq, fr = _group_sequence(w, h, s, n_steps + 1)
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
