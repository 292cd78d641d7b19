"""GPU parity at the reference's NON-DEFAULT run-time settings (util/settings.cpp:80-88, changed between frames by ROS dynamic
reconfigure: cfg/LSDParams.cfg:13-34, IOWrapper/ROS/rosReconfigure.h:81-91).  Every other parity test runs at the defaults, so a
kernel that hard-codes a default, compares a threshold with the wrong operator, or reads a setting from the wrong context would pass
there.  Here the context (abi.Context(..., **g)) and the oracle (oracle.set_globals(**g)) run under the same settings -- the
oracle is pinned to the reference-compiled library at each of them by tests/test_ref_pin_globals.py:
  * the depth map, pass by pass and through updateKeyframe / finalizeKeyFrame + createKeyFrame / update_keyframe_refs: bit for bit;
  * SE3 evaluation and tracking (both modes), Sim3 evaluation and batch tracking, permaRef batch tracking: the tolerances of
    test_gpu_track.py, test_gpu_sim3.py and test_gpu_perma.py, identical LM call counters;
  * a closed track + map loop replayed step by step (oracle/replay.py follows the context's settings), a change of settings
    between two steps, and two contexts with different settings in one group call."""
import contextlib

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from oracle import replay
from tests.test_gpu_depth import Pair
from tests.test_gpu_group import _assert_same, _observe
from tests.test_gpu_sim3 import _check_eval as _check_sim3_eval
from tests.test_gpu_sim3 import _check_track as _check_sim3_track
from tests.test_gpu_sim3 import _d
from tests.test_gpu_sim3 import _init as _sim3_init
from tests.test_gpu_sim3 import _sim3_err
from tests.test_gpu_track import _cmp_eval
from tests.test_ref_pin_globals import SETS
from tests.util import IDENT, pose_err, rot_angle

pytestmark = pytest.mark.gpu

G = {name: g for name, (g, _) in SETS.items()}
COMBINED = G["combined"]
DEPTH_SETS = [s for s in G if s != "useAffineLightningEstimation=0"]          # that one is read by the trackers only
TRACK_SETS = [s for s in G if s.startswith(("cameraPixelNoise2", "useAffine", "minUseGrad")) or s == "combined"]
MIN_USE_GRAD_SETS = [s for s in G if "minUseGrad" in G[s]]


@contextlib.contextmanager
def _under(oracle, g, w, h, K, max_frames=12):
    """a context created with the settings g, and the oracle switched to them; both back at the defaults afterwards"""
    oracle.set_globals(**g)
    ctx = abi.Context(w, h, K, max_frames=max_frames, **g)
    try:
        yield ctx
    finally:
        ctx.close()
        oracle.set_globals()


@pytest.fixture(params=DEPTH_SETS)
def depth_ctx(request, oracle, seq_small):
    with _under(oracle, G[request.param], seq_small.w, seq_small.h, seq_small.K) as ctx:
        yield ctx


@pytest.fixture(params=TRACK_SETS)
def track_ctx(request, oracle, seq_small):
    with _under(oracle, G[request.param], seq_small.w, seq_small.h, seq_small.K) as ctx:
        yield ctx


def _new_depth(p, k):
    """the keyframe's depth was read since its last update (importFrame, SlamSystem.cpp:907-912), on both sides"""
    p.o.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
    p.ctx.L.lsdgpu_ref_import(p.ctx.ptr, 0)
    p.sync_counters()


def _kf_depth_equal(ctx, okf, fid):
    """Frame::setDepth's pyramids (what the tracker reads) bit for bit"""
    for lvl in range(5):
        assert np.array_equal(ctx.download(fid, abi.BUF_IDEPTH, lvl).view(np.uint32), okf.idepth(lvl).view(np.uint32)), lvl
        assert np.array_equal(ctx.download(fid, abi.BUF_IDEPTH_VAR, lvl).view(np.uint32), okf.idepthVar(lvl).view(np.uint32)), lvl


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def test_observe_from_gt_depth_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    """observeDepth with two reference frames (line stereo, the minUseGrad gates of the observe pass)"""
    p = Pair(depth_ctx, oracle, seq_small, frames_small, "gt")
    ofs = [p.add_frame(k) for k in (1, 2)]
    p.sync_counters()
    p.odm.observeDepth(ofs)
    p.gdm.observeDepth([1, 2])
    assert p.compare(exact=True)["n_valid"] > 3000


def test_random_init_observe_and_update_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    """random hypotheses drive the line stereo through its failure branches (the -2 of a negative inverse depth among them)"""
    p = Pair(depth_ctx, oracle, seq_small, frames_small, "random")
    of = p.add_frame(4)
    p.odm.observeDepth([of])
    p.gdm.observeDepth([4])
    p.compare(exact=True)
    for k in (6, 8, 10):
        of = p.add_frame(k)
        _new_depth(p, k)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
        p.compare(exact=True)
    _kf_depth_equal(depth_ctx, p.okf, 0)


def test_fill_holes_regularize_and_integral_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    p = Pair(depth_ctx, oracle, seq_small, frames_small, "random")
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
    assert np.array_equal(p.gdm.integral(), p.odm.integral())
    for occl in (False, True):
        p.odm.regularize(occl, 24)
        p.gdm.regularize(occl, 24)
        p.compare(exact=True)


def test_update_keyframe_sequence_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    """updateKeyframe = observe + the fused fill-holes and regulariser (depth.cuh) + Frame::setDepth, 1 and 2 reference frames"""
    p = Pair(depth_ctx, oracle, seq_small, frames_small, "gt")
    for ks in ([1], [2, 3], [5]):
        ofs = [p.add_frame(k) for k in ks]
        _new_depth(p, ks[0])
        p.odm.updateKeyframe(ofs)
        p.gdm.updateKeyframe(ks)
        assert p.compare(exact=True)["n_valid"] > 3000
        _kf_depth_equal(depth_ctx, p.okf, 0)


def _sim3(oracle, fn, *args):
    out = np.zeros(8, np.float64)
    arrs = [np.ascontiguousarray(a, np.float64) for a in args]
    getattr(oracle.lib(), fn)(*[_d(a) for a in arrs], _d(out))
    return out


def test_finalize_create_keyframe_and_refs_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    """finalizeKeyFrame + createKeyFrame (propagation, rescale) and then update_keyframe_refs with frames tracked on the previous
    keyframe -- the scene at mean inverse depth 1 on keyframe 0, as in test_gpu_depth's test of the same sequence"""
    d0 = frames_small[0][1]
    sc = float(np.mean(1.0 / d0[d0 > 0]))
    frames = {k: (frames_small[k][0], (frames_small[k][1] * sc).astype(np.float32)) for k in range(13)}

    def qt(k):
        q = seq_small.frame_to_ref_qt(k).copy()
        q[4:7] *= sc
        return q
    ctx = depth_ctx
    p = Pair(ctx, oracle, seq_small, frames, "gt")
    for k in (1, 2, 3):
        of = p.add_frame(k, qt(k))
        _new_depth(p, k)
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
    _kf_depth_equal(ctx, of9, 9)
    c2w9 = of9.thisToParent()
    items = [(k, _sim3(oracle, "lsdo_sim3d_mul", _sim3(oracle, "lsdo_sim3d_inverse", c2w9), p.oframes[k].thisToParent()))
             for k in (4, 5)]
    before = p.gdm.current().copy()
    p.odm.updateKeyframe([p.oframes[4], p.oframes[5]])
    p.gdm.updateKeyframe(items)
    rep = p.compare(exact=True)
    after = p.gdm.current()
    both = (before["isValid"] != 0) & (after["isValid"] != 0)
    assert rep["n_valid"] > 3000 and int((before["idepth"][both] != after["idepth"][both]).sum()) > 200     # they did observe


@pytest.mark.parametrize("set_name", MIN_USE_GRAD_SETS)
def test_set_depth_gt_pyramids(oracle, seq_small, frames_small, set_name):
    """Frame::setDepthFromGroundTruth keeps a pixel iff its gradient passes minUseGrad (Frame.cpp)"""
    img0, d0 = frames_small[0]
    with _under(oracle, G[set_name], seq_small.w, seq_small.h, seq_small.K, max_frames=4) as ctx:
        ctx.upload(0, img0)
        ctx.set_depth_gt(0, d0)
        okf = oracle.Frame(0, img0, seq_small.K)
        okf.setDepthFromGroundTruth(d0)
        _kf_depth_equal(ctx, okf, 0)
        assert (okf.idepth(0) > 0).sum() > 1000


# ---- trackers ---------------------------------------------------------------------------------------------------------------
def _se3_setup(ctx, oracle, seq, frames, k):
    img0, d0 = frames[0]
    ctx.upload(0, img0)
    ctx.set_depth_gt(0, d0)
    okf = oracle.Frame(0, img0, seq.K)
    okf.setDepthFromGroundTruth(d0)
    ctx.upload(k, frames[k][0])
    return okf, oracle.Frame(k, frames[k][0], seq.K)


def test_se3_eval_each_level(track_ctx, oracle, seq_small, frames_small):
    okf, of = _se3_setup(track_ctx, oracle, seq_small, frames_small, 3)
    trk = abi.SE3Tracker(track_ctx)
    inv = np.zeros(7)
    oracle.lib().lsdo_se3d_inverse(_d(seq_small.frame_to_ref_qt(3)), _d(inv))
    g = track_ctx.get_globals()
    for level in (4, 3, 2, 1):
        for pose, a, b in ((IDENT.astype(np.float32), 1.0, 0.0), (inv.astype(np.float32), 0.98, 1.5)):
            got = trk.eval(0, 3, level, pose, a, b, write_mask=level == 1)
            oracle.set_globals(exactTrackingSums=1, **g)
            exact = oracle.se3_eval(okf, of, level, pose, a, b)
            oracle.set_globals(**g)
            want = oracle.se3_eval(okf, of, level, pose, a, b, write_mask=level == 1)
            # affine b is a difference of fp32 sums that cancel: besides _cmp_eval's 5e-3 grey levels it may differ from the
            # reference's sequential sums by their own error, their distance to the same sums taken exactly (up to 1e-2 at
            # level 1 with minUseGrad 2.5, where the device lands on the exact value)
            noise = abs(want.affine_b_lastIt - exact.affine_b_lastIt)
            assert abs(got.affine_b_lastIt - want.affine_b_lastIt) <= 5e-3 + noise, (level, a, got.affine_b_lastIt, want.affine_b_lastIt, noise)
            want.affine_b_lastIt = got.affine_b_lastIt
            _cmp_eval(got, want)
            if level == 1:
                assert (track_ctx.download(3, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < 1e-4


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 8])
def test_se3_track(track_ctx, oracle, seq_small, frames_small, mode, k):
    okf, of = _se3_setup(track_ctx, oracle, seq_small, frames_small, k)
    trk = abi.SE3Tracker(track_ctx, mode=mode)
    pose_g = trk.trackFrame(0, k, IDENT)
    r = oracle.se3_track(okf, of, IDENT)
    pose_o = np.array(r.frameToRef_qt)
    dt, ang = pose_err(pose_g, pose_o)
    assert dt <= 1e-4, (dt, pose_g, pose_o)
    assert ang <= 1e-4 * max(rot_angle(pose_o), 1e-2) + 1e-7, ang
    assert trk.trackingWasGood == bool(r.trackingWasGood) and trk.diverged == bool(r.diverged)
    assert abs(trk.lastResidual - r.lastResidual) <= 1e-3 * abs(r.lastResidual) + 1e-6
    assert abs(trk.affineEstimation_a - r.affineEstimation_a) <= 1e-3 and abs(trk.affineEstimation_b - r.affineEstimation_b) <= 5e-2
    assert list(trk.last.numCalcResidualCalls) == list(r.numCalcResidualCalls)
    assert list(trk.last.numCalcWarpUpdateCalls) == list(r.numCalcWarpUpdateCalls)
    assert (track_ctx.download(k, abi.BUF_GOODMASK) != of.refPixelWasGood()).mean() < 1e-3


def _keyframes_640(ctx, oracle, seq, kfs=((0, 1.0), (6, 1.0), (12, 1.05))):
    of = {}
    for k, sc in kfs:
        img, z = seq.render(k)
        z = (z * sc).astype(np.float32)
        ctx.upload(k, img)
        ctx.set_depth_gt(k, z)
        of[k] = oracle.Frame(k, img, seq.K)
        of[k].setDepthFromGroundTruth(z)
    return of


@pytest.mark.parametrize("set_name", TRACK_SETS)
def test_sim3_eval_and_track_batch(oracle, set_name):
    seq = synth.Sequence(640, 480, seed=1234)
    with _under(oracle, G[set_name], 640, 480, seq.K, max_frames=8) as ctx:
        of = _keyframes_640(ctx, oracle, seq)
        trk = abi.Sim3Tracker(ctx)
        for (ref, fr), lvl, a, b in (((0, 6), 4, 1.0, 0.0), ((0, 6), 2, 1.0, 0.0), ((6, 0), 1, 0.97, 1.5), ((0, 12), 3, 1.0, 0.0)):
            r2f = np.zeros(8)
            oracle.lib().lsdo_sim3d_inverse(_d(_sim3_init(seq, fr, ref)), _d(r2f))
            want = oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b)
            assert want.warpedSize > 100
            _check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), want)
        pairs = [(a, b) for a in of for b in of if a != b]
        inits = np.array([_sim3_init(seq, fr, ref) for ref, fr in pairs])
        res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
        g = ctx.get_globals()
        for (ref, fr), init, r in zip(pairs, inits, res):
            want = oracle.sim3_track(of[ref], of[fr], init, 4, 1)
            oracle.set_globals(exactAffineSums=1, **g)
            exact = oracle.sim3_track(of[ref], of[fr], init, 4, 1)
            oracle.set_globals(**g)
            # the five affine-lighting sums of calcSim3Buffers carry fp32 noise that feeds back through every accepted step
            # (test_gpu_sim3._oracle_track); off the defaults it can flip an LM decision of the reference arithmetic (minUseGrad 10,
            # pair 12 -> 0) or move its translation by 5e-4 (cameraPixelNoise2 1, pair 0 -> 6), and the device follows the same
            # arithmetic with those sums exact.  So: the device against the exact-sum twin always, and against the reference
            # arithmetic wherever that agrees with its own exact-sum twin
            _check_sim3_track(r, exact)
            if list(want.numCalcResidualCalls) == list(exact.numCalcResidualCalls) and \
                    max(_sim3_err(want.frameToRef_qts, exact.frameToRef_qts)) <= 5e-5:
                _check_sim3_track(r, want)


@pytest.mark.parametrize("set_name", TRACK_SETS)
def test_perma_track_batch(oracle, set_name):
    seq = synth.Sequence(640, 480, seed=1234)
    with _under(oracle, G[set_name], 640, 480, seq.K, max_frames=8) as ctx:
        trk = abi.SE3Tracker(ctx)
        prs = {}
        for k in (0, 6, 12):
            img, d = seq.render(k)
            ctx.upload(k, img)
            ctx.set_depth_gt(k, d)
            okf = oracle.Frame(k, img, seq.K)
            okf.setDepthFromGroundTruth(d)
            prs[k] = oracle.PermaRef(okf)
            assert trk.setPermaRef(k) == prs[k].n > 200
        img, _ = seq.render(9)
        ctx.upload(9, img)
        of = oracle.Frame(9, img, seq.K)
        ids, inits = [], []
        for k in prs:
            gt_inv = np.zeros(7)
            oracle.lib().lsdo_se3d_inverse(_d(seq.frame_to_ref_qt(9, ref=k)), _d(gt_inv))
            ids += [k, k]
            inits += [gt_inv, IDENT]
        n_good = 0
        for k, init, g in zip(ids, inits, trk.trackFrameOnPermaref(ids, 9, np.array(inits))):
            o = prs[k].track(of, init)
            assert bool(g.diverged) == bool(o.diverged)
            if o.diverged:
                continue
            dt, ang = pose_err(np.array(g.frameToRef_qt), np.array(o.frameToRef_qt))
            assert dt <= 1e-4 and ang <= 2e-6, (k, dt, ang)
            assert list(g.numCalcResidualCalls) == list(o.numCalcResidualCalls)
            assert list(g.numCalcWarpUpdateCalls) == list(o.numCalcWarpUpdateCalls)
            assert abs(g.lastResidual - o.lastResidual) <= 1e-3 * abs(o.lastResidual) + 1e-6
            assert bool(g.trackingWasGood) == bool(o.trackingWasGood)
            n_good += int(o.trackingWasGood)
        assert n_good >= 1


# ---- closed loop, mid-run change, group -------------------------------------------------------------------------------------
def _assert_step_ok(r):
    assert r["pose_rel"] <= 1e-4 + r["ref_noise_rel"], (r["frame"], r["pose_rel"], r["ref_noise_rel"])
    assert r["rot_rad"] <= 1e-6 + r["ref_noise_rot"], (r["frame"], r["rot_rad"])
    assert r["map_ok"], (r["frame"], r["map"])


def _defaults():
    g = abi.Globals()
    abi.load().lsdgpu_default_globals(g)
    return {name: getattr(g, name) for name, _ in abi.Globals._fields_}


def _same_globals(a, b):
    """settings a (every field) are the defaults overridden by b"""
    return all(np.float32(a[k]) == np.float32(b.get(k, d)) for k, d in _defaults().items())


def test_closed_loop_replay_under_combined_settings(seq_small, frames_small, oracle):
    """25 frames, keyframe changes at 10 and 20, every step replayed on the oracle under the context's settings"""
    reps = replay.run_with_replay(seq_small, frames_small, 26, kf_every=10, globals_kw=COMBINED)
    assert len(reps) == 25 and [r["frame"] for r in reps if r["kf_change"]] == [10, 20]
    for r in reps:
        assert _same_globals(r["globals"], COMBINED)
        _assert_step_ok(r)
    assert sum(r["counts_equal"] for r in reps) >= len(reps) - 2


def test_settings_changed_between_two_steps(seq_small, frames_small, oracle):
    """dynConfCb changes the settings between two frames: the step before the change ran with the old values, the step after it
    with the new ones (and not with the old: replaying it under those gives another result)"""
    change_at = 4
    images = {k: frames_small[k][0] for k in range(9)}
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=8)
    gs = GpuStream(ctx, mode=1, kf_every=6, fused_call=False)
    gs.init_gt(0, frames_small[0][0], frames_small[0][1])
    reps, stale = [], None
    try:
        for k in range(1, 9):
            if k == change_at:
                ctx.set_globals(**COMBINED)
            snap = replay.Snapshot(gs, images)
            holder = {}
            orig_clear = ctx.clear_good_mask

            def clear_and_keep(fid, _orig=orig_clear, _h=holder):
                _h["mask"] = ctx.download(fid, abi.BUF_GOODMASK)
                return _orig(fid)
            ctx.clear_good_mask = clear_and_keep
            try:
                gs.step(k, images[k])
            finally:
                ctx.clear_good_mask = orig_clear
            out = replay.replay_step(seq_small, snap, k, images[k], gs)
            reps.append(replay.finish_replay(seq_small, snap, out, gs, mask_before_clear=holder.get("mask")))
            if k == change_at:
                out = replay.replay_step(seq_small, snap, k, images[k], gs, globals_kw=_defaults())
                stale = replay.finish_replay(seq_small, snap, out, gs, mask_before_clear=holder.get("mask"))
    finally:
        ctx.close()
        oracle.set_globals()
    for r in reps:
        assert _same_globals(r["globals"], COMBINED if r["frame"] >= change_at else {})
        _assert_step_ok(r)
    assert any(r["kf_change"] for r in reps)
    assert not stale["map_ok"], stale["map"]


def test_group_with_different_settings_equals_single_calls():
    """two contexts on the same frames, one at the defaults and one at the combined set, in one lsdgpu_track_and_map_group call
    per frame == two single lsdgpu_track_and_map calls, bit for bit; the two streams' results differ"""
    seq = synth.Sequence(320, 240, seed=1234)
    frames = [seq.render(k) for k in range(13)]
    settings = [{}, COMBINED]

    def run(grouped):
        streams = []
        for s, g in enumerate(settings):
            gs = GpuStream(abi.Context(seq.w, seq.h, seq.K, max_frames=8, **g), mode=1, kf_every=10, kf_phase=2 * s)
            gs.init_gt(0, frames[0][0], frames[0][1])
            streams.append(gs)
        group = GpuStreamGroup(streams)
        log = []
        try:
            for k in range(1, 13):
                kf = [gs.next_is_keyframe_change() for gs in streams]
                if grouped:
                    group.step([k, k], images=[frames[k][0]] * 2)
                    qts = [group._qts[i].copy() if kf[i] else None for i in range(2)]
                else:
                    for gs in streams:
                        gs.step(k, frames[k][0])
                    qts = [gs._qts.copy() if kf[i] else None for i, gs in enumerate(streams)]
                log.append([dict(_observe(gs, k, q), kf=kf[i]) for i, (gs, q) in enumerate(zip(streams, qts))])
        finally:
            for gs in streams:
                gs.ctx.close()
        return log
    single, group = run(False), run(True)
    assert [[s for s in range(2) if step[s]["kf"]] for step in single].count([]) == 10       # one keyframe change per stream
    _assert_same(group, single)
    for key in ("result", "depth"):
        assert all(step[0][key] != step[1][key] for step in single), key
    for key in ("pose", "mask"):
        assert any(step[0][key] != step[1][key] for step in single), key
