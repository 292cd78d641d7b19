"""GPU parity at the reference's NON-DEFAULT run-time settings (util/settings.cpp:80-88, changed between frames by ROS dynamic
reconfigure: cfg/LSDParams.cfg:13-34, IOWrapper/ROS/rosReconfigure.h:81-91).  Every other parity test runs at the defaults, so a
kernel that hard-codes a default, compares a threshold with the wrong operator, or reads a setting from the wrong context would pass
there.  Here the context (abi.Context(..., **g)) and the oracle (oracle.set_globals(**g)) run under the same settings -- the
oracle is pinned to the reference-compiled library at each of them by tests/test_ref_pin_globals.py:
  * the depth map, pass by pass and through updateKeyframe / finalizeKeyFrame + createKeyFrame / update_keyframe_refs: bit for bit;
  * SE3 evaluation and tracking (both modes), Sim3 evaluation and batch tracking, permaRef batch tracking: the tolerances of
    tests/util.py's checks, identical LM call counters;
  * a closed track + map loop replayed step by step (oracle/replay.py follows the context's settings), a change of settings
    between two steps, and two contexts with different settings in one group call."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from oracle import replay
from tests import device_cases as cases
from tests.pin_cases import SETS
from tests.util import assert_same, assert_step_ok, kf_depth_equal, observe, under

pytestmark = pytest.mark.gpu

G = {name: g for name, (g, _) in SETS.items()}
COMBINED = G["combined"]
DEPTH_SETS = [s for s in G if s != "useAffineLightningEstimation=0"]          # that one is read by the trackers only
TRACK_SETS = [s for s in G if s.startswith(("cameraPixelNoise2", "useAffine", "minUseGrad")) or s == "combined"]
MIN_USE_GRAD_SETS = [s for s in G if "minUseGrad" in G[s]]


@pytest.fixture(params=DEPTH_SETS)
def depth_ctx(request, oracle, seq_small):
    with under(oracle, G[request.param], seq_small.w, seq_small.h, seq_small.K) as ctx:
        yield ctx


@pytest.fixture(params=TRACK_SETS)
def track_ctx(request, oracle, seq_small):
    with under(oracle, G[request.param], seq_small.w, seq_small.h, seq_small.K) as ctx:
        yield ctx


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def test_observe_from_gt_depth_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    cases.observe_from_gt(depth_ctx, oracle, seq_small, frames_small)


def test_random_init_observe_and_update_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    cases.random_init_observe_and_update(depth_ctx, oracle, seq_small, frames_small)


def test_fill_holes_regularize_and_integral_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    cases.fill_holes_and_regularize(depth_ctx, oracle, seq_small, frames_small)


def test_update_keyframe_sequence_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    cases.update_keyframe_sequence(depth_ctx, oracle, seq_small, frames_small)


def test_finalize_create_keyframe_and_refs_bit_exact(depth_ctx, oracle, seq_small, frames_small):
    cases.finalize_create_and_refs(depth_ctx, oracle, seq_small, frames_small)


@pytest.mark.parametrize("set_name", MIN_USE_GRAD_SETS)
def test_set_depth_gt_pyramids(oracle, seq_small, frames_small, set_name):
    """Frame::setDepthFromGroundTruth keeps a pixel iff its gradient passes minUseGrad (Frame.cpp)"""
    img0, d0 = frames_small[0]
    with under(oracle, G[set_name], seq_small.w, seq_small.h, seq_small.K, max_frames=4) as ctx:
        ctx.upload(0, img0)
        ctx.set_depth_gt(0, d0)
        okf = oracle.Frame(0, img0, seq_small.K)
        okf.setDepthFromGroundTruth(d0)
        kf_depth_equal(ctx, okf, 0)
        assert (okf.idepth(0) > 0).sum() > 1000


# ---- trackers ---------------------------------------------------------------------------------------------------------------
def test_se3_eval_each_level(track_ctx, oracle, seq_small, frames_small):
    cases.se3_eval_each_level(track_ctx, oracle, seq_small, frames_small, sum_noise=True)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 8])
def test_se3_track(track_ctx, oracle, seq_small, frames_small, mode, k):
    cases.se3_track(track_ctx, oracle, seq_small, frames_small, mode, k)


@pytest.mark.parametrize("set_name", TRACK_SETS)
def test_sim3_eval_and_track_batch(oracle, set_name):
    seq = synth.Sequence(640, 480, seed=1234)
    with under(oracle, G[set_name], 640, 480, seq.K, max_frames=8) as ctx:
        of = cases.gt_keyframes(ctx, oracle, seq)
        trk = abi.Sim3Tracker(ctx)
        cases.sim3_eval(trk, oracle, seq, of)
        cases.sim3_batch(trk, oracle, seq, of, exact_twin=True)


@pytest.mark.parametrize("set_name", TRACK_SETS)
def test_perma_track_batch(oracle, set_name):
    seq = synth.Sequence(640, 480, seed=1234)
    with under(oracle, G[set_name], 640, 480, seq.K, max_frames=8) as ctx:
        trk, prs = cases.perma_setup(ctx, oracle, seq, (0, 6, 12), 200)
        assert cases.perma_batch(ctx, oracle, seq, trk, prs, 9) >= 1


# ---- closed loop, mid-run change, group -------------------------------------------------------------------------------------
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
        assert_step_ok(r)
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
        assert_step_ok(r)
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
                log.append([dict(observe(gs, k, q), kf=kf[i]) for i, (gs, q) in enumerate(zip(streams, qts))])
        finally:
            for gs in streams:
                gs.ctx.close()
        return log
    single, group = run(False), run(True)
    assert [[s for s in range(2) if step[s]["kf"]] for step in single].count([]) == 10       # one keyframe change per stream
    assert_same(group, single)
    for key in ("result", "depth"):
        assert all(step[0][key] != step[1][key] for step in single), key
    for key in ("pose", "mask"):
        assert any(step[0][key] != step[1][key] for step in single), key
