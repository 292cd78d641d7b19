"""GPU parity through cameras other than synth.pinhole_K (tests/cameras.py: aspect, offset, general at 320x240, euroc640).

Every other device test runs a camera with fx == fy and the principal point at the image centre, where a kernel that reads fx for
fy, fxi for fyi or cx for cy, and a host that builds the level intrinsics in the wrong precision, give the same bits.  Here the
device is checked through each camera against the oracle -- which tests/test_ref_pin_cameras.py pins to the reference-compiled
library through the same cameras -- and against the reference's recorded values:
  * the frame builders and the ground-truth idepth pyramids: bit for bit;
  * the depth-map scenarios of tests/test_gpu_motions.py (tests/device_cases.py): bit for bit, and four of them through `general`
    under the vertical motion, which runs the y-dominant depth formula;
  * SE3 evaluation on levels 4-1 and trackFrame in modes 0 and 1: the tolerances of tests/util.py;
  * Sim3 evaluation, trackFrameSim3 (one by one and batched), permaRef overlap and trackFrameOnPermaref on keyframes the
    device's mapper finished, against the oracle; for `general` also on the pin's mapped keyframes against the recorded
    reference values;
  * the map's point-cloud export (host and device output) against the viewer oracle with the level intrinsics of the pinned
    Frame::K(level), and the keyframeMsg packing against the oracle;
  * replayed closed loops of 25 steps with two keyframe changes: `general` at 320x240, euroc640 at 640x480;
  * one group call over three streams with different cameras: equal to the single calls bit for bit, one stream replayed."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from lsd_slam_b200.stream import GpuStream
from oracle import replay
from tests import cameras
from tests import device_cases as cases
from tests import pin_cases as pin
from tests.util import (CLOUD_FILTERS, _level_cam, assert_same, assert_step_ok, check_perma_track, check_sim3_eval,
                        check_sim3_track, kf_depth_equal, oracle_cloud, oracle_sim3_track, perma_noise, same_cloud)

pytestmark = pytest.mark.gpu

SMALL = list(cameras.SMALL)


@pytest.fixture(params=SMALL)
def camera(request):
    return request.param


@pytest.fixture()
def stream(camera):
    """(320x240 sequence, lazily rendered frames) of the camera, shared with the pin"""
    return cameras.stream(camera)


@pytest.fixture()
def ctx(oracle, stream):
    seq, _ = stream
    c = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    yield c
    c.close()
    oracle.set_globals()


# ---- frames, bit for bit ----------------------------------------------------------------------------------------------------
def test_frame_builders_and_idepth_pyramids_bit_exact(ctx, oracle, stream):
    seq, frames = stream
    img, d = frames[0]
    ctx.upload(0, img)
    ctx.set_depth_gt(0, d)
    of = oracle.Frame(0, img, seq.K)
    of.setDepthFromGroundTruth(d)
    for lvl in range(5):
        assert np.array_equal(ctx.download(0, abi.BUF_IMAGE, lvl), of.image(lvl)), lvl
        assert np.array_equal(ctx.download(0, abi.BUF_GRADIENTS, lvl), of.gradients(lvl)), lvl
    assert np.array_equal(ctx.download(0, abi.BUF_MAXGRAD, 0), of.maxGradients(0))
    kf_depth_equal(ctx, of, 0)


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def test_observe_from_gt_depth_bit_exact(ctx, oracle, stream):
    cases.observe_from_gt(ctx, oracle, *stream)


def test_random_init_observe_and_update_bit_exact(ctx, oracle, stream):
    cases.random_init_observe_and_update(ctx, oracle, *stream)


def test_fill_holes_and_regularize_on_the_observed_map_bit_exact(ctx, oracle, stream):
    cases.fill_holes_and_regularize_observed(ctx, oracle, *stream)


def test_update_keyframe_sequence_bit_exact(ctx, oracle, stream):
    cases.update_keyframe_sequence(ctx, oracle, *stream)


def test_propagate_and_create_keyframe_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe(ctx, oracle, *stream, False)


def test_propagate_and_create_keyframe_with_tracking_mask_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe_device_mask(ctx, oracle, *stream)


def test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, stream):
    cases.finalize_create_and_refs(ctx, oracle, *stream)


@pytest.mark.parametrize("scenario", ["observe_from_gt", "random_init_observe_and_update", "update_keyframe_sequence",
                                      "finalize_create_and_refs"])
def test_vertical_motion_depth_map_bit_exact(oracle, scenario):
    """`general` under the vertical motion: the y-dominant depth formula of the line stereo (alpha and oldY through fyi)"""
    seq, frames = cameras.stream(cameras.VERTICAL)
    c = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    try:
        getattr(cases, scenario)(c, oracle, seq, frames)
    finally:
        c.close()
        oracle.set_globals()


# ---- SE3 tracker --------------------------------------------------------------------------------------------------------------
def test_se3_eval_each_level(ctx, oracle, stream):
    cases.se3_eval_each_level(ctx, oracle, *stream, sum_noise=True)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 8])
def test_se3_track(ctx, oracle, stream, mode, k):
    cases.se3_track(ctx, oracle, *stream, mode, k)


# ---- Sim3 and permaRef on keyframes the device's mapper finished --------------------------------------------------------------
@pytest.fixture(scope="module", params=SMALL)
def mapped(request, oracle):
    run = cases.MappedRun(oracle, 320, 240, request.param, seq=cameras.stream(request.param)[0])
    yield run
    run.close()


def test_mapped_keyframes_mirror_bit_exact(mapped):
    cases.mapped_mirror_bit_exact(mapped)


def test_sim3_eval_on_mapped_keyframes(mapped, oracle):
    cases.mapped_sim3_eval(mapped, oracle)


def test_track_frame_sim3_on_mapped_keyframes(mapped, oracle):
    """to POSE_TOL of the oracle's all-sums-exact twin, and of the reference arithmetic plus its own distance to that twin:
    through `offset`, 10 -> 5 over levels 4..1, the reference's fp32 sums of the normal equations alone move its translation by
    1.17e-4 (relative), and the device lies 6.6e-6 from the twin (DESIGN.md section 5, Cameras)"""
    cases.mapped_sim3_track(mapped, oracle, sum_noise=True)


def test_track_frame_sim3_batch_on_mapped_keyframes(mapped, oracle):
    cases.mapped_sim3_batch(mapped, oracle, sum_noise=True)


def test_perma_ref_on_mapped_keyframes(mapped, oracle):
    cases.mapped_perma(mapped, oracle, noise_aware=True)


# ---- Sim3 and permaRef on the pin's mapped keyframes, against the reference's recorded values (`general`) --------------------
_gold = None


def _g(key):
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_CAMERAS)
    return _gold[f"general/{key}"]


@pytest.fixture(scope="module")
def loaded(oracle):
    """the C restatement's Mapped run through `general` with its finished keyframes loaded on a device context"""
    seq, frames = cameras.stream("general")
    oracle.set_globals()
    m = pin.mapped(False, seq, frames)
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    dm = abi.DepthMap(ctx)
    for k, f in m.of.items():
        ctx.upload(k, frames[k][0])
        dm.setHypotheses(k, cases.hyp_of_planes(oracle, f.idepth(0), f.idepthVar(0)), do_set_depth=True)
    yield m, ctx
    ctx.close()


def test_sim3_on_pinned_keyframes_against_reference(loaded, oracle):
    m, ctx = loaded
    for k, f in m.of.items():
        kf_depth_equal(ctx, f, k)
    trk = abi.Sim3Tracker(ctx)
    for ref, fr in m.pairs():
        for perturb in (True, False):
            r2f = m.ref_to_frame(ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in pin.AB:
                    want = pin.sim3_eval_result(_g(f"sim3_eval_mapped/{ref}->{fr}/p{int(perturb)}/L{lvl}/a{a}"))
                    check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), want)
    inits = {(ref, fr): m.frame_to_ref(ref, fr) for ref, fr in m.pairs()}
    batch = trk.trackFrameSim3Batch([p[0] for p in inits], [p[1] for p in inits], np.array(list(inits.values())), 4, 1)
    for ((ref, fr), init), r in zip(inits.items(), batch):
        for lo, hi in ((4, 1), (3, 2)):
            trk.trackFrameSim3(ref, fr, init, lo, hi)
            assert not trk.diverged
            if (lo, hi) == (4, 1):
                assert bytes(trk.last) == bytes(r)
            want, exact = oracle_sim3_track(oracle, m.of[ref], m.of[fr], init, lo, hi)
            check_sim3_track(trk.last, pin.sim3_track_result(_g(f"sim3_track_mapped/{ref}->{fr}/{lo}{hi}"), want))
            check_sim3_track(trk.last, exact, res_tol=5e-4)


def test_perma_ref_on_pinned_keyframes_against_reference(loaded, oracle):
    m, ctx = loaded
    se3 = abi.SE3Tracker(ctx)
    prs = {k: oracle.PermaRef(f) for k, f in m.of.items()}
    for k, pr in prs.items():
        assert se3.setPermaRef(k) == pr.n
    poses = pin.overlap_poses(prs)
    ids = [k for k in prs for _ in range(6)]
    got = se3.checkPermaRefOverlap(ids, np.array([q for k in prs for q in poses[k] + [pin.perma_gt(m, k, pin.PERMA_FRAME)]]))
    want = np.concatenate([_g(f"perma_mapped/kf{k}/overlap_values") for k in prs])
    assert np.allclose(got, want, rtol=2e-5, atol=1e-6), np.abs(got - want).max()
    img = m.frames[pin.PERMA_FRAME][0]
    ctx.upload(pin.PERMA_FRAME, img)
    of = oracle.Frame(pin.PERMA_FRAME, img, m.seq.K)
    runs = [(k, name, init) for k in prs for name, init in (("gt", pin.perma_gt(m, k, pin.PERMA_FRAME)), ("identity", pin.IDENT))]
    res = se3.trackFrameOnPermaref([k for k, _, _ in runs], pin.PERMA_FRAME, np.array([init for _, _, init in runs]))
    n_good = 0
    for (k, name, init), g in zip(runs, res):
        want = pin.perma_track_result(_g(f"perma_mapped/kf{k}/track_{name}"), prs[k].track(of, init))
        n_good += check_perma_track(g, want, perma_noise(oracle, prs[k], of, init))
    ctx.release(pin.PERMA_FRAME)
    assert n_good >= 2


# ---- the map's point cloud ----------------------------------------------------------------------------------------------------
def test_cloud_export_and_packing_match_oracle(ctx, oracle, stream):
    """the keyframes of a 26-frame run (keyframe every 8): the export of every filter, level and layout, into host and into device
    memory, equal to the viewer oracle fed with the level intrinsics of the pinned Frame::K(level); keyframeMsg's packing of the
    active keyframe equal to the oracle's of the same map"""
    import torch
    seq, frames = stream
    gs = GpuStream(ctx, mode=1, kf_every=8, keep_keyframes=True)
    gs.init_gt(0, *frames[0])
    for k in range(1, 26):
        gs.step(k, frames[k][0])
    ids, c2w = gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    assert len(ids) >= 4
    ctx.cloud_reserve(len(ids))
    of = oracle.Frame(0, frames[0][0], seq.K)
    for level in (0, 1):
        K, _ = of.K(level)
        assert _level_cam(ctx, level) == (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])), level
        for layout in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
            for filt in CLOUD_FILTERS:
                pts, counts = ctx.export_pointcloud(ids, c2w, level=level, filter=filt, layout=layout)
                ref, ref_counts = oracle_cloud(ctx, ids, c2w, level, filt, layout)
                assert (counts == ref_counts).all(), (level, layout, filt)
                same_cloud(pts, ref)
                if filt is None:
                    assert len(pts) > 1000
                out = torch.full((max(len(pts), 1), 4), 3.0, dtype=torch.float32, device="cuda")
                dpts, dcounts = ctx.export_pointcloud(ids, c2w, level=level, filter=filt, layout=layout, out=out)
                assert np.array_equal(dcounts, ref_counts)
                same_cloud(dpts.cpu().numpy(), ref)
    kf = gs.kf_id
    okf = oracle.Frame(kf, frames[kf][0], seq.K)
    pin.set_depth(okf, gs.map.current())
    for lvl in (0, 1, 3):
        want = okf.pack_pointcloud(lvl)
        assert ctx.pack_pointcloud(kf, lvl).tobytes() == want.tobytes(), lvl
        assert (want["idepth_var"] > 0).sum() > 50


# ---- closed loops -----------------------------------------------------------------------------------------------------------
def _replayed_loop(seq, frames, sample=None):
    reps = replay.run_with_replay(seq, frames, 26, kf_every=10, sample=sample)
    assert [r["frame"] for r in reps if r["kf_change"]] == [10, 20]
    for r in reps:
        assert_step_ok(r)
    return reps


def test_closed_loop_replay_general(oracle):
    """25 steps, keyframe changes at 10 and 20, every step replayed on the oracle from the device's state"""
    assert len(_replayed_loop(*cameras.stream("general"))) == 25


def test_closed_loop_replay_euroc640(oracle):
    """the K UndistorterOpenCV gives for the EuRoC camera at 640x480, every other step and both keyframe changes replayed"""
    seq = cameras.sequence("euroc640")
    assert len(_replayed_loop(seq, cameras.Frames(seq), sample=set(range(2, 26, 2)))) == 12


# ---- a group call over streams with different cameras --------------------------------------------------------------------------
PHASES = [8, 12, 15]            # keyframe changes at frames 12, 8 and 5
REPLAYED = 2                    # the `general` stream


def test_group_of_different_cameras_equals_single_calls(oracle):
    """aspect, offset and general advanced by one group call per step == three single calls, bit for bit.  The group's `general`
    stream is replayed on the oracle: every step's pose from the device's state before it, and the keyframe change's map bit for
    bit from the device's pose and mask (the other steps' good masks are cleared inside the call)"""
    seqs = [lambda w, h, n=n: cameras.sequence(n) for n in SMALL]
    single = cases.run_streams(320, 240, PHASES, 14, lambda k: False, sequences=seqs)
    seq, frames = cameras.stream(SMALL[REPLAYED])
    images = {k: frames[k][0] for k in range(15)}
    pending, reps = [], []

    def replay_previous(k, streams):
        gs = streams[REPLAYED]
        if pending:
            snap, fid = pending.pop()
            out = replay.replay_step(seq, snap, fid, images[fid], gs)
            reps.append(replay.finish_replay(seq, snap, out, gs))
        snap = replay.Snapshot(gs, images)
        snap.kf_change = gs.next_is_keyframe_change()           # with the stream's keyframe phase
        pending.append((snap, k))

    group = cases.run_streams(320, 240, PHASES, 14, lambda k: True, before_step=replay_previous, sequences=seqs)
    oracle.set_globals()
    assert not any(o["diverged"] for step in single for o in step)
    assert [sum(o["kf"] for o in (step[s] for step in single)) for s in range(3)] == [1, 1, 1]
    assert_same(group, single)
    assert len(reps) == 13 and [r["frame"] for r in reps if r["kf_change"]] == [5]
    for r in reps:
        assert r["pose_rel"] <= 1e-4 + r["ref_noise_rel"], (r["frame"], r["pose_rel"], r["ref_noise_rel"])
        assert r["rot_rad"] <= 1e-6 + r["ref_noise_rot"], (r["frame"], r["rot_rad"])
        assert r["counts_equal"], r["frame"]
        if r["kf_change"]:
            assert r["map_ok"], r["map"]
