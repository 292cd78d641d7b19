"""Minimized frames (lsdgpu_frame_minimize / lsdgpu_frame_activate, Frame::minimizeInMemory and FrameMemory::activateFrame,
DataStructures/Frame.cpp:377-395 and FrameMemory.cpp:129-137).  Every comparison is byte for byte against the same calls on a
context that never minimizes; the other suites pin that context to the reference."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi
from lsd_slam_b200.stream import GpuStream, sim3_mul_qts

pytestmark = pytest.mark.gpu

LEVELS = 5


def _sim3_inv(a):
    qi = np.array([-a[0], -a[1], -a[2], a[3]])
    s = 1.0 / a[7]
    u = np.cross(qi[:3], -a[4:7])
    u = u + u
    t = -a[4:7] + qi[3] * u + np.cross(qi[:3], u)
    return np.concatenate([qi, s * t, [s]])


def _snapshot(ctx, fid):
    """every buffer lsdgpu_frame_download serves, at every level, and the frame's host-side state"""
    snap = {}
    has_depth = True
    for lvl in range(LEVELS):
        snap[("image", lvl)] = ctx.download(fid, abi.BUF_IMAGE, lvl).tobytes()
        snap[("grad", lvl)] = ctx.download(fid, abi.BUF_GRADIENTS, lvl).tobytes()
        try:
            snap[("idepth", lvl)] = ctx.download(fid, abi.BUF_IDEPTH, lvl).tobytes()
            snap[("idepthVar", lvl)] = ctx.download(fid, abi.BUF_IDEPTH_VAR, lvl).tobytes()
        except abi.LsdGpuError:
            has_depth = False
    snap["maxgrad"] = ctx.download(fid, abi.BUF_MAXGRAD, 0).tobytes()
    snap.update(_host_state(ctx, fid))
    return snap, has_depth


def _host_state(ctx, fid):
    q, pid, itr = ctx.get_pose(fid)
    s = {"pose": (np.asarray(q).tobytes(), pid, np.float32(itr).tobytes()), "counters": ctx.get_counters(fid),
         "stats": ctx.depth_stats(fid)}
    try:
        s["react"] = tuple(a.tobytes() for a in ctx.reactivation_data(fid))
    except abi.LsdGpuError:
        s["react"] = None
    return s


def _goodmask(ctx, fid):
    return ctx.download(fid, abi.BUF_GOODMASK, 1)


def _stream(seq, n, kf_every, max_frames, first_id=0, **kw):
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=max_frames)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every, keep_keyframes=True, **kw)
    img, d = seq.render(0)
    gs.init_gt(first_id, img, d)
    for k in range(1, n):
        gs.step(first_id + k, seq.render(k)[0])
    return gs


PERMA_POSE = np.array([0, 0, 0, 1, 0.01, -0.005, 0.002], np.float64)


def _buffers(ctx, fid, with_perma):
    """_snapshot plus, for a frame with a permaRef, the permaRef overlap at a fixed pose (reads the permaRef buffers)"""
    snap, has_depth = _snapshot(ctx, fid)
    if with_perma:
        snap["perma"] = abi.SE3Tracker(ctx).checkPermaRefOverlap([fid], PERMA_POSE[None]).tobytes()
    return snap, has_depth


def _dirty_free_slots(ctx, before, other_img, other_depth, with_perma):
    """Fills every free slot with another keyframe -- its image, gradients, maxGradients, idepth pyramid, reactivation data,
    permaRef and setDepth statistics all differ from the minimized frame's -- and frees the slots again, so that whichever slot
    the frame is activated into holds none of its old contents: activation has to rebuild and restore everything."""
    dm, trk = abi.DepthMap(ctx), abi.SE3Tracker(ctx)
    ids = []
    while True:
        d = 900 + len(ids)
        try:
            ctx.upload(d, other_img)
        except abi.LsdGpuError as e:
            assert "no free frame slot" in str(e)
            break
        ids.append(d)
    assert ids
    for d in ids:
        ctx.set_depth_gt(d, other_depth)
        dm.initializeFromGTDepth(d)
        ctx.take_reactivation_data(d)
        trk.setPermaRef(d)
        snap, _ = _buffers(ctx, d, with_perma)
        for k, v in before.items():
            if isinstance(k, tuple) or k in ("maxgrad", "perma") or (k == "react" and v is not None):
                assert snap[k] != v, (d, k)
    dm.invalidate()
    for d in ids:
        ctx.release(d)


def _round_trip(ctx, fid, other, expect_mask_cleared=False, with_perma=False):
    before, has_depth = _buffers(ctx, fid, with_perma)
    mask_before = _goodmask(ctx, fid)
    n0 = ctx.launch_count()
    ctx.minimize(fid)
    assert ctx.launch_count() - n0 == 1
    ctx.minimize(fid)                                   # already minimized: nothing
    assert ctx.launch_count() - n0 == 1
    # in place on the record
    assert _host_state(ctx, fid) == {k: before[k] for k in ("pose", "counters", "stats", "react")}
    assert ctx.download(fid, abi.BUF_IMAGE, 0).tobytes() == before[("image", 0)]
    if has_depth:
        assert ctx.download(fid, abi.BUF_IDEPTH, 0).tobytes() == before[("idepth", 0)]
        assert ctx.download(fid, abi.BUF_IDEPTH_VAR, 0).tobytes() == before[("idepthVar", 0)]
    _dirty_free_slots(ctx, before, *other, with_perma)
    n1 = ctx.launch_count()
    ctx.activate(fid)
    assert ctx.launch_count() - n1 == 3                 # unpack, image pyramid, gradients
    n2 = ctx.launch_count()
    ctx.activate(fid)                                   # already active: nothing
    assert ctx.launch_count() == n2
    after, has_depth_after = _buffers(ctx, fid, with_perma)
    assert has_depth_after == has_depth
    assert after.keys() == before.keys()
    for k in before:
        assert after[k] == before[k], k
    assert (_goodmask(ctx, fid) == 1).all()             # clear_refPixelWasGood, Frame.cpp:388
    if expect_mask_cleared:
        assert not (mask_before == 1).all()


def test_round_trip_mapped_keyframe(seq_small, frames_small):
    """a GT-initialised keyframe mapped over 10 frames, finalized (reactivation data) and with a permaRef"""
    gs = _stream(seq_small, 12, 10, 8)
    ctx = gs.ctx
    assert gs.kf_id == 10
    assert gs.tracker.setPermaRef(0) > 0
    assert _host_state(ctx, 0)["react"] is not None
    _round_trip(ctx, 0, frames_small[7], with_perma=True)
    ctx.close()


@pytest.mark.parametrize("model", ["ptam", "opencv"])
def test_round_trip_undistorted_keyframe(seq_small, frames_small, model):
    size = (seq_small.w, seq_small.h)
    if model == "ptam":
        u = abi.UndistorterPTAM([0.535719308086809, 0.669566858850269, 0.493248545285398, 0.500408664348414, 0.897966326944875],
                                size, "crop", size)
    else:       # the TUM fr1 calibration at half resolution
        u = abi.UndistorterOpenCV([258.65, 258.25, 159.3, 127.65, 0.2624, -0.9531, -0.0054, 0.0026], size, "crop", size)
        assert u.status == 0
    ctx = abi.Context(seq_small.w, seq_small.h, u.getK(), max_frames=4)
    u.install(ctx)
    ctx.upload_distorted(3, frames_small[0][0])
    ctx.set_depth_gt(3, frames_small[0][1])
    ctx.set_pose(3, [0.1, 0.2, 0.3, 0.9, 1, 2, 3, 1.5], 7, 0.25)
    ctx.set_counters(3, 4, 5)
    _round_trip(ctx, 3, frames_small[7])
    ctx.close()


def test_round_trip_tracked_frame(seq_small, frames_small):
    """a plain frame from the prefetch ring, tracked (so it has a good mask), never mapped"""
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=4)
    ctx.upload(0, frames_small[0][0])
    ctx.set_depth_gt(0, frames_small[0][1])
    abi.DepthMap(ctx).initializeFromGTDepth(0)
    ctx.stage_reserve(1)
    ctx.stage_put(0, frames_small[2][0])
    ctx.frame_from_stage(2, 0)
    trk = abi.SE3Tracker(ctx)
    trk.importFrame(0)
    trk.trackFrame(0, 2, np.array([0, 0, 0, 1, 0, 0, 0], np.float64))
    assert not trk.diverged
    _round_trip(ctx, 2, frames_small[7], expect_mask_cleared=True)
    ctx.close()


def test_in_place_perma_and_cloud(seq_small, frames_small):
    """the permaRef batches and the cloud export over a mix of minimized and active keyframes equal the all-active calls"""
    gs = _stream(seq_small, 22, 6, 12)
    ctx, trk = gs.ctx, gs.tracker
    kfs = gs.keyframe_ids
    assert len(kfs) >= 4
    finished = kfs[:-1]
    for k in finished:
        trk.setPermaRef(k)
    ctx.upload(200, frames_small[5][0])
    rng = np.random.default_rng(5)
    qts = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], np.float64), (len(finished), 1))
    qts[:, 4:7] = rng.normal(0, 0.01, (len(finished), 3))
    c2w = gs.keyframe_cam_to_world_f7()
    ctx.cloud_reserve(3)

    def run():
        usage = trk.checkPermaRefOverlap(finished, qts).tobytes()
        track = [bytes(r) for r in trk.trackFrameOnPermaref(finished, 200, qts)]
        clouds = [tuple(a.tobytes() for a in ctx.export_pointcloud(kfs, c2w, level=0, layout=lay)) for lay in (abi.CLOUD_PLY, abi.CLOUD_VERTEX)]
        return usage, track, clouds

    want = run()
    for k in finished[::2]:
        ctx.minimize(k)
    assert run() == want
    with pytest.raises(abi.LsdGpuError, match=f"{finished[0]}.*minimized"):
        ctx.export_pointcloud(kfs, c2w, level=1)
    ctx.close()


def _continued(seq, minimize):
    n, kf_every = 70, 10
    gs = _stream(seq, n, kf_every, 6 if minimize else 16, **({"max_active_keyframes": 0} if minimize else {}))
    ctx = gs.ctx
    assert len(gs.keyframe_ids) == 7
    if minimize:                                        # more keyframes than frame slots: the six finished ones are minimized
        for k in gs.keyframe_ids[:-1]:
            with pytest.raises(abi.LsdGpuError, match=f"frame {k} is minimized"):
                ctx.download(k, abi.BUF_GRADIENTS, 0)
    # re-activate keyframe 10 and map 5 more frames on it (DepthMap::setFromExistingKF, DepthMap.cpp:920-962)
    ctx.activate(10)
    ctx._ck(ctx.L.lsdgpu_depth_set_from_existing_kf(ctx.ptr, 10))
    gs.kf_id, gs.kf_every, gs.last_pose = 10, 0, np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    for i in range(5):
        gs.step(100 + i, seq.render(11 + i)[0])
    results = [bytes(gs.tracker.last)]
    # Sim3 between re-activated keyframes
    for k in (20, 30):
        ctx.activate(k)
    c2w = dict(zip(gs.keyframe_ids, gs.keyframe_cam_to_world))
    pairs = [(10, 20), (20, 10), (20, 30), (30, 20)]
    inits = np.stack([sim3_mul_qts(_sim3_inv(c2w[r]), c2w[f]) for r, f in pairs])
    s3 = abi.Sim3Tracker(ctx)
    sim3 = [bytes(r) for r in s3.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)]
    poses = [(np.asarray(q).tobytes(), pid, itr) for q, pid, itr in (ctx.get_pose(k) for k in gs.keyframe_ids + [100 + 4])]
    ctx.cloud_reserve(4)
    cloud = ctx.export_pointcloud(gs.keyframe_ids, gs.keyframe_cam_to_world_f7(), level=0)
    out = {"poses": np.array(gs.poses).tobytes(), "results": results, "frame_poses": poses,
           "depth": abi.DepthMap(ctx).current().tobytes(), "sim3": sim3, "cloud": tuple(a.tobytes() for a in cloud)}
    ctx.close()
    return out


def test_continued_operation_matches_resident_run(seq_small):
    a = _continued(seq_small, False)
    b = _continued(seq_small, True)
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], k


def test_refusals(seq_small, frames_small):
    gs = _stream(seq_small, 12, 10, 4, first_id=37)
    ctx, L, p = gs.ctx, gs.ctx.L, gs.ctx.ptr
    assert gs.kf_id == 47
    gs.tracker.setPermaRef(37)
    ctx.minimize(37)
    dm = abi.DepthMap(ctx)
    depth0 = dm.current().tobytes()
    state0 = _host_state(ctx, 37)
    img = np.ascontiguousarray(frames_small[1][0])
    u8 = img.ctypes.data_as(C.POINTER(C.c_uint8))
    f32 = np.zeros(seq_small.w * seq_small.h * 8, np.float32)
    fp = f32.ctypes.data_as(C.POINTER(C.c_float))
    qt = np.array([0, 0, 0, 1, 0, 0, 0, 1], np.float64)
    dp = qt.ctypes.data_as(C.POINTER(C.c_double))
    one = (C.c_int * 1)(37)
    res = abi.TrackResult()
    s3res = abi.Sim3Result()
    ev = abi.EvalResult()
    s3ev = abi.Sim3EvalResult()
    hyp = (abi.Hyp * (seq_small.w * seq_small.h))()
    pts = np.zeros(seq_small.w * seq_small.h, abi.CLOUD_PLY_DTYPE)
    npts = C.c_int64()
    flt = abi.default_cloud_filter()
    ctx.stage_reserve(1)
    ctx.stage_put(0, img)
    ctx.cloud_reserve(2)
    other = 48                                             # the last tracked frame, in a slot
    step = abi.GroupStep()
    step.ctx, step.kf_id, step.frame_id, step.gray, step.stage_index = p, 47, 37, u8, -1
    step.frameToRef_init_qt[:] = [0, 0, 0, 1, 0, 0, 0]
    calls = {
        "se3_track kf": lambda: L.lsdgpu_se3_track(p, 37, other, dp, None, 1, C.byref(res)),
        "se3_track frame": lambda: L.lsdgpu_se3_track(p, 47, 37, dp, None, 1, C.byref(res)),
        "se3_eval": lambda: L.lsdgpu_se3_eval(p, 37, other, 1, fp, 1.0, 0.0, None, 0, C.byref(ev)),
        "sim3_track_batch": lambda: L.lsdgpu_sim3_track_batch(p, 1, one, (C.c_int * 1)(47), dp, 4, 1, None, C.byref(s3res)),
        "sim3_eval": lambda: L.lsdgpu_sim3_eval(p, 47, 37, 2, dp, 1.0, 0.0, None, C.byref(s3ev)),
        "ref_import": lambda: L.lsdgpu_ref_import(p, 37),
        "set_perma_ref": lambda: L.lsdgpu_frame_set_perma_ref(p, 37, None),
        "perma_track frame": lambda: L.lsdgpu_perma_track_batch(p, 1, (C.c_int * 1)(37), 37, dp, C.byref(res)),
        "init_from_gt": lambda: L.lsdgpu_depth_init_from_gt(p, 37),
        "set_hypotheses": lambda: L.lsdgpu_depth_set_hypotheses(p, 37, hyp, 1, 1),
        "set_from_existing_kf": lambda: L.lsdgpu_depth_set_from_existing_kf(p, 37),
        "update_keyframe": lambda: L.lsdgpu_depth_update_keyframe(p, one, 1),
        "observe": lambda: L.lsdgpu_depth_observe(p, one, 1),
        "propagate": lambda: L.lsdgpu_depth_propagate(p, 37),
        "create_keyframe": lambda: L.lsdgpu_depth_create_keyframe(p, 37, dp),
        "take_reactivation": lambda: L.lsdgpu_frame_take_reactivation_data(p, 37),
        "pack_pointcloud": lambda: L.lsdgpu_keyframe_pack_pointcloud(p, 37, 0, pts.ctypes.data_as(C.c_void_p)),
        "cloud level 1": lambda: L.lsdgpu_map_export_pointcloud(p, 1, one, f32[:7].ctypes.data_as(C.POINTER(C.c_float)), 1,
                                                                C.byref(flt), 0, pts.ctypes.data_as(C.c_void_p), len(pts), C.byref(npts), None),
        "download gradients": lambda: L.lsdgpu_frame_download(p, 37, abi.BUF_GRADIENTS, 0, f32.ctypes.data_as(C.c_void_p)),
        "download image level 1": lambda: L.lsdgpu_frame_download(p, 37, abi.BUF_IMAGE, 1, f32.ctypes.data_as(C.c_void_p)),
        "download maxgrad": lambda: L.lsdgpu_frame_download(p, 37, abi.BUF_MAXGRAD, 0, f32.ctypes.data_as(C.c_void_p)),
        "download goodmask": lambda: L.lsdgpu_frame_download(p, 37, abi.BUF_GOODMASK, 1, f32.ctypes.data_as(C.c_void_p)),
        "set_depth_gt": lambda: L.lsdgpu_frame_set_depth_gt(p, 37, fp, 1.0),
        "set_idepth": lambda: L.lsdgpu_frame_set_idepth(p, 37, fp, fp),
        "clear_good_mask": lambda: L.lsdgpu_frame_clear_good_mask(p, 37),
        "upload": lambda: L.lsdgpu_frame_upload_u8(p, 37, u8),
        "frame_from_stage": lambda: L.lsdgpu_frame_from_stage(p, 37, 0),
        "track_and_map kf": lambda: L.lsdgpu_track_and_map(p, 37, 50, u8, -1, dp, None, 1, 0, C.byref(res), dp),
        "track_and_map frame": lambda: L.lsdgpu_track_and_map(p, 47, 37, u8, -1, dp, None, 1, 0, C.byref(res), dp),
        "group step": lambda: L.lsdgpu_track_and_map_group(1, C.byref(step), C.byref(res), None),
    }
    for name, call in calls.items():
        launches = ctx.launch_count()
        assert call() != 0, name
        msg = L.lsdgpu_last_error(p).decode()
        assert re.search(r"\b37\b", msg) and "minimized" in msg, (name, msg)
        assert ctx.launch_count() == launches, name
        assert _host_state(ctx, 37) == state0, name
        assert L.lsdgpu_frame_get_pose(p, 50, None, None, None) != 0, name          # no frame was built
    assert dm.current().tobytes() == depth0
    assert dm.activeKeyFrame() == 47
    # the active keyframe cannot be minimized
    with pytest.raises(abi.LsdGpuError, match="active keyframe"):
        ctx.minimize(47)
    assert ctx.download(47, abi.BUF_GRADIENTS, 2).size
    # no free slot: the frame stays minimized
    ctx.upload(60, frames_small[2][0])
    ctx.upload(61, frames_small[3][0])
    with pytest.raises(abi.LsdGpuError, match="no free frame slot to activate frame 37"):
        ctx.activate(37)
    assert _host_state(ctx, 37) == state0
    assert ctx.download(37, abi.BUF_IMAGE, 0).size
    with pytest.raises(abi.LsdGpuError, match="minimized"):
        ctx.download(37, abi.BUF_IMAGE, 1)
    assert dm.current().tobytes() == depth0
    # activate after a release: the frame is gone
    ctx.release(37)
    ctx.release(61)
    with pytest.raises(abi.LsdGpuError, match="unknown frame id"):
        ctx.activate(37)
    with pytest.raises(abi.LsdGpuError, match="unknown frame id"):
        ctx.get_pose(37)
    ctx.close()


def test_host_demo_prune_matches_python_loop(tmp_path, seq_small, frames_small):
    """host_demo with 4 frame slots, every keyframe kept and FrameMemory::pruneActiveFrames after each keyframe change
    reproduces the Python loop's poses"""
    from lsd_slam_b200 import build
    build.build_host()
    n, kf_every = 16, 3
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        np.array([seq_small.w, seq_small.h, n], np.int32).tofile(f)
        seq_small.K.astype(np.float32).tofile(f)
        frames_small[0][1].astype(np.float32).tofile(f)
        for k in range(n):
            frames_small[k][0].tofile(f)
    r = subprocess.run([build.DEMO_OUT, str(path), str(kf_every), "prune", "4", "2"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    rows = np.array([[float(x) for x in ln.split()] for ln in r.stdout.strip().splitlines()])
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=8)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every)
    gs.init_gt(0, frames_small[0][0], frames_small[0][1])
    for k in range(1, n):
        gs.step(k, frames_small[k][0])
    py = np.array(gs.poses)
    assert rows.shape[0] == n - 1
    assert np.allclose(rows[:, 1:8], py, atol=1e-9), np.abs(rows[:, 1:8] - py).max()
    ctx.close()
