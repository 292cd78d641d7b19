"""Frame memory: minimized frames (lsdgpu_frame_minimize / lsdgpu_frame_activate, Frame::minimizeInMemory and
FrameMemory::activateFrame, DataStructures/Frame.cpp:377-395 and FrameMemory.cpp:129-137) and offloaded ones (lsdgpu_frame_offload /
lsdgpu_frame_memory_usage): a minimized frame's record split into a host body in pinned host memory and a device residue, as the
reference keeps minimized frames in host RAM (FrameMemory.cpp:149-166).  The tests that depend on where a record lives run for both
tiers: "device" minimizes only, "host" minimizes and then offloads.  Every comparison is byte for byte against the same calls on a
context, or at a point of the run, that never minimizes; the other suites pin those calls to the reference."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi
from lsd_slam_b200.stream import GpuStream, sim3_mul_qts

LEVELS = 5
W, H = 320, 240
TIERS = ["device", "host"]
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
PERMA_POSE = np.array([0, 0, 0, 1, 0.01, -0.005, 0.002], np.float64)
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s on an H100


def _a256(n):
    return -(-n // 256) * 256


def _layout(has_depth, react, perma_pts):
    """(device residue, host body) bytes of a 320x240 record, each part at a 256-byte boundary (DESIGN.md section 3)"""
    n0 = W * H
    residue = _a256(24) + _a256(16 * perma_pts) + _a256(4 * perma_pts)
    body = _a256(4 * n0) + (2 * _a256(4 * n0) if has_depth else 0) + (2 * _a256(4 * n0) + _a256(n0) if react else 0)
    return residue, body


def _sim3_inv(a):
    qi = np.array([-a[0], -a[1], -a[2], a[3]])
    s = 1.0 / a[7]
    u = np.cross(qi[:3], -a[4:7])
    u = u + u
    t = -a[4:7] + qi[3] * u + np.cross(qi[:3], u)
    return np.concatenate([qi, s * t, [s]])


def _host_state(ctx, fid):
    q, pid, itr = ctx.get_pose(fid)
    s = {"pose": (np.asarray(q).tobytes(), pid, np.float32(itr).tobytes()), "counters": ctx.get_counters(fid),
         "stats": ctx.depth_stats(fid)}
    try:
        s["react"] = tuple(a.tobytes() for a in ctx.reactivation_data(fid))
    except abi.LsdGpuError:
        s["react"] = None
    return s


def _level0(ctx, fid, has_depth):
    whats = (abi.BUF_IMAGE, abi.BUF_IDEPTH, abi.BUF_IDEPTH_VAR) if has_depth else (abi.BUF_IMAGE,)
    return {w: ctx.download(fid, w, 0).tobytes() for w in whats}


def _snapshot(ctx, fid):
    """every plane lsdgpu_frame_download serves at every level, the frame's host-side state and whether it has depth"""
    snap, has_depth = {}, True
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


def _buffers(ctx, fid, with_perma):
    """_snapshot plus, for a frame with a permaRef, the permaRef overlap at a fixed pose (reads the permaRef buffers)"""
    snap, has_depth = _snapshot(ctx, fid)
    if with_perma:
        snap["perma"] = abi.SE3Tracker(ctx).checkPermaRefOverlap([fid], PERMA_POSE[None]).tobytes()
    return snap, has_depth


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


def _probe(ctx, fid, probe_id, probe_img):
    """what the keyframe serves to the next calls: the idepth pyramid after lsdgpu_ref_import and the tracking result of a frame
    on it"""
    trk = abi.SE3Tracker(ctx)
    counters = ctx.get_counters(fid)
    trk.importFrame(fid)
    out = {("ref_idepth", lvl): ctx.download(fid, abi.BUF_IDEPTH, lvl).tobytes() for lvl in range(LEVELS)}
    ctx.upload(probe_id, probe_img)
    trk.trackFrame(fid, probe_id, IDENT)
    out["track"] = bytes(trk.last)
    ctx.release(probe_id)
    ctx.set_counters(fid, *counters)                    # the tracking counted itself on the keyframe
    return out


def _round_trip(ctx, fid, other, tier, perma_pts=0, probe=None, expect_mask_cleared=False):
    """minimizes frame `fid` (and offloads it for the host tier), reads it in place, dirties every free slot and activates it:
    every buffer, the host-side state and what the frame serves to the next calls come back unchanged"""
    before = {} if probe is None else _probe(ctx, fid, *probe)      # clears depthHasBeenUpdatedFlag
    bufs, has_depth = _buffers(ctx, fid, perma_pts > 0)
    before.update(bufs)
    mask_before = _goodmask(ctx, fid)
    residue, body = _layout(has_depth, before["react"] is not None, perma_pts)
    base = ctx.memory_usage()
    n0 = ctx.launch_count()
    ctx.minimize(fid)
    assert ctx.launch_count() - n0 == 1                 # one k_record_copy
    ctx.minimize(fid)                                   # already minimized: nothing
    assert ctx.launch_count() - n0 == 1
    assert ctx.memory_usage() == (base.n_device + 1, base.device_bytes + residue + body, base.n_host, base.host_bytes)
    if tier == "host":
        ctx.offload(fid)
        assert ctx.launch_count() - n0 == 2             # one k_record_copy
        offloaded = (base.n_device, base.device_bytes + residue, base.n_host + 1, base.host_bytes + body)
        assert ctx.memory_usage() == offloaded
        ctx.offload(fid)                                # already offloaded: nothing
        assert ctx.launch_count() - n0 == 2
        assert ctx.memory_usage() == offloaded
    # in place on the record
    assert _host_state(ctx, fid) == {k: before[k] for k in ("pose", "counters", "stats", "react")}
    names = {abi.BUF_IMAGE: "image", abi.BUF_IDEPTH: "idepth", abi.BUF_IDEPTH_VAR: "idepthVar"}
    for w, b in _level0(ctx, fid, has_depth).items():
        assert b == before[(names[w], 0)], w
    _dirty_free_slots(ctx, bufs, *other, perma_pts > 0)
    n1 = ctx.launch_count()
    ctx.activate(fid)
    assert ctx.launch_count() - n1 == 3                 # unpack, image pyramid, gradients: the same kernels from either tier
    ctx.activate(fid)                                   # already active: nothing
    assert ctx.launch_count() - n1 == 3
    assert ctx.memory_usage() == base
    assert (_goodmask(ctx, fid) == 1).all()             # clear_refPixelWasGood, Frame.cpp:388
    if expect_mask_cleared:
        assert not (mask_before == 1).all()
    after = {} if probe is None else _probe(ctx, fid, *probe)
    bufs, has_depth_after = _buffers(ctx, fid, perma_pts > 0)
    after.update(bufs)
    assert has_depth_after == has_depth
    assert after.keys() == before.keys()
    for k in before:
        assert after[k] == before[k], k


# ---- round trips ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tier", TIERS)
def test_round_trip_mapped_keyframe(seq_small, frames_small, tier):
    """a GT-initialised keyframe mapped over 10 frames, finalized (reactivation data) and with a permaRef"""
    gs = _stream(seq_small, 12, 10, 8)
    ctx = gs.ctx
    assert gs.kf_id == 10
    n = gs.tracker.setPermaRef(0)
    assert n > 0 and _host_state(ctx, 0)["react"] is not None
    _round_trip(ctx, 0, frames_small[7], tier, perma_pts=n, probe=(300, frames_small[3][0]))
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("model", ["ptam", "opencv"])
def test_round_trip_undistorted_keyframe(seq_small, frames_small, model, tier):
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
    _round_trip(ctx, 3, frames_small[7], tier, probe=(300, frames_small[1][0]))
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tier", TIERS)
def test_round_trip_tracked_frame(seq_small, frames_small, tier):
    """a plain frame from the prefetch ring, tracked (so it has a good mask), never mapped: the body is its image only"""
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=4)
    ctx.upload(0, frames_small[0][0])
    ctx.set_depth_gt(0, frames_small[0][1])
    abi.DepthMap(ctx).initializeFromGTDepth(0)
    ctx.stage_reserve(1)
    ctx.stage_put(0, frames_small[2][0])
    ctx.frame_from_stage(2, 0)
    trk = abi.SE3Tracker(ctx)
    trk.importFrame(0)
    trk.trackFrame(0, 2, IDENT)
    assert not trk.diverged
    _round_trip(ctx, 2, frames_small[7], tier, expect_mask_cleared=True)
    ctx.close()


@pytest.mark.gpu
def test_offload_and_activate_do_not_wait_for_the_device(seq_small, frames_small):
    """behind a sleep on the caller's stream, minimize, offload and activate only enqueue; activation straight after the offload,
    with no host synchronise in between, restores the frame"""
    import torch
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=4)
    try:
        ctx.upload(0, frames_small[0][0])
        ctx.set_depth_gt(0, frames_small[0][1])
        ctx.upload(1, frames_small[1][0])
        ctx.minimize(1)
        ctx.offload(1)                                   # the host pool exists before the timed calls
        ctx.activate(1)
        before, _ = _snapshot(ctx, 0)
        t = torch.from_numpy(np.ascontiguousarray(frames_small[2][0])).cuda()
        torch.cuda.synchronize()
        s = torch.cuda.current_stream()
        torch.cuda._sleep(SLEEP_CYCLES)
        ctx.upload(2, t)                                 # the context's stream now waits for the sleep
        ctx.minimize(0)
        ctx.offload(0)
        ctx.activate(0)
        ctx.minimize(0)
        ctx.offload(0)
        assert not s.query()
        torch.cuda.synchronize()
        assert ctx.memory_usage().n_host == 1
        ctx.activate(0)
        after, _ = _snapshot(ctx, 0)
        assert after == before
    finally:
        ctx.close()


# ---- in-place reads ------------------------------------------------------------------------------------------------------------
def _finished_keyframes(seq):
    """a stream with 4+ finished keyframes, each with a permaRef, and frame 200 to track on them"""
    gs = _stream(seq, 22, 6, 12)
    for k in gs.keyframe_ids[:-1]:
        gs.tracker.setPermaRef(k)
    gs.ctx.upload(200, seq.render(5)[0])
    gs.ctx.cloud_reserve(3)
    return gs


@pytest.mark.gpu
@pytest.mark.parametrize("tier", TIERS)
def test_in_place_reads_equal_the_all_active_context(seq_small, tier):
    """getters, a pending meanIdepth, reactivation data, level-0 downloads (host, and CUDA tensor behind a sleeping producer
    stream), the permaRef batches and the cloud export (host and device output, both layouts) over keyframes mixing active and
    minimized ones (a third of the finished ones offloaded for the host tier) equal the same calls on a context where every
    keyframe stays active"""
    import torch
    ref, mix = _finished_keyframes(seq_small), _finished_keyframes(seq_small)
    kfs = ref.keyframe_ids
    finished = kfs[:-1]
    assert len(finished) >= 3
    minimized = finished[0::3] + finished[1::3]
    offloaded = finished[0::3] if tier == "host" else []
    for k in minimized:
        mix.ctx.minimize(k)
    for k in offloaded:
        mix.ctx.offload(k)                               # before any depth-stats read: the pending meanIdepth moves with the residue
    assert mix.ctx.memory_usage()[::2] == (len(minimized) - len(offloaded), len(offloaded))
    rng = np.random.default_rng(5)
    qts = np.tile(IDENT, (len(finished), 1))
    qts[:, 4:7] = rng.normal(0, 0.01, (len(finished), 3))
    c2w = ref.keyframe_cam_to_world_f7()

    def run(gs):
        ctx, trk = gs.ctx, gs.tracker
        out = {k: _host_state(ctx, k) for k in kfs}
        for k in finished:
            out[("level0", k)] = _level0(ctx, k, True)
        out["usage"] = trk.checkPermaRefOverlap(finished, qts).tobytes()
        out["track"] = [bytes(r) for r in trk.trackFrameOnPermaref(finished, 200, qts)]
        for lay in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
            pts, counts = ctx.export_pointcloud(kfs, c2w, level=0, layout=lay)
            out[("cloud", lay)] = (pts.tobytes(), counts.tobytes())
            dev = torch.zeros((len(kfs) * (W - 2) * (H - 2), 4), dtype=torch.float32, device="cuda")
            dpts, dcounts = ctx.export_pointcloud(kfs, c2w, level=0, layout=lay, out=dev)
            out[("cloud_device", lay)] = (dpts.cpu().numpy().tobytes(), dcounts.tobytes())
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            dst = torch.full((H, W), -7.0, dtype=torch.float32, device="cuda")
            for k in finished:
                for w in (abi.BUF_IMAGE, abi.BUF_IDEPTH, abi.BUF_IDEPTH_VAR):
                    out[("device_download", k, w)] = (ctx.download(k, w, 0, out=dst) * 1).cpu().numpy().tobytes()
        return out

    want, got = run(ref), run(mix)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k
    k = finished[0]
    assert got[("device_download", k, abi.BUF_IMAGE)] == want[("level0", k)][abi.BUF_IMAGE]
    with pytest.raises(abi.LsdGpuError, match=f"{k}.*minimized"):
        mix.ctx.export_pointcloud(kfs, c2w, level=1)
    # the setters act on the minimized frame
    mix.ctx.set_pose(k, [0.1, 0.2, 0.3, 0.9, 1, 2, 3, 1.5], 7, 0.25)
    mix.ctx.set_counters(k, 4, 5)
    q, pid, itr = mix.ctx.get_pose(k)
    assert list(q) == [0.1, 0.2, 0.3, 0.9, 1, 2, 3, 1.5] and pid == 7 and itr == np.float32(0.25)
    assert mix.ctx.get_counters(k) == (4, 5)
    ref.ctx.close()
    mix.ctx.close()


# ---- refusals and accounting ---------------------------------------------------------------------------------------------------
def _minimized_frame(seq, tier):
    """a stream of frames 37..48 with keyframe 47; keyframe 37, with a permaRef, minimized (and offloaded for the host tier)"""
    gs = _stream(seq, 12, 10, 4, first_id=37)
    assert gs.kf_id == 47
    gs.tracker.setPermaRef(37)
    gs.ctx.minimize(37)
    if tier == "host":
        gs.ctx.offload(37)
    return gs


def _refusals(ctx, seq, frames, fid, other_kf, other):
    """(rc, message) of every entry point that refuses a minimized frame, called on frame `fid`; none launches anything, changes
    the frame's host-side state or builds frame 50"""
    L, p = ctx.L, ctx.ptr
    state0 = _host_state(ctx, fid)
    img = np.ascontiguousarray(frames[1][0])
    u8 = img.ctypes.data_as(C.POINTER(C.c_uint8))
    f32 = np.zeros(seq.w * seq.h * 8, np.float32)
    fp = f32.ctypes.data_as(C.POINTER(C.c_float))
    qt = np.array([0, 0, 0, 1, 0, 0, 0, 1], np.float64)
    dp = qt.ctypes.data_as(C.POINTER(C.c_double))
    one = (C.c_int * 1)(fid)
    res, s3res, ev, s3ev = abi.TrackResult(), abi.Sim3Result(), abi.EvalResult(), abi.Sim3EvalResult()
    hyp = (abi.Hyp * (seq.w * seq.h))()
    pts = np.zeros(seq.w * seq.h, abi.CLOUD_PLY_DTYPE)
    npts = C.c_int64()
    flt = abi.default_cloud_filter()
    ctx.stage_reserve(1)
    ctx.stage_put(0, img)
    ctx.cloud_reserve(2)
    step = abi.GroupStep()
    step.ctx, step.kf_id, step.frame_id, step.gray, step.stage_index = p, other_kf, fid, u8, -1
    step.frameToRef_init_qt[:] = [0, 0, 0, 1, 0, 0, 0]
    vp = lambda a: a.ctypes.data_as(C.c_void_p)         # noqa: E731
    calls = {
        "se3_track kf": lambda: L.lsdgpu_se3_track(p, fid, other, dp, None, 1, C.byref(res)),
        "se3_track frame": lambda: L.lsdgpu_se3_track(p, other_kf, fid, dp, None, 1, C.byref(res)),
        "se3_eval": lambda: L.lsdgpu_se3_eval(p, fid, other, 1, fp, 1.0, 0.0, None, 0, C.byref(ev)),
        "sim3_track_batch": lambda: L.lsdgpu_sim3_track_batch(p, 1, one, (C.c_int * 1)(other_kf), dp, 4, 1, None, C.byref(s3res)),
        "sim3_eval": lambda: L.lsdgpu_sim3_eval(p, other_kf, fid, 2, dp, 1.0, 0.0, None, C.byref(s3ev)),
        "ref_import": lambda: L.lsdgpu_ref_import(p, fid),
        "set_perma_ref": lambda: L.lsdgpu_frame_set_perma_ref(p, fid, None),
        "perma_track frame": lambda: L.lsdgpu_perma_track_batch(p, 1, one, fid, dp, C.byref(res)),
        "init_from_gt": lambda: L.lsdgpu_depth_init_from_gt(p, fid),
        "set_hypotheses": lambda: L.lsdgpu_depth_set_hypotheses(p, fid, hyp, 1, 1),
        "set_from_existing_kf": lambda: L.lsdgpu_depth_set_from_existing_kf(p, fid),
        "update_keyframe": lambda: L.lsdgpu_depth_update_keyframe(p, one, 1),
        "observe": lambda: L.lsdgpu_depth_observe(p, one, 1),
        "propagate": lambda: L.lsdgpu_depth_propagate(p, fid),
        "create_keyframe": lambda: L.lsdgpu_depth_create_keyframe(p, fid, dp),
        "take_reactivation": lambda: L.lsdgpu_frame_take_reactivation_data(p, fid),
        "pack_pointcloud": lambda: L.lsdgpu_keyframe_pack_pointcloud(p, fid, 0, vp(pts)),
        "cloud level 1": lambda: L.lsdgpu_map_export_pointcloud(p, 1, one, f32[:7].ctypes.data_as(C.POINTER(C.c_float)), 1,
                                                                C.byref(flt), 0, vp(pts), len(pts), C.byref(npts), None),
        "download gradients": lambda: L.lsdgpu_frame_download(p, fid, abi.BUF_GRADIENTS, 0, vp(f32)),
        "download image level 1": lambda: L.lsdgpu_frame_download(p, fid, abi.BUF_IMAGE, 1, vp(f32)),
        "download maxgrad": lambda: L.lsdgpu_frame_download(p, fid, abi.BUF_MAXGRAD, 0, vp(f32)),
        "download goodmask": lambda: L.lsdgpu_frame_download(p, fid, abi.BUF_GOODMASK, 1, vp(f32)),
        "set_depth_gt": lambda: L.lsdgpu_frame_set_depth_gt(p, fid, fp, 1.0),
        "set_idepth": lambda: L.lsdgpu_frame_set_idepth(p, fid, fp, fp),
        "clear_good_mask": lambda: L.lsdgpu_frame_clear_good_mask(p, fid),
        "upload": lambda: L.lsdgpu_frame_upload_u8(p, fid, u8),
        "frame_from_stage": lambda: L.lsdgpu_frame_from_stage(p, fid, 0),
        "track_and_map kf": lambda: L.lsdgpu_track_and_map(p, fid, 50, u8, -1, dp, None, 1, 0, C.byref(res), dp),
        "track_and_map frame": lambda: L.lsdgpu_track_and_map(p, other_kf, fid, u8, -1, dp, None, 1, 0, C.byref(res), dp),
        "group step": lambda: L.lsdgpu_track_and_map_group(1, C.byref(step), C.byref(res), None),
    }
    out = {}
    for name, call in calls.items():
        launches = ctx.launch_count()
        rc = call()
        out[name] = (rc, L.lsdgpu_last_error(p).decode())
        assert ctx.launch_count() == launches, name
        assert _host_state(ctx, fid) == state0, name
        assert L.lsdgpu_frame_get_pose(p, 50, None, None, None) != 0, name          # no frame was built
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("tier", TIERS)
def test_refusals_and_accounting(seq_small, frames_small, tier):
    """every call that needs a frame in a slot refuses a minimized one, from either tier with the same message, and changes
    nothing; minimize, offload and activate refuse the active keyframe and unknown ids; release brings both tiers back to zero"""
    gs = _minimized_frame(seq_small, tier)
    ctx, dm = gs.ctx, gs.map
    state0, depth0 = _host_state(ctx, 37), dm.current().tobytes()
    got = _refusals(ctx, seq_small, frames_small, 37, 47, 48)
    for name, (rc, msg) in got.items():
        assert rc != 0 and re.search(r"\b37\b", msg) and "minimized" in msg, (name, msg)
    if tier == "host":
        a = _minimized_frame(seq_small, "device")
        assert got == _refusals(a.ctx, seq_small, frames_small, 37, 47, 48)
        a.ctx.close()
    assert dm.current().tobytes() == depth0
    assert dm.activeKeyFrame() == 47
    usage = ctx.memory_usage()
    assert usage[::2] == ((0, 1) if tier == "host" else (1, 0))
    # a frame in a slot, the active keyframe and unknown ids
    n = ctx.launch_count()
    for call, fid, msg in ((ctx.offload, 48, "frame 48 is active.*minimize it first"), (ctx.offload, 47, "frame 47 is active"),
                           (ctx.offload, 12345, "unknown frame id"), (ctx.minimize, 47, "active keyframe"),
                           (ctx.minimize, 12345, "unknown frame id"), (ctx.activate, 12345, "unknown frame id")):
        with pytest.raises(abi.LsdGpuError, match=msg):
            call(fid)
    assert ctx.launch_count() == n and ctx.memory_usage() == usage
    assert ctx.download(47, abi.BUF_GRADIENTS, 2).size
    assert ctx.download(48, abi.BUF_GRADIENTS, 2).size
    # no free slot: the frame stays minimized
    ctx.upload(60, frames_small[2][0])
    ctx.upload(61, frames_small[3][0])
    with pytest.raises(abi.LsdGpuError, match="no free frame slot to activate frame 37"):
        ctx.activate(37)
    assert ctx.memory_usage() == usage and _host_state(ctx, 37) == state0
    assert ctx.download(37, abi.BUF_IMAGE, 0).size
    with pytest.raises(abi.LsdGpuError, match="minimized"):
        ctx.download(37, abi.BUF_IMAGE, 1)
    assert dm.current().tobytes() == depth0
    # release: both tiers back to zero, and the frame is gone
    ctx.release(61)
    ctx.minimize(60)
    assert ctx.memory_usage().n_device == usage.n_device + 1
    ctx.release(37)
    ctx.release(60)
    assert ctx.memory_usage() == (0, 0, 0, 0)
    for call in (ctx.activate, ctx.offload, ctx.get_pose):
        with pytest.raises(abi.LsdGpuError, match="unknown frame id"):
            call(37)
    ctx.close()


@pytest.mark.gpu
def test_destroy_returns_the_records(seq_small, frames_small):
    """contexts destroyed with device-tier and host-tier records give back their device memory: the free memory after each of
    three such contexts is the same"""
    import torch
    free = []
    for _ in range(3):
        ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=4)
        for k in range(4):
            ctx.upload(k, frames_small[k][0])
            ctx.set_depth_gt(k, frames_small[k][1])
            ctx.minimize(k)
        for k in (0, 2):
            ctx.offload(k)
        assert ctx.memory_usage()[::2] == (2, 2)
        ctx.close()
        torch.cuda.synchronize()
        free.append(torch.cuda.mem_get_info()[0])
    assert abs(free[2] - free[1]) < (2 << 20), free


# ---- streams -------------------------------------------------------------------------------------------------------------------
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


@pytest.mark.gpu
def test_continued_operation_matches_resident_run(seq_small):
    a = _continued(seq_small, False)
    b = _continued(seq_small, True)
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], k


def _stream_outputs(seq, **kw):
    gs = _stream(seq, 40, 6, 6 if kw else 16, **kw)
    ctx = gs.ctx
    usage = ctx.memory_usage()
    out = {"poses": np.array(gs.poses).tobytes(), "kf_c2w": np.array(gs.keyframe_cam_to_world).tobytes(),
           "kf_poses": [(np.asarray(q).tobytes(), pid, itr) for q, pid, itr in (ctx.get_pose(k) for k in gs.keyframe_ids)],
           "depth": gs.map.current().tobytes(), "level0": [_level0(ctx, k, True) for k in gs.keyframe_ids]}
    ctx.cloud_reserve(4)
    out["cloud"] = tuple(a.tobytes() for a in ctx.export_pointcloud(gs.keyframe_ids, gs.keyframe_cam_to_world_f7(), level=0))
    ctx.close()
    return out, usage, len(gs.keyframe_ids)


@pytest.mark.gpu
@pytest.mark.parametrize("max_device_records", [0, 1])
def test_stream_with_host_records_matches_resident_run(seq_small, max_device_records):
    want, usage0, n_kf = _stream_outputs(seq_small)
    got, usage, _ = _stream_outputs(seq_small, max_active_keyframes=2, max_device_records=max_device_records)
    assert usage0 == (0, 0, 0, 0)
    n_min = n_kf - 1 - 2                                  # finished keyframes beyond the two active ones
    assert n_min >= 3
    assert usage.n_device == max_device_records and usage.n_host == n_min - max_device_records
    residue, body = _layout(True, True, 0)
    assert usage.host_bytes == usage.n_host * body
    assert usage.device_bytes == usage.n_host * residue + usage.n_device * (residue + body)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k


def test_stream_rejects_bad_device_record_limits():
    for kw in ({"keep_keyframes": True, "max_device_records": 1},
               {"keep_keyframes": True, "max_active_keyframes": 2, "max_device_records": -1}):
        with pytest.raises(ValueError, match="max_device_records"):
            GpuStream(None, **kw)


@pytest.mark.gpu
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
