"""Device-resident input and output (the *_device entry points of include/lsdgpu.h): frames built from CUDA tensors, frame planes
and the map's point cloud written into CUDA tensors, all ordered on the caller's stream.  Every result is compared byte for byte
with the host entry point it mirrors on the same context or on an identical one; the other suites pin those to the reference."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from tests.device_cases import GROUP_KF_EVERY, _group_sequence
from tests.util import assert_same, observe, same_cloud

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W, H = 320, 240
LEVELS = 5
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s on an H100


def _cuda(img, extra=0):
    """img as a uint8 CUDA tensor; extra > 0: a view of the first columns of a tensor `extra` columns wider (pitch w + extra)"""
    h, w = img.shape
    t = torch.zeros((h, w + extra), dtype=torch.uint8, device="cuda")
    t[:, :w] = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    return t[:, :w]


def _planes(ctx, fid):
    """what Frame::Frame builds: the image and gradients of every level and maxGradients, as bytes"""
    out = {}
    for lvl in range(LEVELS):
        out[("image", lvl)] = ctx.download(fid, abi.BUF_IMAGE, lvl).tobytes()
        out[("grad", lvl)] = ctx.download(fid, abi.BUF_GRADIENTS, lvl).tobytes()
    out["maxgrad"] = ctx.download(fid, abi.BUF_MAXGRAD, 0).tobytes()
    return out


def _unknown(ctx, fid):
    try:
        ctx.get_pose(fid)
    except abi.LsdGpuError:
        return True
    return False


# ---- frames in ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [0, 3])
def test_upload_from_cuda_tensor_equals_host_upload(extra):
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4)
    try:
        img = seq.render(3)[0]
        t = _cuda(img, extra)
        assert t.stride(0) == W + extra
        ctx.upload(1, img)
        ctx.upload(2, t)
        assert _planes(ctx, 2) == _planes(ctx, 1)
    finally:
        ctx.close()


def _raw(w, h, seed=3):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h // 8 + 2, w // 8 + 2)).astype(np.float32)
    img = np.kron(base, np.ones((8, 8), np.float32))[:h, :w] + rng.normal(0, 6, (h, w))
    return np.clip(img, 0, 255).astype(np.uint8)


UNDISTORTERS = {
    "ptam": lambda: abi.UndistorterPTAM([0.53, 0.71, 0.49, 0.51, 0.897], (400, 300), "crop", (W, H)),
    "pass-through": lambda: abi.UndistorterPTAM([0.5, 0.7, 0.49, 0.51, 0.0], (W, H), "crop", (W, H)),
    "opencv": lambda: abi.UndistorterOpenCV([458.654, 457.296, 367.215, 248.375, -0.2834, 0.0740, 0.00019, 1.76e-05], (752, 480),
                                            "full", (W, H)),
}


@pytest.mark.parametrize("model", sorted(UNDISTORTERS))
@pytest.mark.parametrize("extra", [0, 3])
def test_distorted_upload_from_cuda_tensor_equals_host_upload(model, extra):
    u = UNDISTORTERS[model]()
    if model == "pass-through":
        assert u.status == 1
    ctx = abi.Context(W, H, u.getK(), max_frames=4)
    try:
        u.install(ctx)
        raw = _raw(u.in_w, u.in_h)
        ctx.upload_distorted(1, raw)
        ctx.upload_distorted(2, _cuda(raw, extra))
        assert _planes(ctx, 2) == _planes(ctx, 1)
    finally:
        ctx.close()


# ---- the prefetch ring and the fused calls --------------------------------------------------------------------------------
def _run_stream(seq, frames, fused, from_device, n=40, kf_every=10):
    ctx = abi.Context(W, H, seq.K, max_frames=8)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every, fused_call=fused)
    log = []
    try:
        gs.init_gt(0, frames[0][0], frames[0][1])
        ctx.stage_reserve(2)
        for k in range(1, n):
            img = frames[k][0]
            if from_device:
                ctx.stage_put(k % 2, _cuda(img, 3 * (k % 2)))
                gs.step(k, stage_index=k % 2)
            else:
                gs.step(k, img)
            kf = gs.kf_id == k
            log.append([observe(gs, k, gs._qts.copy() if kf else None)])
        log.append([{"keyframes": np.stack(gs.keyframe_cam_to_world).tobytes(), "poses": np.stack(gs.poses).tobytes()}])
    finally:
        ctx.close()
    return log


@pytest.mark.parametrize("fused", [True, False])
def test_stream_fed_from_cuda_tensors_is_bit_identical(fused):
    seq = synth.Sequence(W, H, seed=1234)
    frames = [seq.render(k) for k in range(40)]
    want = _run_stream(seq, frames, fused, from_device=False)
    got = _run_stream(seq, frames, fused, from_device=True)
    assert_same(got, want)


def _run_group(from_device, phases=(0, 3, 7), n=25):
    streams, seqs = [], []
    for s, ph in enumerate(phases):
        seq, fr = _group_sequence(W, H, s, n + 1)
        ctx = abi.Context(W, H, seq.K, max_frames=8)
        gs = GpuStream(ctx, mode=1, kf_every=GROUP_KF_EVERY, kf_phase=ph)
        gs.init_gt(0, fr[0][0], fr[0][1])
        ctx.stage_reserve(2)
        streams.append(gs)
        seqs.append(fr)
    group = GpuStreamGroup(streams)
    log = []
    try:
        for k in range(1, n + 1):
            kf = [gs.next_is_keyframe_change() for gs in streams]
            if from_device:
                for gs, fr in zip(streams, seqs):
                    gs.ctx.stage_put(k % 2, _cuda(fr[k][0], k % 2))
                group.step([k] * len(streams), stage_indices=[k % 2] * len(streams))
            else:
                group.step([k] * len(streams), images=[fr[k][0] for fr in seqs])
            log.append([observe(gs, k, group._qts[i].copy() if kf[i] else None) for i, gs in enumerate(streams)])
    finally:
        for gs in streams:
            gs.ctx.close()
    return log


def test_group_fed_from_cuda_tensors_is_bit_identical():
    assert_same(_run_group(from_device=True), _run_group(from_device=False))


# ---- outputs --------------------------------------------------------------------------------------------------------------
def _mapped_stream(n_frames=20, kf_every=8, max_frames=12):
    seq = synth.Sequence(W, H, seed=4321)
    ctx = abi.Context(W, H, seq.K, max_frames=max_frames)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every, keep_keyframes=True)
    img, d = seq.render(0)
    gs.init_gt(0, img, d)
    for k in range(1, n_frames):
        gs.step(k, seq.render(k)[0])
    return seq, gs


def _device_download(ctx, fid, what, level, sentinel=0x5A):
    """-> (lsdgpu_frame_download_device's plane as bytes or None if rejected, whether the buffer beyond it or all of it on a
    rejection kept the sentinel)"""
    big = torch.full(((W * H * 16) + 64,), sentinel, dtype=torch.uint8, device="cuda")
    rc = ctx.L.lsdgpu_frame_download_device(ctx.ptr, fid, what, level, big.data_ptr(), big.numel(),
                                            torch.cuda.current_stream().cuda_stream)
    host = big.cpu().numpy()
    if rc != 0:
        return None, bool((host == sentinel).all())
    return host, True


def test_download_into_cuda_tensors_equals_host_download():
    seq, gs = _mapped_stream()
    ctx = gs.ctx
    try:
        kf_old, kf_new = gs.keyframe_ids[0], gs.kf_id
        ctx.upload(50, seq.render(20)[0])                      # tracked, with a good mask
        gs.tracker.trackFrame(kf_new, 50, gs.last_pose)
        ctx.upload(51, seq.render(21)[0])                      # no depth, no good mask: the mask reads as all 1s
        ctx.minimize(kf_old)
        cases = 0
        for fid in (kf_new, 50, 51, kf_old):
            for what in range(6):
                for level in range(LEVELS):
                    try:
                        want = ctx.download(fid, what, level)
                    except abi.LsdGpuError:
                        got, untouched = _device_download(ctx, fid, what, level)
                        assert got is None and untouched, (fid, what, level)
                        continue
                    dtype = torch.uint8 if what == abi.BUF_GOODMASK else torch.float32
                    out = torch.full((W * H * 4,), 7, dtype=dtype, device="cuda")
                    v = ctx.download(fid, what, level, out=out)
                    assert tuple(v.shape) == want.shape
                    assert v.cpu().numpy().tobytes() == want.tobytes(), (fid, what, level)
                    cases += 1
        assert cases >= 30
        assert (ctx.download(51, abi.BUF_GOODMASK) == 1).all()
        assert not (ctx.download(50, abi.BUF_GOODMASK) == 1).all()
    finally:
        ctx.close()


_cloud_cache = {}


def _cloud_stream():
    if "gs" not in _cloud_cache:
        seq, gs = _mapped_stream(n_frames=30, kf_every=8, max_frames=16)
        assert len(gs.keyframe_ids) >= 3
        gs.ctx.cloud_reserve(2)                               # the host export runs in batches of 2 keyframes
        _cloud_cache["gs"] = gs
    return _cloud_cache["gs"]


@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("layout", [abi.CLOUD_PLY, abi.CLOUD_VERTEX])
def test_export_into_cuda_tensor_equals_host_export(level, layout):
    gs = _cloud_stream()
    ctx, ids, c2w = gs.ctx, gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    want, want_counts = ctx.export_pointcloud(ids, c2w, level=level, layout=layout)
    n = len(want)
    bound = len(ids) * ((W >> level) - 2) * ((H >> level) - 2)
    for cap in (bound, n):                                  # the emit launch alone, and the count launch first
        out = torch.full((cap, 4), 3.0, dtype=torch.float32, device="cuda")
        pts, counts = ctx.export_pointcloud(ids, c2w, level=level, layout=layout, out=out)
        assert pts.shape == (n, 4) and pts.data_ptr() == out.data_ptr()
        assert np.array_equal(counts, want_counts)
        same_cloud(pts.cpu().numpy(), np.ascontiguousarray(want).view(np.uint32).reshape(-1, 4))
        if cap > n:
            assert (out[n:] == 3.0).all()


def _export_device(ctx, ids, c2w, out_ptr, capacity, level=0, layout=abi.CLOUD_PLY, stream=None):
    ids = np.ascontiguousarray(ids, np.int32)
    c2w = np.ascontiguousarray(c2w, np.float32)
    counts = np.full((len(ids), 2), -1, np.int32)
    npts = C.c_int64(-1)
    f = abi.default_cloud_filter()
    rc = ctx.L.lsdgpu_map_export_pointcloud_device(ctx.ptr, len(ids), ids.ctypes.data_as(C.POINTER(C.c_int)),
                                                   c2w.ctypes.data_as(C.POINTER(C.c_float)), level, C.byref(f), layout, out_ptr,
                                                   capacity, C.byref(npts), counts.ctypes.data_as(C.POINTER(C.c_int32)),
                                                   stream if stream is not None else torch.cuda.current_stream().cuda_stream)
    return rc, npts.value, counts


def test_export_capacity_one_point_short():
    gs = _cloud_stream()
    ctx, ids, c2w = gs.ctx, gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    n, want_counts = ctx.count_pointcloud(ids, c2w)
    assert n > 0
    out = torch.full((n, 4), -7.0, dtype=torch.float32, device="cuda")
    rc, npts, counts = _export_device(ctx, ids, c2w, out.data_ptr(), n - 1)
    assert rc == abi.CLOUD_ERR_CAPACITY
    assert npts == n and np.array_equal(counts, want_counts)
    assert (out == -7.0).all()
    rc, npts, counts = _export_device(ctx, ids, c2w, None, 0)               # count only
    assert rc == 0 and npts == n and np.array_equal(counts, want_counts)


# ---- ordering on the caller's stream --------------------------------------------------------------------------------------
def test_input_written_behind_a_sleep_on_the_callers_stream_is_read():
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4)
    try:
        img = seq.render(5)[0]
        src = _cuda(img)
        t = torch.zeros((H, W + 3), dtype=torch.uint8, device="cuda")[:, :W]
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.copy_(src)
            ctx.upload(2, t)
        ctx.upload(1, img)
        assert _planes(ctx, 2) == _planes(ctx, 1)
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.fill_(0)
            t.copy_(src)
            ctx.stage_reserve(1)
            ctx.stage_put(0, t)
            t.fill_(0)                                       # after the call: must not reach the ring
        ctx.frame_from_stage(3, 0)
        assert _planes(ctx, 3) == _planes(ctx, 1)
        torch.cuda.synchronize()
    finally:
        ctx.close()


def test_output_consumed_on_the_callers_stream_right_after_the_call():
    gs = _cloud_stream()
    ctx, ids, c2w = gs.ctx, gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    want_img = ctx.download(gs.kf_id, abi.BUF_IDEPTH, 1)
    want_pts, _ = ctx.export_pointcloud(ids, c2w)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        out = torch.zeros(want_img.size, dtype=torch.float32, device="cuda")
        v = ctx.download(gs.kf_id, abi.BUF_IDEPTH, 1, out=out)
        got_img = (v * 1).clone()
        cloud = torch.zeros((len(want_pts) + 5, 4), dtype=torch.float32, device="cuda")
        pts, _ = ctx.export_pointcloud(ids, c2w, out=cloud)
        got_pts = pts.clone()
    side.synchronize()
    assert got_img.cpu().numpy().tobytes() == want_img.tobytes()
    same_cloud(got_pts.cpu().numpy(), np.ascontiguousarray(want_pts).view(np.uint32).reshape(-1, 4))


def test_uploads_and_downloads_do_not_wait_for_the_device():
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4)
    try:
        img = seq.render(5)[0]
        t = _cuda(img, 3)
        out = torch.empty((H, W), dtype=torch.float32, device="cuda")
        ctx.stage_reserve(1)
        torch.cuda.synchronize()
        s = torch.cuda.current_stream()
        torch.cuda._sleep(SLEEP_CYCLES)
        ctx.upload(1, t)
        ctx.stage_put(0, t)
        ctx.download(1, abi.BUF_IMAGE, 0, out=out)
        assert not s.query()
        torch.cuda.synchronize()
        ctx.upload(2, img)
        assert out.cpu().numpy().tobytes() == ctx.download(2, abi.BUF_IMAGE, 0).tobytes()
    finally:
        ctx.close()


# ---- rejections -----------------------------------------------------------------------------------------------------------
def test_rejected_calls_change_nothing():
    seq, gs = _mapped_stream(n_frames=10, kf_every=8)
    ctx = gs.ctx
    L, p = ctx.L, ctx.ptr
    stream = torch.cuda.current_stream().cuda_stream
    try:
        img = seq.render(3)[0]
        dev = _cuda(img)
        host = np.ascontiguousarray(img)
        pinned = torch.from_numpy(host).pin_memory()
        ctx.stage_reserve(1)
        for fid, ptr, pitch in [(90, host.ctypes.data, W), (91, pinned.data_ptr(), W), (92, dev.data_ptr(), W - 1),
                                (93, None, W)]:
            assert L.lsdgpu_frame_upload_device_u8(p, fid, ptr, pitch, stream) != 0
            assert L.lsdgpu_last_error(p).decode()
            assert _unknown(ctx, fid), fid
        assert L.lsdgpu_stage_put_device(p, 1, dev.data_ptr(), W, stream) != 0          # no entry 1
        assert L.lsdgpu_stage_put_device(p, 0, host.ctypes.data, W, stream) != 0
        assert L.lsdgpu_frame_upload_distorted_device_u8(p, 94, dev.data_ptr(), W, stream) != 0   # no undistorter
        assert _unknown(ctx, 94)

        # outputs: misaligned, one byte short, host memory -- nothing written
        n = W * H
        flat = torch.full((n * 4 + 8,), -3.0, dtype=torch.float32, device="cuda")
        fid = gs.kf_id
        for what, ptr, cap in [(abi.BUF_GRADIENTS, flat[1:].data_ptr(), n * 16),
                               (abi.BUF_IMAGE, flat.data_ptr() + 2, n * 4),
                               (abi.BUF_IMAGE, flat.data_ptr(), n * 4 - 1),
                               (abi.BUF_IMAGE, host.ctypes.data, n * 4)]:
            assert L.lsdgpu_frame_download_device(p, fid, what, 0, ptr, cap, stream) != 0
        assert (flat == -3.0).all()
        ids, c2w = gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
        cloud = torch.full((n * 4 + 8,), -3.0, dtype=torch.float32, device="cuda")
        rc, _, counts = _export_device(ctx, ids, c2w, cloud[1:].data_ptr(), n)
        assert rc != 0 and rc != abi.CLOUD_ERR_CAPACITY and (counts == -1).all()
        rc, _, _ = _export_device(ctx, ids, c2w, host.ctypes.data, 10)
        assert rc != 0
        f = abi.default_cloud_filter(sparsifyFactor=2)
        assert L.lsdgpu_map_export_pointcloud_device(p, 1, np.int32([fid]).ctypes.data_as(C.POINTER(C.c_int)),
                                                     c2w[-1:].ctypes.data_as(C.POINTER(C.c_float)), 0, C.byref(f), 0,
                                                     cloud.data_ptr(), n, None, None, stream) != 0
        assert (cloud == -3.0).all()

        # a minimized frame: not re-uploaded, only the planes it keeps are served
        old = gs.keyframe_ids[0]
        ctx.minimize(old)
        assert L.lsdgpu_frame_upload_device_u8(p, old, dev.data_ptr(), W, stream) != 0
        assert "minimized" in L.lsdgpu_last_error(p).decode()
        assert L.lsdgpu_frame_download_device(p, old, abi.BUF_GRADIENTS, 0, flat.data_ptr(), n * 16, stream) != 0
        assert (flat == -3.0).all()
        with pytest.raises(abi.LsdGpuError):
            ctx.download(old, abi.BUF_GRADIENTS, 0)
        torch.cuda.synchronize()
    finally:
        ctx.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_memory_of_another_device_is_rejected():
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4, device=0)
    try:
        t = torch.zeros((H, W), dtype=torch.uint8, device="cuda:1")
        with pytest.raises(ValueError):
            ctx.upload(1, t)
        assert ctx.L.lsdgpu_frame_upload_device_u8(ctx.ptr, 1, t.data_ptr(), W, None) != 0
        assert "device 1" in ctx.L.lsdgpu_last_error(ctx.ptr).decode()
        assert _unknown(ctx, 1)
    finally:
        ctx.close()
