"""Depth in and out of device memory (lsdgpu_frame_set_depth_gt_device, lsdgpu_frame_set_idepth_device,
lsdgpu_depth_set_hypotheses_device, lsdgpu_depth_download_device, lsdgpu_keyframe_pack_pointcloud_device): ground-truth depth,
idepth planes and hypotheses taken from CUDA tensors, the depth map and keyframeMsg records written into CUDA tensors, all ordered
on the caller's stream.  Every result is compared byte for byte with the host entry point it mirrors, on the same context or on an
identical one; the other suites pin those to the reference."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream
from tests.util import assert_same, observe

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W, H = 320, 240
LEVELS = 5
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s on an H100
SENTINEL = 0x5A


def _cuda_f32(a, extra=0, fill=float("nan")):
    """a (h, w) float32 array as a CUDA tensor; extra > 0: a view of the first columns of a tensor `extra` columns wider, whose
    other columns hold `fill` (they must never be read)"""
    h, w = a.shape
    t = torch.full((h, w + extra), fill, dtype=torch.float32, device="cuda")
    t[:, :w] = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    return t[:, :w]


def _cuda_bytes(a):
    """the bytes of a host array as a flat uint8 CUDA tensor"""
    return torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8).copy()).cuda()


def _depth_planes(ctx, fid):
    """idepth and idepthVar of every level (levels 1..4 are built on demand from level 0), as bytes"""
    return {(what, lvl): ctx.download(fid, what, lvl).tobytes() for what in (abi.BUF_IDEPTH, abi.BUF_IDEPTH_VAR) for lvl in range(LEVELS)}


def _hard_depth(ctx, seq, fid, k=0):
    """the frame's metric depth with NaN, 0, negative and infinite values, and a minUseGrad equal to the maxGradients of some
    interior pixels (the `>=` of Frame.cpp:269), returned with that minUseGrad"""
    depth = seq.render(k)[1].astype(np.float32).copy()
    rng = np.random.default_rng(11)
    for v in (np.nan, 0.0, -1.0, -0.0, np.inf, 1e-30):
        idx = rng.integers(0, depth.size, 400)
        depth.reshape(-1)[idx] = v
    depth[0, :] = 2.0                                  # the frame border: always -1
    depth[:, -1] = 3.0
    mg = ctx.download(fid, abi.BUF_MAXGRAD)
    interior = np.zeros_like(mg, bool)
    interior[1:-1, 1:-1] = True
    vals = np.sort(mg[interior & (mg > 0)])
    th = vals[len(vals) // 2]
    depth[interior & (mg == th)] = 4.0                 # valid depth on the edge of the gradient test
    return depth, float(th)


# ---- ground-truth depth in ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cov_scale", [1.0, 2.75])
@pytest.mark.parametrize("extra", [0, 5])
def test_set_depth_gt_from_cuda_tensor_equals_host_call(extra, cov_scale):
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4)
    try:
        img = seq.render(0)[0]
        ctx.upload(1, img)
        ctx.upload(2, img)
        depth, th = _hard_depth(ctx, seq, 1)
        ctx.set_globals(minUseGrad=th)
        t = _cuda_f32(depth, extra)
        assert t.stride(0) == W + extra
        ctx.set_depth_gt(1, depth, cov_scale)
        ctx.set_depth_gt(2, t, cov_scale)
        want = _depth_planes(ctx, 1)
        assert _depth_planes(ctx, 2) == want
        id0 = ctx.download(1, abi.BUF_IDEPTH)
        mg = ctx.download(1, abi.BUF_MAXGRAD)
        assert (id0 > 0).sum() > 1000 and (id0 == -1).sum() > 1000
        assert ((mg == np.float32(th)) & (id0 > 0)).any()               # the `>=` edge took valid depth
        dm = abi.DepthMap(ctx)
        dm.initializeFromGTDepth(1)
        want_hyp = dm.current().tobytes()
        dm.initializeFromGTDepth(2)
        assert dm.current().tobytes() == want_hyp
        assert ctx.depth_stats(2) == ctx.depth_stats(1)
    finally:
        ctx.close()


def _run_stream(w, h, from_device, n=30):
    seq = synth.Sequence(w, h, seed=1234)
    frames = [seq.render(k) for k in range(n)]
    ctx = abi.Context(w, h, seq.K, max_frames=8)
    gs = GpuStream(ctx, mode=1, kf_every=10)
    log = []
    try:
        img, depth = frames[0]
        if from_device:
            t_img = torch.zeros((h, w + 7), dtype=torch.uint8, device="cuda")[:, :w]
            t_img.copy_(torch.from_numpy(img))
            gs.init_gt(0, t_img, _cuda_f32(depth, 3))
        else:
            gs.init_gt(0, img, depth)
        log.append([{"depth": gs.map.current().tobytes(), "planes": _depth_planes(ctx, 0)}])
        for k in range(1, n):
            gs.step(k, frames[k][0])
            log.append([observe(gs, k, gs._qts.copy() if gs.kf_id == k else None)])
        log.append([{"keyframes": np.stack(gs.keyframe_cam_to_world).tobytes(), "poses": np.stack(gs.poses).tobytes()}])
    finally:
        ctx.close()
    return log


@pytest.mark.parametrize("size", [(320, 240), (640, 480)])
def test_stream_started_from_cuda_tensors_is_bit_identical(size):
    assert_same(_run_stream(*size, from_device=True), _run_stream(*size, from_device=False))


def _idepth_planes(seq, k=0):
    depth = seq.render(k)[1].astype(np.float32)
    rng = np.random.default_rng(5)
    valid = rng.random(depth.shape) < 0.7
    idepth = np.where(valid, 1.0 / depth, -1).astype(np.float32)
    var = np.where(valid, rng.uniform(1e-4, 1e-2, depth.shape), -1).astype(np.float32)
    return idepth, var


@pytest.mark.parametrize("extra", [0, 9])
def test_set_idepth_from_cuda_tensors_equals_host_call(extra):
    seq = synth.Sequence(W, H, seed=1234)
    idepth, var = _idepth_planes(seq)
    results = []
    for from_device in (False, True):
        ctx = abi.Context(W, H, seq.K, max_frames=4)
        try:
            ctx.upload(0, seq.render(0)[0])
            if from_device:
                ctx.set_idepth(0, _cuda_f32(idepth, extra), _cuda_f32(var, extra))
            else:
                ctx.set_idepth(0, idepth, var)
            level0 = (ctx.download(0, abi.BUF_IDEPTH).tobytes(), ctx.download(0, abi.BUF_IDEPTH_VAR).tobytes())
            trk = abi.SE3Tracker(ctx, mode=1)
            trk.importFrame(0)
            planes = _depth_planes(ctx, 0)
            ctx.upload(3, seq.render(3)[0])
            pose = trk.trackFrame(0, 3, np.array([0, 0, 0, 1, 0, 0, 0], np.float64))
            results.append((level0, planes, pose.tobytes(), bytes(trk.last)))
        finally:
            ctx.close()
    host, dev = results
    assert dev[0] == host[0]
    assert host[0] == (idepth.tobytes(), var.tobytes())
    assert dev[1] == host[1]
    assert dev[2] == host[2] and dev[3] == host[3]


# ---- hypotheses in and out ------------------------------------------------------------------------------------------------
def _mapped_stream(n_frames=12, kf_every=8, max_frames=16):
    seq = synth.Sequence(W, H, seed=4321)
    ctx = abi.Context(W, H, seq.K, max_frames=max_frames)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every, keep_keyframes=True)
    img, d = seq.render(0)
    gs.init_gt(0, img, d)
    for k in range(1, n_frames):
        gs.step(k, seq.render(k)[0])
    return seq, gs


def test_depth_download_into_cuda_tensor_equals_host_download():
    seq, gs = _mapped_stream()
    try:
        want = gs.map.current()
        assert (want["isValid"] > 0).sum() > 1000
        n = W * H * 32
        out = torch.full((n + 48,), SENTINEL, dtype=torch.uint8, device="cuda")
        v = gs.map.current(out=out)
        assert tuple(v.shape) == (H, W, 32) and v.data_ptr() == out.data_ptr()
        assert v.cpu().numpy().tobytes() == want.tobytes()
        assert (out[n:] == SENTINEL).all()
        f = abi.hyp_fields(v)
        for name in ("isValid", "blacklisted", "validity_counter", "idepth_smoothed", "idepth_var", "nextStereoFrameMinID"):
            assert f[name].cpu().numpy().tobytes() == np.ascontiguousarray(want[name]).tobytes(), name
        assert (v[:, :, 1:4] == 0).all()                                  # pad bytes 0, as the host twin writes them
    finally:
        gs.ctx.close()


def _edited_hypotheses(hyp):
    """the mapped state with records the host twin normalises: isValid = 2, non-zero pad bytes"""
    h = hyp.copy()
    rng = np.random.default_rng(3)
    m = rng.random(h.shape) < 0.1
    h["isValid"][m & (h["isValid"] > 0)] = 2
    h["_pad"][m] = 0x7F
    h["validity_counter"][m] += 3
    return h


def _map_state(ctx, dm, kf):
    return {"hyp": dm.current().tobytes(), "planes": _depth_planes(ctx, kf), "stats": ctx.depth_stats(kf),
            "counters": ctx.get_counters(kf), "active": dm.activeKeyFrame()}


@pytest.mark.parametrize("reactivated,do_set_depth", [(False, False), (False, True), (True, False), (True, True)])
def test_set_hypotheses_from_cuda_tensor_equals_host_call(reactivated, do_set_depth):
    seq, gs = _mapped_stream()
    ctx, dm = gs.ctx, gs.map
    try:
        hyp = _edited_hypotheses(dm.current())
        kf = gs.keyframe_ids[0]
        states = []
        for src in (hyp, _cuda_bytes(hyp)):
            ctx.set_counters(kf, 5, 6)
            dm.setHypotheses(kf, src, reactivated=reactivated, do_set_depth=do_set_depth)
            states.append(_map_state(ctx, dm, kf))
        assert states[1] == states[0]
        assert states[0]["active"] == kf
        assert (states[0]["counters"] == (0, 0)) == reactivated
    finally:
        ctx.close()


def test_hypotheses_round_trip_through_a_tensor():
    seq, gs = _mapped_stream()
    ctx, dm = gs.ctx, gs.map
    try:
        want = dm.current().tobytes()
        t = dm.current(out=torch.empty(W * H * 32, dtype=torch.uint8, device="cuda"))
        dm.reset()
        dm.setHypotheses(gs.kf_id, t, do_set_depth=False)
        assert dm.current().tobytes() == want
    finally:
        ctx.close()


# ---- keyframeMsg records out ----------------------------------------------------------------------------------------------
def test_pack_pointcloud_into_cuda_tensor_equals_host_packing():
    seq, gs = _mapped_stream()
    ctx = gs.ctx
    try:
        for kf in (gs.keyframe_ids[0], gs.kf_id):
            for level in range(LEVELS):
                want = ctx.pack_pointcloud(kf, level)
                n = want.size * 12
                out = torch.full((n + 20,), SENTINEL, dtype=torch.uint8, device="cuda")
                v = ctx.pack_pointcloud(kf, level, out=out)
                assert tuple(v.shape) == (want.size, 12) and v.data_ptr() == out.data_ptr()
                assert v.cpu().numpy().tobytes() == want.tobytes(), (kf, level)
                assert (out[n:] == SENTINEL).all()
    finally:
        ctx.close()


# ---- ordering on the caller's stream --------------------------------------------------------------------------------------
def test_inputs_written_behind_a_sleep_on_the_callers_stream_are_read():
    seq, gs = _mapped_stream()
    ctx, dm = gs.ctx, gs.map
    try:
        img, depth = seq.render(20)
        idepth, var = _idepth_planes(seq, 20)
        hyp = _edited_hypotheses(dm.current())
        for fid in (40, 41, 42, 43):
            ctx.upload(fid, img)
        ctx.set_depth_gt(40, depth)
        ctx.set_idepth(42, idepth, var)
        kf = gs.keyframe_ids[0]
        dm.setHypotheses(kf, hyp, do_set_depth=False)
        want_hyp = dm.current().tobytes()
        dm.reset()
        src_d, src_i, src_v, src_h = _cuda_f32(depth), _cuda_f32(idepth), _cuda_f32(var), _cuda_bytes(hyp)
        t_d, t_i, t_v = (torch.zeros((H, W), dtype=torch.float32, device="cuda") for _ in range(3))
        t_h = torch.zeros(W * H * 32, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            for t, s in ((t_d, src_d), (t_i, src_i), (t_v, src_v), (t_h, src_h)):
                t.copy_(s)
            ctx.set_depth_gt(41, t_d)
            ctx.set_idepth(43, t_i, t_v)
            dm.setHypotheses(kf, t_h, do_set_depth=False)
            for t in (t_d, t_i, t_v, t_h):                                # after the calls: must not reach them
                t.zero_()
        assert _depth_planes(ctx, 41) == _depth_planes(ctx, 40)
        assert _depth_planes(ctx, 43) == _depth_planes(ctx, 42)
        assert dm.current().tobytes() == want_hyp
        torch.cuda.synchronize()
    finally:
        ctx.close()


def test_outputs_consumed_on_the_callers_stream_right_after_the_call():
    seq, gs = _mapped_stream()
    ctx, dm = gs.ctx, gs.map
    try:
        want_hyp = dm.current().tobytes()
        want_pc = ctx.pack_pointcloud(gs.kf_id, 1).tobytes()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            o_h = torch.zeros(W * H * 32, dtype=torch.uint8, device="cuda")
            got_h = (dm.current(out=o_h) + 0).clone()
            o_p = torch.zeros((W // 2) * (H // 2) * 12, dtype=torch.uint8, device="cuda")
            got_p = (ctx.pack_pointcloud(gs.kf_id, 1, out=o_p) + 0).clone()
        side.synchronize()
        assert got_h.cpu().numpy().tobytes() == want_hyp
        assert got_p.cpu().numpy().tobytes() == want_pc
    finally:
        ctx.close()


def test_depth_calls_do_not_wait_for_the_device():
    seq = synth.Sequence(W, H, seed=1234)
    ctx = abi.Context(W, H, seq.K, max_frames=4)
    gs = GpuStream(ctx, mode=1)
    try:
        img, depth = seq.render(0)
        idepth, var = _idepth_planes(seq)
        t_img = torch.from_numpy(img).cuda()
        t_d, t_i, t_v = _cuda_f32(depth, 2), _cuda_f32(idepth), _cuda_f32(var)
        o_h = torch.empty(W * H * 32, dtype=torch.uint8, device="cuda")
        o_p = torch.empty(W * H * 12, dtype=torch.uint8, device="cuda")
        ctx.upload(1, img)
        torch.cuda.synchronize()
        s = torch.cuda.current_stream()
        torch.cuda._sleep(SLEEP_CYCLES)
        gs.init_gt(0, t_img, t_d)                                         # gtDepthInit: upload + setDepthFromGroundTruth + init
        ctx.set_idepth(1, t_i, t_v)
        gs.map.current(out=o_h)
        gs.map.setHypotheses(0, o_h, do_set_depth=True)
        ctx.pack_pointcloud(0, 0, out=o_p)
        assert not s.query()
        torch.cuda.synchronize()
        assert ctx.download(1, abi.BUF_IDEPTH).tobytes() == idepth.tobytes()
        ctx2 = abi.Context(W, H, seq.K, max_frames=4)                    # the same gtDepthInit from host memory
        try:
            want = GpuStream(ctx2, mode=1)
            want.init_gt(0, img, depth)
            assert o_h.cpu().numpy().tobytes() == want.map.current().tobytes()
            assert o_p.cpu().numpy().tobytes() == ctx2.pack_pointcloud(0, 0).tobytes()
        finally:
            ctx2.close()
    finally:
        ctx.close()


# ---- rejections -----------------------------------------------------------------------------------------------------------
def _snapshot(ctx, dm, fids):
    return {"hyp": dm.current().tobytes(), "planes": {f: _depth_planes(ctx, f) for f in fids},
            "active": dm.activeKeyFrame()}


def test_rejected_calls_change_nothing():
    seq, gs = _mapped_stream()
    ctx, dm = gs.ctx, gs.map
    L, p = ctx.L, ctx.ptr
    stream = torch.cuda.current_stream().cuda_stream
    try:
        old = gs.keyframe_ids[0]
        ctx.minimize(old)
        fid = gs.kf_id
        before = _snapshot(ctx, dm, [fid])
        n = W * H
        depth = seq.render(5)[1].astype(np.float32)
        host = np.ascontiguousarray(depth)
        pinned = torch.from_numpy(host).pin_memory()
        dev = torch.full((n + 16,), 0.5, dtype=torch.float32, device="cuda")           # 16-byte aligned (a fresh allocation)
        d0 = dev.data_ptr()
        hyp_host = np.zeros(n * 32, np.uint8)

        def rejected(rc):
            assert rc != 0 and L.lsdgpu_last_error(p).decode()

        for ptr, pitch, f in [(host.ctypes.data, W * 4, fid), (pinned.data_ptr(), W * 4, fid), (None, W * 4, fid),
                              (d0, W * 4 - 4, fid), (d0, W * 4 + 2, fid), (d0 + 2, W * 4, fid),
                              (d0, W * 4, 77), (d0, W * 4, old)]:
            rejected(L.lsdgpu_frame_set_depth_gt_device(p, f, ptr, pitch, 1.0, stream))
            rejected(L.lsdgpu_frame_set_idepth_device(p, f, d0, ptr, pitch, stream))
            rejected(L.lsdgpu_frame_set_idepth_device(p, f, ptr, d0, pitch, stream))
        rejected(L.lsdgpu_frame_set_depth_gt_device(p, old, d0, W * 4, 1.0, stream))
        assert "minimized" in L.lsdgpu_last_error(p).decode()

        hyp_dev = torch.zeros(n * 32 + 64, dtype=torch.uint8, device="cuda")
        h0 = hyp_dev.data_ptr()
        for ptr, f in [(hyp_host.ctypes.data, fid), (None, fid), (h0 + 4, fid), (h0 + 8, fid), (h0, 77), (h0, old)]:
            for r, s in ((0, 0), (1, 1)):
                rejected(L.lsdgpu_depth_set_hypotheses_device(p, f, ptr, r, s, stream))

        out = torch.full((n * 32 + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        o0 = out.data_ptr()
        for ptr, cap in [(o0, n * 32 - 1), (o0 + 4, n * 32), (o0 + 8, n * 32), (hyp_host.ctypes.data, n * 32), (None, n * 32)]:
            rejected(L.lsdgpu_depth_download_device(p, ptr, cap, stream))
        for f, lvl, ptr, cap in [(fid, 0, o0, n * 12 - 1), (fid, 2, o0, (n >> 4) * 12 - 1), (fid, 0, o0 + 2, n * 12),
                                 (fid, 0, hyp_host.ctypes.data, n * 12), (fid, 5, o0, n * 12), (fid, -1, o0, n * 12),
                                 (77, 0, o0, n * 12), (old, 0, o0, n * 12)]:
            rejected(L.lsdgpu_keyframe_pack_pointcloud_device(p, f, lvl, ptr, cap, stream))
        torch.cuda.synchronize()
        assert (out == SENTINEL).all()
        assert (dev == 0.5).all()
        assert _snapshot(ctx, dm, [fid]) == before
        with pytest.raises(abi.LsdGpuError):
            ctx.get_pose(77)                                                # still unknown
        with pytest.raises(abi.LsdGpuError, match="minimized"):
            ctx.set_depth_gt(old, depth)                                    # still minimized
        # a frame without depth: the pack is rejected as by the host twin
        ctx.upload(60, seq.render(3)[0])
        with pytest.raises(abi.LsdGpuError, match="no depth"):
            ctx.pack_pointcloud(60, 0)
        rejected(L.lsdgpu_keyframe_pack_pointcloud_device(p, 60, 0, o0, n * 12, stream))
        torch.cuda.synchronize()
        assert (out == SENTINEL).all()
    finally:
        ctx.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_memory_of_another_device_is_rejected():
    seq, gs = _mapped_stream(n_frames=3)
    ctx, dm = gs.ctx, gs.map
    try:
        fid = gs.kf_id
        before = _snapshot(ctx, dm, [fid])
        t = torch.zeros((H, W), dtype=torch.float32, device="cuda:1")
        b = torch.zeros(W * H * 32, dtype=torch.uint8, device="cuda:1")
        with pytest.raises(ValueError):
            ctx.set_depth_gt(fid, t)
        with pytest.raises(ValueError):
            dm.current(out=b)
        L, p = ctx.L, ctx.ptr
        for rc in (L.lsdgpu_frame_set_depth_gt_device(p, fid, t.data_ptr(), W * 4, 1.0, None),
                   L.lsdgpu_frame_set_idepth_device(p, fid, t.data_ptr(), t.data_ptr(), W * 4, None),
                   L.lsdgpu_depth_set_hypotheses_device(p, fid, b.data_ptr(), 0, 1, None),
                   L.lsdgpu_depth_download_device(p, b.data_ptr(), b.numel(), None),
                   L.lsdgpu_keyframe_pack_pointcloud_device(p, fid, 0, b.data_ptr(), b.numel(), None)):
            assert rc != 0 and "device 1" in L.lsdgpu_last_error(p).decode()
        torch.cuda.synchronize(1)
        assert (b == 0).all()
        assert _snapshot(ctx, dm, [fid]) == before
    finally:
        ctx.close()
