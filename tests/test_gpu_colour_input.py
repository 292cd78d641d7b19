"""Colour and 4:2:2 camera images on the device (lsdgpu_set_input_format, lsdgpu_stage_put_raw*): the conversion cv_bridge /
cv::cvtColor does in front of the undistorter (ROSImageStreamThread.cpp:117, LiveSLAMWrapper.cpp:116-121), fused into the frame
construction and the prefetch ring.  Every 24-bit colour goes through the device and hashes to OpenCV 4.13's table; every format,
camera and route builds the frame the existing gray path builds from the converted image, byte for byte; runs fed colour through
the ring equal runs fed the converted gray images bit for bit; and every refused call changes nothing."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from tests import colour_input_oracle as co
from tests.device_cases import GROUP_KF_EVERY, _group_sequence
from tests.util import assert_same, observe

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W, H = 640, 480
LEVELS = 5
ENCODINGS = ["mono8", "rgb8", "bgr8", "rgba8", "bgra8", "yuv422", "yuv422_yuy2"]
# pass-through at the context's size; both models from a 752 x 480 camera
CAMERAS = {
    "pass-through": lambda w, h: abi.UndistorterPTAM([0.5, 0.7, 0.49, 0.51, 0.0], (w, h), "crop", (w, h)),
    "ptam": lambda w, h: abi.UndistorterPTAM([0.535719, 0.669567, 0.493249, 0.500409, 0.897966], (752, 480), "full", (w, h)),
    "opencv": lambda w, h: abi.UndistorterOpenCV([458.654, 457.296, 367.215, 248.375, -0.2834, 0.0740, 0.00019, 1.76e-05],
                                                 (752, 480), "crop", (w, h)),
}


def _planes(ctx, fid):
    """what Frame::Frame builds: the image and gradients of every level and maxGradients, as bytes"""
    out = {}
    for lvl in range(LEVELS):
        out[("image", lvl)] = ctx.download(fid, abi.BUF_IMAGE, lvl).tobytes()
        out[("grad", lvl)] = ctx.download(fid, abi.BUF_GRADIENTS, lvl).tobytes()
    out["maxgrad"] = ctx.download(fid, abi.BUF_MAXGRAD, 0).tobytes()
    return out


def _cuda(raw, extra):
    """raw as a uint8 CUDA tensor whose row pitch is `extra` bytes larger than its row (odd for odd extra)"""
    flat = np.ascontiguousarray(raw).reshape(raw.shape[0], -1)
    h, row = flat.shape
    t = torch.zeros(h * (row + extra) + row, dtype=torch.uint8, device="cuda")
    t[: h * (row + extra)].view(h, row + extra)[:, :row] = torch.from_numpy(flat).cuda()
    return t.as_strided(raw.shape, (row + extra,) + ((raw.shape[2], 1) if raw.ndim == 3 else (1,)))


def _scene_raw(w, h, enc, seed):
    """a textured raw image in encoding enc: a blocky random scene, its colour channels or chroma drawn independently"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h // 8 + 2, w // 8 + 2)).astype(np.float32)
    g = np.clip(np.kron(base, np.ones((8, 8), np.float32))[:h, :w] + rng.normal(0, 6, (h, w)), 0, 255).astype(np.uint8)
    return _colourize(g, enc, rng)


def _colourize(gray, enc, rng):
    """an image in encoding enc whose luma follows `gray`: channels offset at random, or random chroma bytes"""
    if enc == "mono8":
        return gray.copy()
    h, w = gray.shape
    if enc.startswith("yuv"):
        out = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        out[..., 1 if enc == "yuv422" else 0] = gray
        return out
    g = gray.astype(np.int32)
    ch = [np.clip(g + rng.integers(-40, 41, (h, w)), 0, 255) for _ in range(3)]
    if enc.endswith("a8"):
        ch.append(rng.integers(0, 256, (h, w)))
    return np.stack(ch, -1).astype(np.uint8)


def _context(camera, enc, w=W, h=H, K=None, **kw):
    u = CAMERAS[camera](w, h)
    ctx = abi.Context(w, h, u.getK() if K is None else K, **kw)
    u.install(ctx)
    ctx.set_input_format(enc)
    return ctx, u


# ---- the exhaustive table ---------------------------------------------------------------------------------------------------
def test_every_colour_through_the_device_hashes_to_opencv():
    """all 2^24 colours as 55 pass-through 640 x 480 rgb8 frames: level 0 of the frames, cut to 2^24 pixels, is cvtColor's table"""
    ctx, _ = _context("pass-through", "rgb8", max_frames=2)
    try:
        n = W * H
        frames = -(-(1 << 24) // n)
        assert frames == 55
        c = np.arange(frames * n, dtype=np.uint32) & 0xFFFFFF
        rgb = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(frames, H, W, 3)
        gray = np.empty(frames * n, np.uint8)
        for k in range(frames):
            ctx.upload_distorted(1, rgb[k])
            lvl0 = ctx.download(1, abi.BUF_IMAGE, 0)
            assert np.array_equal(lvl0, np.round(lvl0)) and lvl0.min() >= 0 and lvl0.max() <= 255
            gray[k * n:(k + 1) * n] = lvl0.reshape(-1).astype(np.uint8)
        assert hashlib.sha256(gray[: 1 << 24].tobytes()).hexdigest() == co.RGB_TABLE_SHA256
    finally:
        ctx.close()


# ---- byte identity with the gray path ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("camera", sorted(CAMERAS))
@pytest.mark.parametrize("enc", ENCODINGS)
def test_every_route_equals_the_gray_path_on_the_converted_image(camera, enc):
    """host, pinned host, a device tensor with an odd pitch, and the ring from host and device memory: every plane of the frame
    equals the frame the MONO8 path builds from cvtColor(raw), and undistort() equals undistort() of cvtColor(raw)"""
    ctx, u = _context(camera, enc, max_frames=8)
    ref, _ = _context(camera, "mono8", max_frames=2)
    try:
        raw = _scene_raw(u.in_w, u.in_h, enc, seed=len(enc) * 7 + len(camera))
        gray = co.to_gray(raw, enc)
        ref.upload_distorted(1, gray)
        want = _planes(ref, 1)
        assert np.array_equal(ctx.undistort(raw), ref.undistort(gray))

        ctx.upload_distorted(1, raw)                                      # pageable host memory
        pinned = torch.from_numpy(np.ascontiguousarray(raw)).pin_memory()
        ctx.upload_distorted(2, pinned.numpy())                           # page-locked host memory, read in place
        ctx.synchronize()
        ctx.upload_distorted(3, _cuda(raw, 3))                            # device, odd pitch
        ctx.stage_reserve(2)
        ctx.stage_put_raw(0, raw)
        ctx.frame_from_stage(4, 0)
        ctx.stage_put_raw(1, _cuda(raw, 5))
        ctx.frame_from_stage(5, 1)
        for fid in (1, 2, 3, 4, 5):
            assert _planes(ctx, fid) == want, fid
    finally:
        ctx.close()
        ref.close()


def test_input_format_persists_across_undistorter_installs():
    ctx, u = _context("pass-through", "bgra8", max_frames=2)
    try:
        CAMERAS["ptam"](W, H).install(ctx)
        raw = _scene_raw(752, 480, "bgra8", seed=5)
        assert ctx.input_format == "bgra8"
        ref, _ = _context("ptam", "mono8", max_frames=2)
        try:
            assert np.array_equal(ctx.undistort(raw), ref.undistort(co.to_gray(raw, "bgra8")))
        finally:
            ref.close()
    finally:
        ctx.close()


# ---- full runs fed colour through the ring ----------------------------------------------------------------------------------
def _run_stream(enc, from_colour, n=20, kf_every=6):
    seq = synth.Sequence(W, H, seed=4321)
    rng = np.random.default_rng(11)
    frames = [seq.render(k) for k in range(n)]
    colour = [_colourize(f[0], enc, rng) for f in frames]
    ctx, _ = _context("pass-through", enc if from_colour else "mono8", K=seq.K, max_frames=8)
    gs = GpuStream(ctx, mode=1, kf_every=kf_every)
    log = []
    try:
        gs.init_gt(0, co.to_gray(colour[0], enc), frames[0][1])
        ctx.stage_reserve(2)
        for k in range(1, n):
            if from_colour:
                ctx.stage_put_raw(k % 2, _cuda(colour[k], k % 2) if k % 3 else colour[k])
            else:
                ctx.stage_put(k % 2, co.to_gray(colour[k], enc))
            gs.step(k, stage_index=k % 2)
            log.append([observe(gs, k, gs._qts.copy() if gs.kf_id == k else None)])
        assert len(gs.keyframe_ids) >= 3                                  # keyframe changes happened
        log.append([{"poses": np.stack(gs.poses).tobytes()}])
    finally:
        ctx.close()
    return log


@pytest.mark.parametrize("enc", ["rgb8", "yuv422"])
def test_stream_fed_colour_through_the_ring_equals_the_gray_run(enc):
    assert_same(_run_stream(enc, True), _run_stream(enc, False))


def _run_group(from_colour, encs=("bgr8", "yuv422_yuy2"), n=12):
    streams, seqs = [], []
    rng = np.random.default_rng(3)
    for s, enc in enumerate(encs):
        seq, fr = _group_sequence(W, H, s, n + 1)
        ctx, _ = _context("pass-through", enc if from_colour else "mono8", K=seq.K, max_frames=8)
        gs = GpuStream(ctx, mode=1, kf_every=GROUP_KF_EVERY, kf_phase=10 + 3 * s)      # a keyframe change in each stream
        colour = [_colourize(f[0], enc, rng) for f in fr]
        gs.init_gt(0, co.to_gray(colour[0], enc), fr[0][1])
        ctx.stage_reserve(2)
        streams.append(gs)
        seqs.append(colour)
    group = GpuStreamGroup(streams)
    log = []
    try:
        for k in range(1, n + 1):
            kf = [gs.next_is_keyframe_change() for gs in streams]
            for gs, colour, enc in zip(streams, seqs, encs):
                if from_colour:
                    gs.ctx.stage_put_raw(k % 2, _cuda(colour[k], 1))
                else:
                    gs.ctx.stage_put(k % 2, co.to_gray(colour[k], enc))
            group.step([k] * len(streams), stage_indices=[k % 2] * len(streams))
            log.append([observe(gs, k, group._qts[i].copy() if kf[i] else None) for i, gs in enumerate(streams)])
    finally:
        for gs in streams:
            gs.ctx.close()
    return log


def test_group_fed_colour_through_the_ring_equals_the_gray_run():
    assert_same(_run_group(True), _run_group(False))


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def _unknown(ctx, fid):
    try:
        ctx.get_pose(fid)
    except abi.LsdGpuError:
        return True
    return False


def test_rejected_calls_change_nothing():
    L = abi.load()
    stream = torch.cuda.current_stream().cuda_stream
    # no undistorter installed
    bare = abi.Context(W, H, np.eye(3, dtype=np.float32), max_frames=2)
    try:
        assert L.lsdgpu_set_input_format(bare.ptr, abi.INPUT_FORMATS["rgb8"][0]) != 0
        bare.stage_reserve(1)
        assert L.lsdgpu_stage_put_raw(bare.ptr, 0, np.zeros(W * H * 3, np.uint8).ctypes.data_as(C.POINTER(C.c_uint8))) != 0
        dev = torch.zeros(W * H * 3, dtype=torch.uint8, device="cuda")
        assert L.lsdgpu_stage_put_raw_device(bare.ptr, 0, dev.data_ptr(), W * 3, stream) != 0
        assert L.lsdgpu_frame_upload_distorted_device_u8(bare.ptr, 7, dev.data_ptr(), W * 3, stream) != 0
        assert _unknown(bare, 7)
    finally:
        bare.close()

    ctx, u = _context("ptam", "rgb8", max_frames=4)
    try:
        raw = _scene_raw(u.in_w, u.in_h, "rgb8", seed=9)
        ctx.stage_reserve(2)
        ctx.stage_put_raw(0, raw)
        ctx.frame_from_stage(1, 0)
        entry = _planes(ctx, 1)
        other = _scene_raw(u.in_w, u.in_h, "rgb8", seed=10)
        d_other = _cuda(other, 0)
        # an unknown format, in C and in Python; the format stays rgb8
        for bad in (-1, 7):
            assert L.lsdgpu_set_input_format(ctx.ptr, bad) != 0
        with pytest.raises(ValueError):
            ctx.set_input_format("bayer_rggb8")
        # a bad ring index, host and device
        for idx in (-1, 2):
            assert L.lsdgpu_stage_put_raw(ctx.ptr, idx, other.ctypes.data_as(C.POINTER(C.c_uint8))) != 0
            assert L.lsdgpu_stage_put_raw_device(ctx.ptr, idx, d_other.data_ptr(), u.in_w * 3, stream) != 0
        # a pitch below in_w * bytes per pixel, and host memory where device memory is needed
        for pitch in (u.in_w, u.in_w * 3 - 1):
            assert L.lsdgpu_stage_put_raw_device(ctx.ptr, 0, d_other.data_ptr(), pitch, stream) != 0
            assert L.lsdgpu_frame_upload_distorted_device_u8(ctx.ptr, 8, d_other.data_ptr(), pitch, stream) != 0
        assert L.lsdgpu_stage_put_raw_device(ctx.ptr, 0, other.ctypes.data, u.in_w * 3, stream) != 0
        torch.cuda.synchronize()
        assert _unknown(ctx, 8)
        ctx.frame_from_stage(2, 0)                                        # entry 0 still holds the first image
        assert _planes(ctx, 2) == entry
        ctx.upload_distorted(3, raw)                                      # and the format is still rgb8
        assert _planes(ctx, 3) == entry
    finally:
        ctx.close()

    # 4:2:2 needs an even input width: the setter, and an install of an odd-width camera while a 4:2:2 format is set
    odd = abi.UndistorterPTAM([0.535719, 0.669567, 0.493249, 0.500409, 0.897966], (641, 481), "crop", (W, H))
    ctx, u = _context("ptam", "yuv422", max_frames=2)
    try:
        with pytest.raises(abi.LsdGpuError):
            odd.install(ctx)
        raw = _scene_raw(u.in_w, u.in_h, "yuv422", seed=12)
        ref, _ = _context("ptam", "mono8", max_frames=2)
        try:
            assert np.array_equal(ctx.undistort(raw), ref.undistort(co.to_gray(raw, "yuv422")))   # the old camera stays
        finally:
            ref.close()
        ctx.set_input_format("mono8")
        odd.install(ctx)
        with pytest.raises(abi.LsdGpuError):
            ctx.set_input_format("yuv422_yuy2")
        assert ctx.input_format == "mono8"
        gray = _scene_raw(641, 481, "mono8", seed=13)
        ref2 = abi.Context(W, H, odd.getK(), max_frames=2)
        try:
            odd.install(ref2)
            assert np.array_equal(ctx.undistort(gray), ref2.undistort(gray))
        finally:
            ref2.close()
    finally:
        ctx.close()
