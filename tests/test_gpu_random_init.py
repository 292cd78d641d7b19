"""DepthMap::initializeRandomly on the device (lsdgpu_depth_init_random) against the reference's own initializeRandomly
(DepthMap.cpp:883-916, compiled unmodified into oracle/_ref/liblsd_ref.so), which draws from this test process's libc rand().
Both sides start from the same depth map (the device's, copied into the reference's currentDepthMap), so every one of the w*h
cells is compared bit for bit -- border cells and the fields an unselected cell keeps included -- and so are Frame::setDepth's
idepth / idepthVar pyramid and numPoints.  The state the call returns must continue the stream exactly as rand() continues it in
the reference process.  Where oracle/_ref is not built the strict-IEEE C restatement of the oracle takes the reference's place
(tests/test_ref_pin.py pins the two to each other)."""
import contextlib
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import IDENT_QTS, GpuStream
from oracle import pyoracle as po
from oracle import ref_build

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "ref" if ref_build.built() else False
SIZES = {0: 8, 1: 32, 2: 64, 3: 128, 4: 256}        # initstate() buffer size of each state type
FIELDS = [f for f in abi.HYP_DTYPE.names if f != "_pad"]
N_NEXT = 1000

_libc = C.CDLL(None)
_libc.initstate.restype = C.c_void_p
_libc.initstate.argtypes = [C.c_uint, C.c_void_p, C.c_size_t]
_libc.setstate.restype = C.c_void_p
_libc.setstate.argtypes = [C.c_void_p]
_libc.rand.restype = C.c_int


@contextlib.contextmanager
def libc_stream(seed, t):
    """rand() of this process seeded in state type t (type 3: what srand(seed) gives); the previous state is restored after"""
    buf = (C.c_int32 * 64)()
    old = _libc.initstate(seed, buf, SIZES[t])
    try:
        yield
    finally:
        _libc.setstate(old)


def libc_draws(n):
    return np.array([_libc.rand() for _ in range(n)], np.int32)


def cells_differing(a, b):
    """number of cells whose fields (all but the padding) differ in any bit"""
    d = np.zeros(a.shape, bool)
    for f in FIELDS:
        x, y = np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f])
        d |= (x.view(np.uint8).reshape(x.shape + (-1,)) != y.view(np.uint8).reshape(y.shape + (-1,))).any(-1)
    return int(d.sum())


class RefSide:
    """the reference's DepthMap with the device map's current state copied in, and its frames"""

    def __init__(self, w, h, K, prior, min_grad=None):
        po.set_globals(fast=REF, **({} if min_grad is None else {"minUseGrad": float(min_grad)}))
        self.K = K
        self.dm = po.DepthMap(w, h, K, fast=REF)
        self.dm.set_current(prior)
        self.frames = []

    def init_random(self, fid, img):
        f = po.Frame(fid, img, self.K, fast=REF)
        self.frames.append(f)
        self.dm.initializeRandomly(f)
        return f

    def close(self):
        po.set_globals(fast=REF)


def check_frame_depth(ctx, fid, of):
    """Frame::setDepth (DepthMap.cpp:915): the idepth / idepthVar pyramid and numPoints"""
    for lvl in range(abi.LEVELS):
        for what, ref in ((abi.BUF_IDEPTH, of.idepth(lvl)), (abi.BUF_IDEPTH_VAR, of.idepthVar(lvl))):
            g = ctx.download(fid, what, lvl)
            assert np.array_equal(g.view(np.uint32), np.ascontiguousarray(ref).view(np.uint32)), (fid, what, lvl)
    assert ctx.depth_stats(fid)[1] == of.L.lsdo_frame_numPoints(of.ptr)


def run_case(w, h, seed, t, k, min_grad=None, scene_seed=1234, mapped_before=False, calls=1):
    seq = synth.Sequence(w, h, seed=scene_seed)
    frames = [seq.render(i)[0] for i in range(calls + 2)]
    ctx = abi.Context(w, h, seq.K, max_frames=6)
    try:
        if min_grad is not None:
            ctx.set_globals(minUseGrad=float(min_grad))
        gdm = abi.DepthMap(ctx)
        first = 0
        if mapped_before:                          # a keyframe mapped with one frame: every field of the map holds something
            img0, d0 = seq.render(0)
            ctx.upload(0, img0)
            ctx.set_depth_gt(0, d0)
            gdm.initializeFromGTDepth(0)
            ctx.upload(1, frames[1])
            ctx.set_pose(1, np.concatenate([seq.frame_to_ref_qt(1), [1.0]]), 0, 0.0)
            gdm.updateKeyframe([1])
            first = 2
        prior = gdm.current()
        if mapped_before:
            assert (prior["isValid"] > 0).sum() > 1000
        st = abi.RandState.from_seed(seed, t)
        st.advance(k, values=False)
        ref = RefSide(w, h, seq.K, prior, min_grad)
        try:
            with libc_stream(seed, t):
                libc_draws(k)
                for c in range(calls):
                    fid = first + c
                    of = ref.init_random(fid, frames[fid])
                    ctx.upload(fid, frames[fid])
                    st = gdm.initializeRandomly(fid, st)
                    want = ref.dm.current()
                    got = gdm.current()
                    assert gdm.activeKeyFrame() == fid
                    assert cells_differing(got, want) == 0, (w, h, seed, t, k, c)
                    assert gdm.last_draws == int((want["isValid"][1:-1, 1:-1] > 0).sum()) > 0     # interior: valid == drawn
                    check_frame_depth(ctx, fid, of)
                nxt = libc_draws(N_NEXT)
            assert np.array_equal(st.copy().advance(N_NEXT), nxt)
        finally:
            ref.close()
        return gdm.last_draws
    finally:
        ctx.close()


@pytest.mark.parametrize("w,h", [(320, 240), (640, 480), (1280, 1024), (336, 240)], ids=lambda v: str(v))
@pytest.mark.parametrize("seed,k", [(1, 0), (1234567, 0), (1, 12345)], ids=["seed1", "seed1234567", "seed1_after12345"])
def test_random_init_matches_reference(w, h, seed, k):
    run_case(w, h, seed, 3, k)


@pytest.mark.parametrize("t", range(5))
def test_random_init_every_state_type(t):
    run_case(320, 240, 1234567, t, 12345)
    run_case(640, 480, 7, t, 0)


@pytest.mark.parametrize("min_grad", [3, 12])
def test_random_init_min_use_grad(min_grad):
    n = run_case(640, 480, 1, 3, 0, min_grad=min_grad)
    n5 = run_case(640, 480, 1, 3, 0)
    assert (n > n5) if min_grad < 5 else (n < n5)


def test_random_init_over_a_mapped_keyframe_twice():
    """the map held a mapped keyframe: border cells and the fields of unselected cells keep what it held; then a second random
    start continues the same stream"""
    run_case(320, 240, 99, 3, 5, mapped_before=True, calls=2)
    run_case(640, 480, 4242, 4, 31, mapped_before=True, calls=2)


def test_stream_init_random_matches_set_hypotheses_start():
    """GpuStream.init_random and 30 tracked and mapped frames (keyframe every 10) equal the same stream started through
    setHypotheses with the reference's own draws"""
    seq = synth.Sequence(320, 240, seed=77)
    imgs = [seq.render(i)[0] for i in range(31)]
    ctx_a = abi.Context(seq.w, seq.h, seq.K, max_frames=8)
    ctx_b = abi.Context(seq.w, seq.h, seq.K, max_frames=8)
    try:
        a, b = GpuStream(ctx_a, kf_every=10), GpuStream(ctx_b, kf_every=10)
        st = a.init_random(0, imgs[0], abi.RandState.from_seed(2024))

        ref = RefSide(seq.w, seq.h, seq.K, abi.DepthMap(ctx_b).current())
        try:
            with libc_stream(2024, 3):
                ref.init_random(0, imgs[0])
                nxt = libc_draws(N_NEXT)
            hyp = ref.dm.current().copy()
        finally:
            ref.close()
        assert np.array_equal(st.copy().advance(N_NEXT), nxt)
        ctx_b.upload(0, imgs[0])
        b.map.setHypotheses(0, hyp, reactivated=False, do_set_depth=True)
        b.kf_id, b.keyframe_ids, b.keyframe_cam_to_world = 0, [0], [IDENT_QTS.copy()]
        assert cells_differing(a.map.current(), b.map.current()) == 0
        for i in range(1, 31):
            pa, pb = a.step(i, imgs[i]), b.step(i, imgs[i])
            assert np.array_equal(pa, pb), i
        assert a.kf_id == b.kf_id and a.kf_id != 0
        assert cells_differing(a.map.current(), b.map.current()) == 0
        for lvl in range(abi.LEVELS):
            assert np.array_equal(ctx_a.download(a.kf_id, abi.BUF_IDEPTH, lvl).view(np.uint32),
                                  ctx_b.download(b.kf_id, abi.BUF_IDEPTH, lvl).view(np.uint32))
    finally:
        ctx_a.close()
        ctx_b.close()


def test_rejected_calls_change_nothing():
    seq = synth.Sequence(320, 240, seed=5)
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=4)
    try:
        gdm = abi.DepthMap(ctx)
        ctx.upload(0, seq.render(0)[0])
        ctx.upload(1, seq.render(1)[0])
        gdm.initializeRandomly(0, abi.RandState.from_seed(3))
        ctx.minimize(1)
        map0, id0 = gdm.current(), ctx.download(0, abi.BUF_IDEPTH, 0)
        good = abi.RandState.from_seed(11, 2)
        bad_type, bad_rear, bad_rear0 = good.copy(), good.copy(), abi.RandState.from_seed(11, 0)
        bad_type.type = 5
        bad_rear.rear = 15
        bad_rear0.rear = 1
        for fid, st, what in ((7, good, "unknown"), (1, good, "minimized"), (0, bad_type, "bad state"), (0, bad_rear, "bad state"),
                              (0, bad_rear0, "bad state")):
            before = bytes(st)
            n = C.c_int64(-1)
            rc = ctx.L.lsdgpu_depth_init_random(ctx.ptr, fid, C.byref(st), C.byref(n))
            assert rc != 0, what
            msg = ctx.L.lsdgpu_last_error(ctx.ptr).decode()
            assert ("minimized" in msg) == (what == "minimized"), msg
            assert bytes(st) == before and n.value == -1
            assert gdm.activeKeyFrame() == 0
            assert cells_differing(gdm.current(), map0) == 0
            assert np.array_equal(ctx.download(0, abi.BUF_IDEPTH, 0).view(np.uint32), id0.view(np.uint32))
    finally:
        ctx.close()


# ---- the C++ adapter: tests/native/host_random_init.cpp ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    exe = tmp_path_factory.mktemp("random_init") / "host_random_init"
    here = os.path.dirname(build.HOST_OUT)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(ROOT, "tests", "native", "host_random_init.cpp"),
                        "-L" + here, "-Wl,-rpath," + here, "-l:liblsdgpu_host.so", "-l:liblsdgpu.so", "-pthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.mark.parametrize("seed,k,t,size", [(1, 0, 3, 0), (1234567, 12345, 3, 0), (99, 777, 1, 32), (5, 3, 0, 8)],
                         ids=["srand1", "srand1234567_after12345", "type1", "type0"])
def test_adapter_initialize_randomly(driver, tmp_path, seed, k, t, size):
    """srand(seed) (or initstate), k rand() calls, DepthMap::initializeRandomly of lsd_host.h: the process's next rand() values are
    the reference's, and the map is what the ABI call makes"""
    seq = synth.Sequence(640, 480, seed=31)
    img = seq.render(0)[0]
    with open(tmp_path / "img.bin", "wb") as f:
        f.write(np.array([seq.w, seq.h], np.int32).tobytes() + np.asarray(seq.K, np.float32).tobytes() + img.tobytes())
    r = subprocess.run([driver, str(tmp_path / "img.bin"), str(tmp_path / "out.bin"), str(seed), str(k), str(size)],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    raw = (tmp_path / "out.bin").read_bytes()
    nxt = np.frombuffer(raw[:4 * N_NEXT], np.int32)
    adapter_map = np.frombuffer(raw[4 * N_NEXT:], abi.HYP_DTYPE).reshape(seq.h, seq.w)

    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=4)
    try:
        gdm = abi.DepthMap(ctx)
        prior = gdm.current()
        ctx.upload(0, img)
        st = abi.RandState.from_seed(seed, t)
        st.advance(k, values=False)
        gdm.initializeRandomly(0, st)
        assert cells_differing(adapter_map, gdm.current()) == 0
    finally:
        ctx.close()

    ref = RefSide(seq.w, seq.h, seq.K, prior)
    try:
        with libc_stream(seed, t):
            libc_draws(k)
            ref.init_random(0, img)
            want = libc_draws(N_NEXT)
    finally:
        ref.close()
    assert np.array_equal(nxt, want)
    assert cells_differing(adapter_map, ref.dm.current()) == 0
