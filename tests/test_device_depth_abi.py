"""CPU-side checks of depth in and out of device memory (lsdgpu_frame_set_depth_gt_device and its four siblings in
include/lsdgpu.h): the five symbols are declared, exported and bound, the Python layer rejects tensors it cannot pass on before it
calls the library, and hyp_fields() views the hypothesis layout field by field."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTH_SYMBOLS = ("lsdgpu_frame_set_depth_gt_device", "lsdgpu_frame_set_idepth_device", "lsdgpu_depth_set_hypotheses_device",
                 "lsdgpu_depth_download_device", "lsdgpu_keyframe_pack_pointcloud_device")


def test_depth_symbols_declared_exported_and_bound():
    from lsd_slam_b200 import abi, build
    build.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lsdgpu.h")).read(), flags=re.S)
    L = ctypes.CDLL(abi.LIB_PATH)
    bound = {s[0]: s for s in abi.SYMBOLS}
    for name in DEPTH_SYMBOLS:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(L, name), name
        assert name in bound, name
        assert bound[name][2][-1] is ctypes.c_void_p, name            # the caller's stream is the last argument


def test_numpy_depth_callers_do_not_load_torch():
    """the host paths of the methods that now also take tensors still run without torch"""
    code = ("import sys, numpy as np; from lsd_slam_b200 import abi\n"
            "class L:\n"
            "    def __getattr__(self, name): return lambda *a: 0\n"
            "ctx = object.__new__(abi.Context); ctx.L, ctx.ptr, ctx.w, ctx.h, ctx.device = L(), None, 8, 4, 0\n"
            "ctx.set_depth_gt(1, np.ones((4, 8), np.float32)); ctx.set_idepth(1, np.ones((4, 8)), np.ones((4, 8)))\n"
            "ctx.pack_pointcloud(1, 0)\n"
            "dm = abi.DepthMap(ctx); dm.current(); dm.setHypotheses(1, np.zeros((4, 8), abi.HYP_DTYPE))\n"
            "assert 'torch' not in sys.modules, 'torch imported'")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


class _Lib:
    """a library stand-in that fails the test if the Python layer calls it"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} called for an argument the Python layer must reject")


W, H = 64, 48


def _ctx():
    from lsd_slam_b200 import abi
    ctx = object.__new__(abi.Context)
    ctx.L, ctx.ptr, ctx.w, ctx.h, ctx.device, ctx.raw_size = _Lib(), None, W, H, 0, None
    return ctx


@pytest.fixture()
def torch():
    return pytest.importorskip("torch")


def _bad_planes(torch):
    return {
        "cpu tensor": torch.zeros((H, W), dtype=torch.float32),
        "float64": torch.zeros((H, W), dtype=torch.float64),
        "float16": torch.zeros((H, W), dtype=torch.float16),
        "uint8": torch.zeros((H, W), dtype=torch.uint8),
        "stride(1) != 1": torch.zeros((W, H), dtype=torch.float32).t(),
        "every other column": torch.zeros((H, 2 * W), dtype=torch.float32)[:, ::2],
        "wrong shape": torch.zeros((H, W + 1), dtype=torch.float32),
        "transposed shape": torch.zeros((W, H), dtype=torch.float32),
        "3-D": torch.zeros((1, H, W), dtype=torch.float32),
        "flat": torch.zeros(H * W, dtype=torch.float32),
    }


def test_depth_planes_rejected_before_the_call(torch):
    ctx = _ctx()
    good = torch.zeros((H, W), dtype=torch.float32)
    for why, t in _bad_planes(torch).items():
        with pytest.raises(ValueError):
            ctx.set_depth_gt(3, t)
        with pytest.raises(ValueError):
            ctx.set_idepth(3, t, good)
        with pytest.raises(ValueError):
            ctx.set_idepth(3, good, t)


def test_set_idepth_needs_two_tensors(torch):
    ctx = _ctx()
    t = torch.zeros((H, W), dtype=torch.float32)
    with pytest.raises(ValueError, match="both"):
        ctx.set_idepth(3, t, np.zeros((H, W), np.float32))
    with pytest.raises(ValueError, match="both"):
        ctx.set_idepth(3, np.zeros((H, W), np.float32), t)


def test_hypothesis_tensors_rejected_before_the_call(torch):
    from lsd_slam_b200 import abi
    ctx = _ctx()
    dm = abi.DepthMap(ctx)
    n = W * H * 32
    for t in [torch.zeros(n, dtype=torch.uint8),                           # a CPU tensor
              torch.zeros(n // 4, dtype=torch.float32),
              torch.zeros(n // 4, dtype=torch.int32),
              torch.zeros(n - 1, dtype=torch.uint8),
              torch.zeros(n + 32, dtype=torch.uint8),
              torch.zeros(2 * n, dtype=torch.uint8)[::2],
              torch.zeros((32, H, W), dtype=torch.uint8).permute(1, 2, 0)]:
        with pytest.raises(ValueError):
            dm.setHypotheses(1, t)
    for t in [torch.zeros(n, dtype=torch.uint8),                           # a CPU tensor
              torch.zeros(n // 4, dtype=torch.float32),
              torch.zeros(n - 1, dtype=torch.uint8),
              torch.zeros(2 * n, dtype=torch.uint8)[::2],
              torch.zeros((32, H, W), dtype=torch.uint8).permute(1, 2, 0)]:
        with pytest.raises(ValueError):
            dm.current(out=t)


def test_pointcloud_tensors_rejected_before_the_call(torch):
    ctx = _ctx()
    for level in (0, 2):
        n = (W >> level) * (H >> level) * 12
        for t in [torch.zeros(n, dtype=torch.uint8),                       # a CPU tensor
                  torch.zeros(n // 4, dtype=torch.float32),
                  torch.zeros(n - 1, dtype=torch.uint8),
                  torch.zeros(2 * n, dtype=torch.uint8)[::2]]:
            with pytest.raises(ValueError):
                ctx.pack_pointcloud(1, level, out=t)


def test_hyp_fields_are_views_of_the_layout(torch):
    """hyp_fields() on a CPU tensor holding HYP_DTYPE records gives each field without a copy"""
    from lsd_slam_b200 import abi
    rng = np.random.default_rng(7)
    h, w = 6, 10
    rec = np.zeros((h, w), abi.HYP_DTYPE)
    rec["isValid"] = rng.integers(0, 2, (h, w))
    for name in ("blacklisted", "validity_counter"):
        rec[name] = rng.integers(-1000, 1000, (h, w))
    for name in ("nextStereoFrameMinID", "idepth", "idepth_var", "idepth_smoothed", "idepth_var_smoothed"):
        rec[name] = rng.normal(0, 3, (h, w)).astype(np.float32)
    t = torch.from_numpy(rec.view(np.uint8).reshape(h, w, 32).copy())
    f = abi.hyp_fields(t)
    assert sorted(f) == sorted(n for n in abi.HYP_DTYPE.names if n != "_pad")
    for name, v in f.items():
        assert tuple(v.shape) == (h, w), name
        assert v.untyped_storage().data_ptr() == t.untyped_storage().data_ptr(), name
        assert np.array_equal(v.numpy(), rec[name]), name
    f["idepth_smoothed"][2, 3] = 4.5                                       # a view: the record changes
    assert t.view(torch.float32)[2, 3, 6].item() == 4.5
    for bad in (t.reshape(-1), t.view(torch.float32), t.reshape(h, w * 32), t[:, ::2]):
        with pytest.raises(ValueError):
            abi.hyp_fields(bad)
