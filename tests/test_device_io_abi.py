"""CPU-side checks of the device-resident input and output entry points (the *_device calls of include/lsdgpu.h): the five
symbols are declared, exported and bound, and the Python layer rejects tensors it cannot pass on before it calls the library."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVICE_SYMBOLS = ("lsdgpu_frame_upload_device_u8", "lsdgpu_frame_upload_distorted_device_u8", "lsdgpu_stage_put_device",
                  "lsdgpu_frame_download_device", "lsdgpu_map_export_pointcloud_device")


def test_device_symbols_declared_exported_and_bound():
    from lsd_slam_b200 import abi, build
    build.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lsdgpu.h")).read(), flags=re.S)
    L = ctypes.CDLL(abi.LIB_PATH)
    bound = {s[0]: s for s in abi.SYMBOLS}
    for name in DEVICE_SYMBOLS:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(L, name), name
        assert name in bound, name
        assert bound[name][2][-1] is ctypes.c_void_p, name            # the caller's stream is the last argument


def test_numpy_callers_do_not_load_torch():
    code = ("import sys, numpy as np; from lsd_slam_b200 import abi, stream; abi.load(); "
            "assert 'torch' not in sys.modules, 'torch imported'")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


class _Lib:
    """a library stand-in that fails the test if the Python layer calls it"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} called for an argument the Python layer must reject")


def _ctx(w=64, h=48):
    from lsd_slam_b200 import abi
    ctx = object.__new__(abi.Context)
    ctx.L, ctx.ptr, ctx.w, ctx.h, ctx.device, ctx.raw_size = _Lib(), None, w, h, 0, (80, 60)
    return ctx


@pytest.fixture()
def torch():
    return pytest.importorskip("torch")


@pytest.mark.parametrize("call", ["upload", "stage_put", "upload_distorted"])
def test_image_tensors_rejected_before_the_call(torch, call):
    ctx = _ctx()
    h, w = (60, 80) if call == "upload_distorted" else (48, 64)
    f = (lambda t: getattr(ctx, call)(3, t))
    bad = {
        "cpu tensor": torch.zeros((h, w), dtype=torch.uint8),
        "float32": torch.zeros((h, w), dtype=torch.float32),
        "int16": torch.zeros((h, w), dtype=torch.int16),
        "stride(1) != 1": torch.zeros((w, h), dtype=torch.uint8).t(),
        "every other column": torch.zeros((h, 2 * w), dtype=torch.uint8)[:, ::2],
        "wrong shape": torch.zeros((h, w + 1), dtype=torch.uint8),
        "transposed shape": torch.zeros((w, h), dtype=torch.uint8),
        "3-D": torch.zeros((1, h, w), dtype=torch.uint8),
    }
    for why, t in bad.items():
        with pytest.raises(ValueError):
            f(t)


def test_distorted_upload_needs_an_undistorter(torch):
    ctx = _ctx()
    ctx.raw_size = None
    with pytest.raises(ValueError, match="undistorter"):
        ctx.upload_distorted(1, torch.zeros((60, 80), dtype=torch.uint8))


def test_output_tensors_rejected_before_the_call(torch):
    from lsd_slam_b200 import abi
    ctx = _ctx()
    for what, t in [(abi.BUF_IMAGE, torch.zeros((48, 64), dtype=torch.float32)),          # a CPU tensor
                    (abi.BUF_IMAGE, torch.zeros((48, 64), dtype=torch.float64)),
                    (abi.BUF_IMAGE, torch.zeros((48, 63), dtype=torch.float32)),          # too small
                    (abi.BUF_IMAGE, torch.zeros((64, 48), dtype=torch.float32).t()),      # not contiguous
                    (abi.BUF_GRADIENTS, torch.zeros((48, 64), dtype=torch.float32)),
                    (abi.BUF_GOODMASK, torch.zeros((24, 32), dtype=torch.float32))]:
        with pytest.raises(ValueError):
            ctx.download(1, what, 0, out=t)
    c2w = np.zeros((1, 7), np.float32)
    c2w[0, 3] = 1
    for t in [torch.zeros((100, 4), dtype=torch.float32),                                  # a CPU tensor
              torch.zeros((100, 4), dtype=torch.float64),
              torch.zeros((100, 3), dtype=torch.float32),
              torch.zeros(400, dtype=torch.float32),
              torch.zeros((4, 100), dtype=torch.float32).t()]:
        with pytest.raises(ValueError):
            ctx.export_pointcloud([0], c2w, filter=abi.CloudFilter(1, 1, 5, 1), out=t)
