"""The C++ adapter fed colour camera images (tests/native/host_colour_input.cpp): getUndistorterForFile, install,
DeviceContext::setInputFormat, Undistorter::undistort and Frame(.., raw, /*distorted=*/true) give the same undistorted image and
the same frame as abi.py's Context.set_input_format, undistort and upload_distorted on the same calibration and raw image."""
import os
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import colour_input_oracle as co
from tests.golden import make_golden_ref_pin_undistort as mg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEXT = dict(mg.cases())
LEVELS = 5


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    exe = tmp_path_factory.mktemp("colour_input") / "host_colour_input"
    here = os.path.dirname(build.HOST_OUT)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(ROOT, "tests", "native", "host_colour_input.cpp"),
                        "-L" + here, "-Wl,-rpath," + here, "-l:liblsdgpu_host.so", "-l:liblsdgpu.so", "-pthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.mark.parametrize("enc", ["mono8", "rgb8", "bgra8", "yuv422"])
@pytest.mark.parametrize("case", ["raw752_full", "w0_same"])
def test_adapter_equals_the_abi(driver, tmp_path, case, enc):
    u = abi.UndistorterPTAM(*mg.parse(TEXT[case]))
    fmt, bpp = co.FORMATS[enc]
    raw = co.random_raw(u.in_w, u.in_h, enc, seed=fmt + 17)
    (tmp_path / "calib.cfg").write_text(TEXT[case])
    raw.tofile(tmp_path / "raw.bin")
    r = subprocess.run([driver, str(tmp_path / "calib.cfg"), str(bpp), str(fmt), str(tmp_path / "raw.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(tmp_path / "out.bin", np.uint8)

    ctx = abi.Context(u.out_w, u.out_h, u.getK(), max_frames=2)
    try:
        u.install(ctx)
        ctx.set_input_format(enc)
        want = [ctx.undistort(raw).tobytes()]
        ctx.upload_distorted(1, raw)
        want += [ctx.download(1, abi.BUF_IMAGE, lvl).tobytes() for lvl in range(LEVELS)]
        want.append(ctx.download(1, abi.BUF_MAXGRAD, 0).tobytes())
    finally:
        ctx.close()
    assert out.tobytes() == b"".join(want)
