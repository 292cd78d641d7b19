"""The C++ adapter's FrameMemory with a device record limit (FrameMemory::setMaxDeviceRecords): pruneActiveFrames offloads the
minimized records beyond the limit to host memory, and every later call that needs such a frame (setFromExistingKF, the Sim3 and
permaRef constraint calls) serves it from there.  tests/native/host_slam_mode_offload.cpp runs host_slam_mode.cpp's SLAM-mode script
with the limit, inline and with the constraint calls on a second thread, and its outputs are compared bit for bit with the same
calls made through abi.py on a context that never minimizes (the harness of test_gpu_host_slam_mode.py, which that module holds to
the reference)."""
import os
import subprocess

import pytest

from tests.test_gpu_host_slam_mode import REACTIVATE, AbiMirror, Run, assert_same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    exe = tmp_path_factory.mktemp("slam_mode_offload") / "host_slam_mode_offload"
    here = os.path.dirname(build.HOST_OUT)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe),
                        os.path.join(ROOT, "tests", "native", "host_slam_mode_offload.cpp"),
                        "-L" + here, "-Wl,-rpath," + here, "-l:liblsdgpu_host.so", "-l:liblsdgpu.so", "-pthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


def _memory(run):
    """the MEMORY lines of a run: (n_device, device_bytes, n_host, host_bytes) before the re-activation, if any, then at the end"""
    return [tuple(int(v) for v in ln[1:]) for ln in run.lines if ln[0] == "MEMORY"]


def test_setFromExistingKF_on_an_offloaded_keyframe(driver, tmp_path, seq_small, frames_small):
    """two active frames and no minimized record in device memory: keyframe 5 is re-activated from host memory by
    setFromExistingKF(Frame*) and tracked and mapped on; the permaRef and Sim3 calls read offloaded keyframes"""
    react = ["--reactivate", str(REACTIVATE[0]), str(REACTIVATE[1])]
    run = Run(driver, tmp_path, seq_small, frames_small, *react, "--prune", "2", "--device-records", "0")
    assert ["REACTIVATE", str(REACTIVATE[1]), "0"] in run.lines
    before, end = _memory(run)
    assert before[0] == 0 and before[2] >= 1, before      # keyframe 5 is minimized, so its record is in host memory
    assert end[0] == 0 and end[2] >= 2, end
    m = AbiMirror(seq_small, frames_small, run, react=REACTIVATE)
    assert_same(run.main, m.main, "tracking and mapping")
    assert_same(run.cons, m.cons, "constraint calls")


def test_constraint_thread_with_offloaded_keyframes(driver, tmp_path, seq_small, frames_small):
    """the constraint calls on a second thread while the main thread prunes and offloads.  Three active frames: the two frames a
    constraint call holds and the active keyframe, so that pruning always finds a frame to minimize; which one it picks depends on
    the threads' timing, and none of the outputs does."""
    run = Run(driver, tmp_path, seq_small, frames_small, "--threads", "--prune", "3", "--device-records", "0")
    (end,) = _memory(run)
    assert end[0] == 0 and end[2] >= 1, end
    m = AbiMirror(seq_small, frames_small, run)
    assert_same(run.main, m.main, "tracking and mapping")
    assert_same(run.cons, m.cons, "constraint calls")
