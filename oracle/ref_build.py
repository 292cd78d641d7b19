"""oracle/ref_build.py -- recipe for oracle/_ref/: the reference's OWN hot-path sources compiled where they lie.

TEST INFRASTRUCTURE.  Compiles, UNMODIFIED and straight from /root/reference (nothing is copied into this repo),

    lsd_slam_core/src/DepthEstimation/DepthMap.cpp, DepthMapPixelHypothesis.cpp
    lsd_slam_core/src/Tracking/SE3Tracker.cpp, Sim3Tracker.cpp, TrackingReference.cpp      (+ LGSX.h)
    lsd_slam_core/src/DataStructures/Frame.cpp, FrameMemory.cpp, FramePoseStruct.cpp
    lsd_slam_core/src/util/settings.cpp, SophusUtil.cpp                                   (+ globalFuncs.h, IndexThreadReduce.h)
    lsd_slam_core/src/util/Undistorter.cpp                                                (UndistorterPTAM; UndistorterOpenCV
                                                                                           compiles but is never constructed)
    lsd_slam_core/thirdparty/Sophus/sophus/{so3,se3,rxso3,sim3}.hpp                       (vendored, header only)

against the stand-in headers in oracle/ref_shim/ (a fixed-size Eigen 3.2 subset, Boost.Thread -> std::, OpenCV debug
images and K storage, empty KeyFrameGraph / g2o declarations, OpenCV calib3d entry points that abort if reached) plus oracle/ref_driver.cpp, which exports the reference's classes under
the C names of oracle/lsd_oracle.h.  The reference's own build system (rosbuild + cmake + Eigen3 + SuiteSparse + X11 +
dynamic_reconfigure, lsd_slam_core/CMakeLists.txt:3-33) cannot run in this image; this is the short recipe instead.

Outputs (git-ignored, shipped to the GPU box with the snapshot):
    oracle/_ref/liblsd_ref.so        scalar code path (no ENABLE_SSE), strict IEEE fp32: the PARITY pin of the oracle
    oracle/_ref/liblsd_ref_sse.so    the stock configuration: -DENABLE_SSE -O3 (CMakeLists.txt:11,37-43), x86-64-v3 instead
                                     of -march=native because the binary is built here and runs on another CPU
    oracle/_ref/test_{so3,se3,sim3,rxso3}   the vendored Sophus test programs (thirdparty/Sophus/sophus/test_*.cpp)
    oracle/_ref/BUILD_INFO.json

/root/reference exists only in the build container: on the GPU box this script is a no-op and the prebuilt files are used.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/lsd_slam_core"
OUT = os.path.join(HERE, "_ref")
SHIM = os.path.join(HERE, "ref_shim")

SOURCES = [
    "src/DepthEstimation/DepthMap.cpp", "src/DepthEstimation/DepthMapPixelHypothesis.cpp",
    "src/Tracking/SE3Tracker.cpp", "src/Tracking/Sim3Tracker.cpp", "src/Tracking/TrackingReference.cpp",
    "src/DataStructures/Frame.cpp", "src/DataStructures/FrameMemory.cpp", "src/DataStructures/FramePoseStruct.cpp",
    "src/util/settings.cpp", "src/util/SophusUtil.cpp", "src/util/Undistorter.cpp",
]
SOPHUS_TESTS = ["so3", "se3", "sim3", "rxso3"]

COMMON = ["-std=gnu++17", "-DNDEBUG", "-fPIC", "-w", "-pthread",
          f"-I{SHIM}", f"-I{REF}/src", f"-I{REF}/thirdparty/Sophus", f"-I{HERE}"]
FLAVOURS = {
    # Release build type (CMakeLists.txt:11) => NDEBUG => enablePrintDebugInfo == false (util/settings.h:44-48)
    "liblsd_ref.so": ["-O2", "-ffp-contract=off", "-fno-fast-math", "-msse2"],
    "liblsd_ref_sse.so": ["-O3", "-DENABLE_SSE", "-march=x86-64-v3", "-msse4.1", "-msse3", "-msse2", "-msse"],
    # the scalar build as a g++ < 6 toolchain resolves the reference's unqualified sqrt() / tan() / atan() calls (see
    # ref_shim/opencv2)
    "liblsd_ref_legacy_math.so": ["-O2", "-ffp-contract=off", "-fno-fast-math", "-msse2", "-DLSD_REF_SHIM_LEGACY_MATH"],
}


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "src"))


def built() -> bool:
    return all(os.path.exists(os.path.join(OUT, n)) for n in FLAVOURS)


def _deps():
    d = [os.path.join(HERE, "ref_driver.cpp"), os.path.join(HERE, "lsd_oracle.h"), os.path.abspath(__file__)]
    for root, _, files in os.walk(SHIM):
        d += [os.path.join(root, f) for f in files]
    return d


def needs_build() -> bool:
    if not built():
        return True
    t = min(os.path.getmtime(os.path.join(OUT, n)) for n in FLAVOURS)
    return any(os.path.getmtime(p) > t for p in _deps())


def build(force: bool = False, verbose: bool = False) -> bool:
    """Returns True when oracle/_ref holds both libraries afterwards."""
    if not available():
        return built()
    if not force and not needs_build():
        return True
    os.makedirs(OUT, exist_ok=True)
    jobs = []
    for name, flags in FLAVOURS.items():
        cmd = ["g++"] + COMMON + flags + ["-shared", "-o", os.path.join(OUT, name)] + \
              [os.path.join(REF, s) for s in SOURCES] + [os.path.join(HERE, "ref_driver.cpp")]
        jobs.append((name, cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for t in SOPHUS_TESTS:
        cmd = ["g++", "-std=gnu++17", "-O1", "-w", f"-I{SHIM}", f"-I{REF}/thirdparty/Sophus",
               os.path.join(REF, "thirdparty/Sophus/sophus", f"test_{t}.cpp"), "-o", os.path.join(OUT, f"test_{t}")]
        jobs.append((f"test_{t}", cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ok = True
    for name, cmd, p in jobs:
        out, _ = p.communicate()
        if p.returncode != 0:
            ok = False
            sys.stderr.write(f"[ref_build] {name} failed:\n{out}\n")
        elif verbose:
            print(f"[ref_build] {name} ok")
    if not ok:
        raise RuntimeError("oracle/_ref build failed")
    # the vendored Sophus test programs, compiled unmodified against ref_shim/Eigen, must pass before anything built against
    # that shim is used (tests/golden/make_golden.py records the reference's outputs from these libraries)
    for t in SOPHUS_TESTS:
        r = subprocess.run([os.path.join(OUT, f"test_{t}")], capture_output=True, text=True, timeout=120)
        if r.returncode != 0 or "passed" not in r.stderr or "failed" in r.stderr:
            raise RuntimeError(f"[ref_build] Sophus test_{t} fails on oracle/ref_shim:\n{r.stderr[-500:]}")
        if verbose:
            print(f"[ref_build] Sophus test_{t} passed")
    info = {"reference": REF, "sources": SOURCES, "flags": {k: COMMON[:5] + v for k, v in FLAVOURS.items()},
            "gxx": subprocess.run(["g++", "--version"], capture_output=True, text=True).stdout.splitlines()[0],
            "shim": "oracle/ref_shim (Eigen 3.2 fixed-size subset, Boost.Thread -> std, OpenCV debug images and Undistorter stand-ins)",
            "sophus_tests": SOPHUS_TESTS}
    with open(os.path.join(OUT, "BUILD_INFO.json"), "w") as f:
        json.dump(info, f, indent=1)
    return True


if __name__ == "__main__":
    print("reference available:", available())
    print("built:", build(force="--force" in sys.argv, verbose=True))
