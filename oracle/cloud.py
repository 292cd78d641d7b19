"""oracle/cloud.py -- TEST INFRASTRUCTURE for the map point-cloud export (lsdgpu_map_export_pointcloud).

Two CPU implementations of lsd_slam_viewer's KeyFrameDisplay::refreshPC + flushPC (KeyFrameDisplay.cpp:106-222, :269-339):

    oracle/liblsd_oracle_cloud.so   the C restatement oracle/lsd_oracle_cloud.inc (strict IEEE fp32, no FMA contraction); built
                                    everywhere, and what the GPU tests compare against
    oracle/_ref/libviewer_ref.so    the viewer's OWN sources, compiled unmodified where they lie (only where the reference tree
                                    exists; the built file travels with the working tree like the rest of oracle/_ref):
                                        lsd_slam_viewer/src/KeyFrameDisplay.cpp, KeyFrameGraphDisplay.cpp, settings.cpp
                                        lsd_slam_viewer/thirdparty/Sophus (header only; identical to the core's vendored copy)
                                    against oracle/ref_shim (GL / QGLViewer / ROS stand-ins, the keyframeMsg structs, Eigen 3.2
                                    subset, Boost.Thread -> std::) plus oracle/ref_viewer_driver.cpp

tests/golden/make_golden_cloud.py records the viewer's outputs as digests (tests/golden/cloud_viewer.json), so that the restatement
stays pinned to the viewer where the reference tree is absent.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liblsd_oracle_cloud.so")
VIEWER = "/root/reference/lsd_slam_viewer"
VIEWER_SO = os.path.join(HERE, "_ref", "libviewer_ref.so")
SHIM = os.path.join(HERE, "ref_shim")
VIEWER_SOURCES = ["src/KeyFrameDisplay.cpp", "src/KeyFrameGraphDisplay.cpp", "src/settings.cpp"]
# the parity flavour of oracle/ref_build.py: strict IEEE fp32 on SSE2, nothing contracted
VIEWER_FLAGS = ["-std=gnu++17", "-DNDEBUG", "-fPIC", "-w", "-pthread", "-O2", "-ffp-contract=off", "-fno-fast-math", "-msse2"]

PLY_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4")])
VERTEX_DTYPE = np.dtype([("point", "<f4", (3,)), ("color", "u1", (4,))])
INPUT_POINT_DENSE = np.dtype([("idepth", "<f4"), ("idepth_var", "<f4"), ("color", "u1", (4,))])


def viewer_available() -> bool:
    return os.path.isdir(os.path.join(VIEWER, "src"))


def build(force: bool = False) -> None:
    """the restatement always; the viewer's library where the reference tree exists"""
    src = os.path.join(HERE, "lsd_oracle_cloud.inc")
    if force or not os.path.exists(ORACLE_SO) or os.path.getmtime(src) > os.path.getmtime(ORACLE_SO):
        subprocess.run(["gcc", "-std=gnu11", "-fPIC", "-shared", "-Wall", "-O2", "-ffp-contract=off", "-fno-fast-math", "-msse2",
                        "-x", "c", src, "-o", ORACLE_SO, "-lm"], check=True, capture_output=True)
    if viewer_available() and (force or not os.path.exists(VIEWER_SO)):
        os.makedirs(os.path.dirname(VIEWER_SO), exist_ok=True)
        cmd = ["g++"] + VIEWER_FLAGS + [f"-I{SHIM}", f"-I{VIEWER}/src", f"-I{VIEWER}/thirdparty/Sophus", "-shared", "-o", VIEWER_SO] + \
              [os.path.join(VIEWER, s) for s in VIEWER_SOURCES] + [os.path.join(HERE, "ref_viewer_driver.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle/_ref/libviewer_ref.so build failed:\n" + r.stdout + r.stderr)


def viewer_built() -> bool:
    return os.path.exists(VIEWER_SO)


_libs: dict = {}


def _lib(name):
    if name not in _libs:
        if name == "oracle":
            build()
            L = C.CDLL(ORACLE_SO)
            L.lsdo_cloud_keyframe.restype = C.c_int
            L.lsdo_cloud_keyframe.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 4 + [C.c_void_p, C.c_float, C.c_float, C.c_int,
                                                                                                 C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        else:
            if not viewer_built():
                build()
            L = C.CDLL(VIEWER_SO)
            L.lsdv_ref_keyframe.restype = C.c_int
            L.lsdv_ref_keyframe.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 4 + [C.c_void_p, C.c_float, C.c_float, C.c_int,
                                                                                               C.c_char_p, C.c_void_p, C.c_void_p,
                                                                                               C.POINTER(C.c_int), C.POINTER(C.c_int)]
            L.lsdv_ref_map_ply.restype = C.c_int
            L.lsdv_ref_map_ply.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 4 + [C.c_void_p, C.c_float, C.c_float,
                                                                                                        C.c_int, C.c_char_p]
        _libs[name] = L
    return _libs[name]


def _filter(f):
    f = dict(f or {})
    return float(f.get("scaledDepthVarTH", 1.0)), float(f.get("absDepthVarTH", 1.0)), int(f.get("minNearSupport", 5))


def keyframe(pc: np.ndarray, cam, camToWorld, filt=None, impl: str = "oracle"):
    """one keyframe: pc = (h, w) INPUT_POINT_DENSE records, cam = (fx, fy, cx, cy) of its level, camToWorld = 7 floats.
    Returns (vertex array, ply array, totalPoints, displayedPoints); impl = "oracle" (C restatement) or "viewer" (viewer's code)."""
    pc = np.ascontiguousarray(pc, INPUT_POINT_DENSE)
    h, w = pc.shape
    c2w = np.ascontiguousarray(camToWorld, np.float32).reshape(7)
    s, a, m = _filter(filt)
    vert = np.zeros(max(1, (w - 2) * (h - 2)), VERTEX_DTYPE)
    ply = np.zeros(max(1, (w - 2) * (h - 2)), PLY_DTYPE)
    total, shown = C.c_int(0), C.c_int(0)
    fx, fy, cx, cy = (float(np.float32(v)) for v in cam)
    if impl == "oracle":
        n = _lib("oracle").lsdo_cloud_keyframe(pc.ctypes.data, w, h, fx, fy, cx, cy, c2w.ctypes.data, s, a, m,
                                               vert.ctypes.data, ply.ctypes.data, C.byref(total))
        shown.value = n
    else:
        with tempfile.TemporaryDirectory() as d:
            n = _lib("viewer").lsdv_ref_keyframe(pc.ctypes.data, w, h, fx, fy, cx, cy, c2w.ctypes.data, s, a, m,
                                                 os.path.join(d, "flush.bin").encode(), vert.ctypes.data, ply.ctypes.data,
                                                 C.byref(total), C.byref(shown))
        if n < 0:
            raise RuntimeError("viewer driver failed")
    return vert[:n].copy(), ply[:n].copy(), total.value, shown.value


def viewer_map_ply(pcs: np.ndarray, cam, camToWorld, filt=None) -> bytes:
    """the bytes of the pc.ply the viewer writes for keyframes pcs (n, h, w) with camToWorld (n, 7), all flushed"""
    pcs = np.ascontiguousarray(pcs, INPUT_POINT_DENSE)
    n, h, w = pcs.shape
    c2w = np.ascontiguousarray(camToWorld, np.float32).reshape(n, 7)
    s, a, m = _filter(filt)
    fx, fy, cx, cy = (float(np.float32(v)) for v in cam)
    with tempfile.TemporaryDirectory() as d:
        _lib("viewer").lsdv_ref_map_ply(n, pcs.ctypes.data, w, h, fx, fy, cx, cy, c2w.ctypes.data, s, a, m, d.encode())
        with open(os.path.join(d, "pc.ply"), "rb") as f:
            return f.read()


def make_case(seed: int, w: int, h: int, adversarial: bool = False, scale: float = 1.0):
    """seeded keyframe planes (h, w) INPUT_POINT_DENSE + a camToWorld (7 floats) + cam (fx, fy, cx, cy): a smooth inverse-depth
    surface with noise on the order of its variance, so that every branch of the filter is taken; adversarial adds idepth <= 0,
    +-Inf and NaN, negative / zero / infinite / NaN variances, and valid pixels on the border rows and columns"""
    # only +, -, *, / and sqrt (correctly rounded everywhere), so that the planes are the same bits on any CPU and numpy build
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    u, v = xx / w - 0.5, yy / h - 0.5
    surf = 0.6 + 0.8 * u * u - 0.5 * u * v + 0.3 * (xx > w / 2)
    var = rng.uniform(0.006, 0.8, (h, w)) ** 2 * 0.5
    idepth = surf + rng.standard_normal((h, w)) * np.sqrt(var) * rng.uniform(0.2, 2.0, (h, w))
    idepth[rng.random((h, w)) < 0.15] = -0.2                    # invalid pixels as the core publishes them
    pc = np.zeros((h, w), INPUT_POINT_DENSE)
    pc["idepth"], pc["idepth_var"] = idepth.astype(np.float32), var.astype(np.float32)
    pc["color"] = rng.integers(0, 256, (h, w), dtype=np.uint8)[..., None]
    if adversarial:
        n = h * w
        for val, frac in ((0.0, 0.02), (-0.0, 0.02), (np.inf, 0.02), (-np.inf, 0.02), (np.nan, 0.03), (1e-30, 0.01), (1e30, 0.01)):
            pc["idepth"].reshape(-1)[rng.random(n) < frac] = val
        for val, frac in ((-1e-3, 0.03), (0.0, 0.03), (np.inf, 0.01), (np.nan, 0.01), (1e-38, 0.01)):
            pc["idepth_var"].reshape(-1)[rng.random(n) < frac] = val
        pc["idepth"][0, :], pc["idepth"][-1, :] = surf[0, :], surf[-1, :]      # valid borders
        pc["idepth"][:, 0], pc["idepth"][:, -1] = surf[:, 0], surf[:, -1]
    q = rng.standard_normal(4)
    q /= np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    c2w = np.concatenate([q * scale, rng.uniform(-2, 2, 3)]).astype(np.float32)
    cam = tuple(float(v) for v in np.float32([0.8 * w, 0.9 * h, w / 2 - 0.5, h / 2 - 0.5]))
    return pc, c2w, cam


def ply_header(n_points: int) -> bytes:
    """the header KeyFrameGraphDisplay.cpp:74-82 writes"""
    return (b"ply\nformat binary_little_endian 1.0\n" + b"element vertex %d\n" % n_points +
            b"property float x\nproperty float y\nproperty float z\nproperty float intensity\nend_header\n")


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print("restatement:", ORACLE_SO, "viewer:", VIEWER_SO if viewer_built() else "not built")
