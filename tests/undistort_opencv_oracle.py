"""ctypes binding of tests/native/undistort_opencv_oracle.c, the tests' plain-C restatement of UndistorterOpenCV
(util/Undistorter.cpp:449-567).  The library is compiled on first use into a temporary directory (never into the tree)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "undistort_opencv_oracle.c")
MODES = {"crop": -1, "full": -2}
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    src = open(SRC, "rb").read()
    out = os.path.join(tempfile.gettempdir(), "lsdgpu_cv_oracle_%d_%s.so" % (os.getuid(), hashlib.sha1(src).hexdigest()[:12]))
    if not os.path.exists(out):
        tmp = out + ".%d" % os.getpid()
        subprocess.run(["gcc", "-std=gnu11", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", tmp, SRC, "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    i16p, u16p, u8p = C.POINTER(C.c_int16), C.POINTER(C.c_uint16), C.POINTER(C.c_uint8)
    L.lsdo_cv_prepare.restype = C.c_int
    L.lsdo_cv_prepare.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, i16p, u16p,
                                  C.POINTER(C.c_double), C.POINTER(C.c_float)]
    L.lsdo_cv_remap.restype = None
    L.lsdo_cv_remap.argtypes = [u8p, C.c_int, C.c_int, i16p, u16p, C.c_int, C.c_int, u8p]
    _lib = L
    return L


class UndistorterOpenCV:
    """the oracle's tables for the parsed calibration (in_calib = fx fy cx cy k1 k2 p1 p2, out_mode "crop" / "full")"""

    def __init__(self, in_calib, in_size, out_mode, out_size):
        L = lib()
        self.in_w, self.in_h = in_size
        self.out_w, self.out_h = out_size
        ic = np.ascontiguousarray(in_calib, np.float32)
        self.map1 = np.zeros((self.out_h, self.out_w, 2), np.int16)
        self.map2 = np.zeros((self.out_h, self.out_w), np.uint16)
        K_new, K = np.zeros(9, np.float64), np.zeros(9, np.float32)
        self.status = L.lsdo_cv_prepare(ic.ctypes.data_as(C.POINTER(C.c_float)), self.in_w, self.in_h, MODES.get(out_mode, 0),
                                        self.out_w, self.out_h, self.map1.ctypes.data_as(C.POINTER(C.c_int16)),
                                        self.map2.ctypes.data_as(C.POINTER(C.c_uint16)), K_new.ctypes.data_as(C.POINTER(C.c_double)),
                                        K.ctypes.data_as(C.POINTER(C.c_float)))
        self.K_new, self.K = K_new.reshape(3, 3), K.reshape(3, 3)

    def undistort(self, raw_u8: np.ndarray) -> np.ndarray:
        return remap(raw_u8, self.map1, self.map2)


def remap(raw_u8: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """cv::remap(raw, out, map1, map2, INTER_LINEAR) with the constant 0 border, u8"""
    raw = np.ascontiguousarray(raw_u8, np.uint8)
    m1, m2 = np.ascontiguousarray(map1, np.int16), np.ascontiguousarray(map2, np.uint16)
    oh, ow = m2.shape
    out = np.zeros((oh, ow), np.uint8)
    u8p = C.POINTER(C.c_uint8)
    lib().lsdo_cv_remap(raw.ctypes.data_as(u8p), raw.shape[1], raw.shape[0], m1.ctypes.data_as(C.POINTER(C.c_int16)),
                        m2.ctypes.data_as(C.POINTER(C.c_uint16)), ow, oh, out.ctypes.data_as(u8p))
    return out
