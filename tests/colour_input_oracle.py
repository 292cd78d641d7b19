"""ctypes binding of tests/native/colour_input_oracle.c, the tests' plain-C restatement of cv::cvtColor's 8-bit gray conversions
(cv_bridge::toCvCopy(img, MONO8), ROSImageStreamThread.cpp:117; cvtColor(.., CV_RGB2GRAY), LiveSLAMWrapper.cpp:116-121).  The
library is compiled on first use into a temporary directory (never into the tree)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "colour_input_oracle.c")
# ROS encoding -> (LSDGPU_PIX_* number, bytes per pixel), as lsd_slam_b200.abi.INPUT_FORMATS
FORMATS = {"mono8": (0, 1), "rgb8": (1, 3), "bgr8": (2, 3), "rgba8": (3, 4), "bgra8": (4, 4), "yuv422": (5, 2),
           "yuv422_yuy2": (6, 2)}
# SHA-256 of the 2^24-entry COLOR_RGB2GRAY table of OpenCV 4.13, indexed by R << 16 | G << 8 | B
RGB_TABLE_SHA256 = "6d4f6d7f4301c52d2672db66451b4a06a5502bef956dd81b577660f956f410ae"
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    src = open(SRC, "rb").read()
    out = os.path.join(tempfile.gettempdir(), "lsdgpu_cvt_oracle_%d_%s.so" % (os.getuid(), hashlib.sha1(src).hexdigest()[:12]))
    if not os.path.exists(out):
        tmp = out + ".%d" % os.getpid()
        subprocess.run(["gcc", "-std=gnu11", "-O2", "-shared", "-fPIC", "-o", tmp, SRC], check=True, capture_output=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    u8p = C.POINTER(C.c_uint8)
    L.lsdo_cvt_gray.restype = C.c_int
    L.lsdo_cvt_gray.argtypes = [C.c_int, u8p, C.c_int, C.c_int, C.c_size_t, u8p]
    L.lsdo_cvt_rgb_table.restype = None
    L.lsdo_cvt_rgb_table.argtypes = [u8p]
    _lib = L
    return L


def to_gray(raw: np.ndarray, encoding: str) -> np.ndarray:
    """cv::cvtColor of a (h, w) mono8 or (h, w, bytes per pixel) image to 8-bit gray"""
    fmt, bpp = FORMATS[encoding]
    raw = np.ascontiguousarray(raw, np.uint8)
    h, w = raw.shape[:2]
    assert raw.shape == ((h, w) if bpp == 1 else (h, w, bpp)), (raw.shape, encoding)
    out = np.empty((h, w), np.uint8)
    u8p = C.POINTER(C.c_uint8)
    assert lib().lsdo_cvt_gray(fmt, raw.ctypes.data_as(u8p), w, h, w * bpp, out.ctypes.data_as(u8p)) == 0
    return out


def rgb_table() -> np.ndarray:
    """the gray value of every 24-bit colour, indexed by R << 16 | G << 8 | B"""
    out = np.empty(1 << 24, np.uint8)
    lib().lsdo_cvt_rgb_table(out.ctypes.data_as(C.POINTER(C.c_uint8)))
    return out


def random_raw(w: int, h: int, encoding: str, seed: int) -> np.ndarray:
    """a uniformly random raw image of the encoding's shape"""
    bpp = FORMATS[encoding][1]
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w) if bpp == 1 else (h, w, bpp), dtype=np.uint8)


def cv2_gray(raw: np.ndarray, encoding: str) -> np.ndarray:
    """the same conversion by OpenCV itself (cv_bridge's codes); needs cv2"""
    import cv2
    code = {"rgb8": cv2.COLOR_RGB2GRAY, "bgr8": cv2.COLOR_BGR2GRAY, "rgba8": cv2.COLOR_RGBA2GRAY, "bgra8": cv2.COLOR_BGRA2GRAY,
            "yuv422": cv2.COLOR_YUV2GRAY_UYVY, "yuv422_yuy2": cv2.COLOR_YUV2GRAY_YUY2}
    if encoding == "mono8":
        return raw.copy()
    return cv2.cvtColor(np.ascontiguousarray(raw), code[encoding])
