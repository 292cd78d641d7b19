"""Writes tests/golden/opencv_undistort.npz: what OpenCV itself computes for UndistorterOpenCV (util/Undistorter.cpp:449-567)
on a fixed set of calibrations -- cv::getOptimalNewCameraMatrix, cv::initUndistortRectifyMap(.., CV_16SC2) and cv::remap
(INTER_LINEAR) of fixed raw images.  Needs the cv2 module (the fixture was made with OpenCV 4.13 on x86-64); the tests only read
the file.  The case list and the raw-image generator live here so that the tests use the same ones.

    python tests/golden/make_golden_opencv_undistort.py
"""
from __future__ import annotations

import os
import zlib

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "opencv_undistort.npz")

TUM_FR1 = [517.3, 516.5, 318.6, 255.3, 0.2624, -0.9531, -0.0054, 0.0026]
EUROC = [458.654, 457.296, 367.215, 248.375, -0.2834, 0.0740, 0.00019, 1.76e-05]
EXAMPLE = [500, 500, 350, 240, 0, 0, 0, 0]                     # lsd_slam_core/calib/OpenCV_example_calib.cfg
RELATIVE = [0.5, 0.7, 0.49, 0.51, -0.1, 0.01, 0.001, -0.002]   # cx < 1: relative units (Undistorter.cpp:519-534)

# (name, fx fy cx cy k1 k2 p1 p2, input size, "crop" / "full", output size); output sizes are multiples of 16
NAMED = [
    ("example_crop", EXAMPLE, (752, 480), "crop", (640, 480)),
    ("example_full", EXAMPLE, (752, 480), "full", (640, 480)),
    ("tum_fr1_crop", TUM_FR1, (640, 480), "crop", (640, 480)),
    ("tum_fr1_full", TUM_FR1, (640, 480), "full", (640, 480)),
    ("euroc_crop", EUROC, (752, 480), "crop", (640, 480)),
    ("euroc_full", EUROC, (752, 480), "full", (640, 480)),
    ("relative_crop", RELATIVE, (640, 480), "crop", (320, 240)),
]
N_RANDOM = 20
SMALL = "relative_crop"                                        # the case whose full maps are stored
RAW_SEEDS = (0, 1)


def random_cases(n=N_RANDOM, seed=20261016):
    """seeded realistic calibrations (pixel units): focal 0.55..1.1 x width, principal point within 5 % of the centre"""
    rng = np.random.default_rng(seed)
    ins, outs = [(640, 480), (752, 480), (1280, 1024), (320, 240)], [(640, 480), (320, 240), (512, 384)]
    cases = []
    for t in range(n):
        (iw, ih), out = ins[t % 4], outs[t % 3]
        f = rng.uniform(0.55, 1.1) * iw
        c = [f, f * rng.uniform(0.98, 1.02), iw / 2 * rng.uniform(0.95, 1.05), ih / 2 * rng.uniform(0.95, 1.05),
             rng.uniform(-0.4, 0.25), rng.uniform(-0.2, 0.2), rng.uniform(-3e-3, 3e-3), rng.uniform(-3e-3, 3e-3)]
        cases.append(("random_%02d" % t, [float(np.float32(v)) for v in c], (iw, ih), ("crop", "full")[t % 2], out))
    return cases


def cases():
    return NAMED + random_cases()


def raw_image(w: int, h: int, seed: int) -> np.ndarray:
    """a deterministic textured u8 image (integer hash, no RNG): every bilinear weight sees varied neighbours"""
    y, x = np.mgrid[0:h, 0:w].astype(np.uint32)
    v = x * np.uint32(2654435761) ^ (y + np.uint32(977 * seed + 1)) * np.uint32(2246822519)
    v ^= v >> np.uint32(15)
    v *= np.uint32(2654435769)
    v ^= v >> np.uint32(13)
    return (v >> np.uint32(24)).astype(np.uint8)


def crc(a: np.ndarray) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xFFFFFFFF


def opencv_tables(cv2, calib, in_size, mode, out_size):
    """UndistorterOpenCV's constructor (Undistorter.cpp:515-548) through cv2"""
    ic = np.array(calib, np.float32)
    iw, ih = in_size
    if ic[2] < 1.0:
        ic[0] *= iw; ic[2] *= iw; ic[1] *= ih; ic[3] *= ih
    K = np.zeros((3, 3)); K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[2, 2] = ic[0], ic[1], ic[2], ic[3], 1
    D = ic[4:].reshape(4, 1).astype(np.float32)
    K_new, _ = cv2.getOptimalNewCameraMatrix(K, D, in_size, 1 if mode == "full" else 0, out_size, centerPrincipalPoint=False)
    map1, map2 = cv2.initUndistortRectifyMap(K, D, None, K_new, out_size, cv2.CV_16SC2)
    K_out = np.zeros((3, 3), np.float32)                       # getK() = K_.t(), main_on_images.cpp:164-167
    K_out[0, 0], K_out[1, 1], K_out[0, 2], K_out[1, 2], K_out[2, 2] = K_new[0, 0], K_new[1, 1], K_new[0, 2], K_new[1, 2], 1
    return K_new, K_out, map1, map2


def main():
    import cv2
    cs = cases()
    rec = {k: [] for k in ("name", "calib", "in_size", "mode", "out_size", "K_new", "K_out", "crc_map1", "crc_map2", "crc_remap")}
    small = {}
    for name, calib, in_size, mode, out_size in cs:
        K_new, K_out, map1, map2 = opencv_tables(cv2, calib, in_size, mode, out_size)
        rec["name"].append(name); rec["calib"].append(np.float32(calib)); rec["in_size"].append(in_size); rec["mode"].append(mode)
        rec["out_size"].append(out_size); rec["K_new"].append(K_new.ravel()); rec["K_out"].append(K_out.ravel())
        rec["crc_map1"].append(crc(map1)); rec["crc_map2"].append(crc(map2))
        rec["crc_remap"].append([crc(cv2.remap(raw_image(*in_size, s), map1, map2, cv2.INTER_LINEAR)) for s in RAW_SEEDS])
        if name == SMALL:
            small = {"small_map1": map1, "small_map2": map2}
    arrs = {k: np.array(v) for k, v in rec.items()}
    arrs["crc_map1"] = arrs["crc_map1"].astype(np.uint32); arrs["crc_map2"] = arrs["crc_map2"].astype(np.uint32)
    arrs["crc_remap"] = arrs["crc_remap"].astype(np.uint32)
    np.savez_compressed(OUT, **arrs, **small, opencv_version=np.array(cv2.__version__))
    print(OUT, os.path.getsize(OUT), "bytes,", len(cs), "cases, OpenCV", cv2.__version__)


if __name__ == "__main__":
    main()
