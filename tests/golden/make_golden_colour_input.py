"""Records tests/golden/colour_input.npz from OpenCV itself (cv2 4.13, the version UndistorterOpenCV is pinned to): the gray
conversions cv_bridge::toCvCopy(img, MONO8) (IOWrapper/ROS/ROSImageStreamThread.cpp:117) and cvtColor(.., CV_RGB2GRAY)
(LiveSLAMWrapper.cpp:116-121) run in front of the undistorter.

  rgb_sha256            SHA-256 of COLOR_RGB2GRAY over all 2^24 colours, indexed by R << 16 | G << 8 | B (the 16 MB table itself
                        is not stored); rgb_sample_idx / rgb_sample_gray: 4096 of its entries
  rgb14_diff_idx        the colours where OpenCV 2.4's 14-bit formula (R * 4899 + G * 9617 + B * 1868 + 8192) >> 14 differs
                        (by one level each)
  small__<enc>__<w>__raw / __gray   cvtColor of a seeded random 2-row image of width w for every encoding (odd widths; the 4:2:2
                        encodings at even widths)
  undist__<cam>__<enc>  SHA-256 of cvtColor followed by the camera's undistorter on raw_seed(<enc>)'s image: "ptam" = the
                        raw752_full calibration of ref_pin_undistort.npz through the oracle's UndistorterPTAM, "opencv" = the
                        example_crop calibration of opencv_undistort.npz through cv2.remap of the maps cv2 builds

No reference source is involved.  Run from the repository root: python -m tests.golden.make_golden_colour_input"""
from __future__ import annotations

import hashlib
import os

import numpy as np

from tests import colour_input_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "colour_input.npz")
ENCODINGS = ["rgb8", "bgr8", "rgba8", "bgra8", "yuv422", "yuv422_yuy2"]
SMALL_WIDTHS = {"odd": [1, 3, 7, 17, 641], "even": [2, 6, 18, 642]}
PTAM_CASE = "raw752_full"
OPENCV_CASE = "example_crop"


def small_widths(enc):
    return SMALL_WIDTHS["even" if enc.startswith("yuv") else "odd"]


def raw_seed(enc: str) -> int:
    return 1000 + ENCODINGS.index(enc)


def sha(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def all_colours() -> np.ndarray:
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def ptam_undistorter():
    from oracle import pyoracle as po
    from tests.golden import make_golden_ref_pin_undistort as mg
    po.build()
    return po.UndistorterPTAM(*mg.parse(dict(mg.cases())[PTAM_CASE]))


def opencv_case():
    z = np.load(os.path.join(HERE, "opencv_undistort.npz"))
    i = list(z["name"]).index(OPENCV_CASE)
    return z["calib"][i], tuple(int(v) for v in z["in_size"][i]), str(z["mode"][i]), tuple(int(v) for v in z["out_size"][i])


def main():
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    rec = {"opencv_version": np.array(cv2.__version__)}
    img = all_colours()
    table = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY).reshape(-1)
    rec["rgb_sha256"] = sha(table)
    idx = np.sort(np.random.default_rng(7).choice(1 << 24, 4096, replace=False)).astype(np.uint32)
    rec["rgb_sample_idx"], rec["rgb_sample_gray"] = idx, table[idx]
    r, g, b = (img[..., k].reshape(-1).astype(np.int64) for k in range(3))
    rec["rgb14_diff_idx"] = np.nonzero(((r * 4899 + g * 9617 + b * 1868 + 8192) >> 14) != table)[0].astype(np.uint32)
    for enc in ENCODINGS:
        for w in small_widths(enc):
            raw = co.random_raw(w, 2, enc, seed=w * 31 + ENCODINGS.index(enc))
            rec[f"small__{enc}__{w}__raw"], rec[f"small__{enc}__{w}__gray"] = raw, co.cv2_gray(raw, enc)
    pt = ptam_undistorter()
    calib, in_size, mode, out_size = opencv_case()
    fx, fy, cx, cy, k1, k2, p1, p2 = (float(v) for v in calib)
    if cx < 1:
        fx, cx, fy, cy = fx * in_size[0], cx * in_size[0], fy * in_size[1], cy * in_size[1]
    K, D = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]]), np.array([k1, k2, p1, p2])
    K_new, _ = cv2.getOptimalNewCameraMatrix(K, D, in_size, {"crop": 0, "full": 1}[mode], out_size)
    m1, m2 = cv2.initUndistortRectifyMap(K, D, None, K_new, out_size, cv2.CV_16SC2)
    for enc in ENCODINGS:
        raw_pt = co.random_raw(pt.in_w, pt.in_h, enc, raw_seed(enc))
        rec[f"undist__ptam__{enc}"] = sha(pt.undistort(co.cv2_gray(raw_pt, enc)))
        raw_cv = co.random_raw(in_size[0], in_size[1], enc, raw_seed(enc))
        rec[f"undist__opencv__{enc}"] = sha(cv2.remap(co.cv2_gray(raw_cv, enc), m1, m2, cv2.INTER_LINEAR))
    np.savez_compressed(OUT, **rec)
    print(OUT, os.path.getsize(OUT), "bytes;", len(rec["rgb14_diff_idx"]), "colours differ under the 14-bit formula")


if __name__ == "__main__":
    main()
