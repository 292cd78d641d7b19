"""Writes tests/golden/ref_pin_undistort.npz: what the reference's own UndistorterPTAM (util/Undistorter.cpp:38-411, compiled
unmodified into oracle/_ref/liblsd_ref.so) computes from a sweep of calibration files -- its verdict, sizes, K as
main_on_images.cpp:164-167 reads it, digests and a sample of its remap tables, digests of undistort() on three raw images, and
Undistorter::getUndistorterForFile's verdict -- plus the distance of the legacy-math build (liblsd_ref_legacy_math.so: tan / atan /
sqrt on doubles, as a g++ < 6 toolchain resolves them) and libm's tanf / atanf on arguments of the tables' range.  The case list
and the raw-image generators live here so that the tests use the same ones.  Written with save_npz_reproducible, so that a re-run
reproduces it byte for byte.

    python -m tests.golden.make_golden_ref_pin_undistort
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_pin_undistort.npz")

# the wide-angle ATAN calibration of the reference's example files (relative units)
FOV = [0.535719308086809, 0.669566858850269, 0.493248545285398, 0.500408664348414, 0.897966326944875]
EXPLICIT = "0.6 0.8 0.5 0.5 0"


def _file(calib, in_size, mode, out_size, eol="\n"):
    return eol.join([" ".join(repr(v) for v in calib), "%d %d" % in_size, mode, "%d %d" % out_size]) + eol


def _named():
    c = []
    for mode_name, mode in (("crop", "crop"), ("full", "full"), ("expl", EXPLICIT)):
        for size_name, out in (("same", (640, 480)), ("320", (320, 240)), ("1280", (1280, 960))):
            c.append((f"fov_{mode_name}_{size_name}", _file(FOV, (640, 480), mode, out)))
    w0 = [0.5, 0.7, 0.49, 0.51, 0.0]
    c += [
        ("w0_same", _file(w0, (640, 480), "crop", (640, 480))),             # pass-through of :370-375
        ("w0_down", _file(w0, (640, 480), "crop", (320, 240))),
        ("w0_up", _file(w0, (640, 480), "full", (1280, 960))),
        # the table's iy == 0 lands on 0.01 in a whole row, ix == 0 / in_width - 1 on 0.01 / in_width - 1.01 (:299-301)
        ("w0_centred_same", _file([0.5, 0.7, 0.5, 0.5, 0.0], (640, 480), "crop", (640, 480))),
        ("w14_full", _file([0.4, 0.55, 0.52, 0.47, 1.4], (640, 480), "full", (640, 480))),    # negative focal lengths
        ("w14_crop", _file([0.4, 0.55, 0.52, 0.47, 1.4], (640, 480), "crop", (640, 480))),
        ("w28_full", _file([0.3, 0.4, 0.5, 0.5, 2.8], (640, 480), "full", (640, 480))),
        ("offc_full_1280x1024", _file([0.7, 0.9, 0.3, 0.8, 0.6], (1280, 1024), "full", (640, 480))),
        ("offc_crop_1280x1024", _file([0.7, 0.9, 0.3, 0.8, 0.6], (1280, 1024), "crop", (640, 480))),
        # cx = cy = 0: every corner ratio of "full" is 0/0; std::max keeps the NaN of :260, so ocy is NaN and every entry -1
        ("nan_full_cx0_cy0", _file([0.5, 0.6, 0.00078125, 0.00104166667, 0.9], (640, 480), "full", (640, 480))),
        ("nan_crop_cx0", _file([0.5, 0.7, 0.00078125, 0.5, 0.9], (640, 480), "crop", (640, 480))),
        ("raw641_crop", _file(FOV, (641, 481), "crop", (640, 480))),
        ("raw641_same", _file(FOV, (641, 481), "crop", (641, 481))),
        ("raw752_full", _file(FOV, (752, 480), "full", (640, 480))),
        ("raw1241_crop", _file([0.55, 1.8, 0.51, 0.49, 0.7], (1241, 376), "crop", (1232, 368))),
        ("tiny64", _file([0.5, 0.7, 0.5, 0.5, 0.9], (64, 48), "crop", (64, 48))),
        ("none", "0.5 0.7 0.5 0.5 0.9\n640 480\nnone\n640 480\n"),
    ]
    return c


def _malformed():
    good = _file(FOV, (640, 480), "crop", (640, 480))
    return [
        ("bad_trailing_blank", good.replace("crop\n", "crop \n")),
        ("bad_crlf", good.replace("\n", "\r\n")),
        ("bad_missing_line4", "\n".join(good.split("\n")[:3]) + "\n"),
        ("bad_four_numbers", good.replace(" " + repr(FOV[4]), "", 1)),
        ("bad_six_numbers", good.replace(repr(FOV[4]), repr(FOV[4]) + " 0.25", 1)),    # sscanf reads the first 5: valid
        # the OpenCV model's first line: getUndistorterForFile dispatches it to UndistorterOpenCV (:70-80); the reference's PTAM
        # constructor, called on it directly, reads its first 5 numbers, whereas the library's adapter refuses it
        ("opencv8", "500 500 320 240 0.1 0.01 0 0\n640 480\ncrop\n640 480\n"),
    ]


def cases():
    return _named() + _malformed()


OPENCV_DISPATCH = {"opencv8"}          # never handed to the reference's getUndistorterForFile (it would construct the OpenCV model)
ROUNDING_CASES = ("fov_crop_same", "w0_same", "w0_centred_same")


def parse(text):
    """the four lines as the parsed APIs take them: (in_calib, in_size, out_calib, out_size); "none" is the zero output
    calibration both the adapter and oracle/_ref's zero-filled object use"""
    l1, l2, l3, l4 = text.split("\n")[:4]
    ic = [float(v) for v in l1.split()][:5]
    oc = l3 if l3 in ("crop", "full") else ([0.0] * 5 if l3 == "none" else [float(v) for v in l3.split()])
    return ic, tuple(int(v) for v in l2.split()), oc, tuple(int(v) for v in l4.split())


def raw_images(w, h):
    """seeded noise, a one-pixel 0/255 checkerboard (every bilinear weight shows) and constant 255 (where the four weights
    round below 1, truncation gives 254)"""
    y, x = np.mgrid[0:h, 0:w]
    noise = np.random.default_rng(zlib.crc32(b"%d %d" % (w, h))).integers(0, 256, (h, w)).astype(np.uint8)
    return [noise, (((x + y) & 1) * 255).astype(np.uint8), np.full((h, w), 255, np.uint8)]


def sha(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8).copy()


def sample_index(name, n, k=4096):
    return np.random.default_rng(zlib.crc32(name.encode())).integers(0, n, k).astype(np.int64)


def write_case(dirname, name, text) -> str:
    p = os.path.join(dirname, name + ".cfg")
    with open(p, "w", newline="") as f:
        f.write(text)
    return p


def sscanf_count(line: str, n: int) -> int:
    """the C library's sscanf of n "%f" conversions, as Undistorter.cpp:72-74 (n = 8) and :116 (n = 5) count them"""
    libc = C.CDLL(None)
    vals = (C.c_float * n)()
    return libc.sscanf(line.encode(), b" ".join([b"%f"] * n), *[C.byref(vals, 4 * i) for i in range(n)])


def libm_args():
    """arguments of the range tan / atan take in the tables and radii: r * dist up to ~1.6, r * d2t up to ~4"""
    t = np.linspace(0.0, 1.55, 257, dtype=np.float32)[1:]
    a = np.linspace(0.0, 4.0, 257, dtype=np.float32)[1:]
    halves = np.array([v / np.float32(2) for v in np.float32([FOV[4], 0.6, 0.7, 0.9, 1.4, 2.8])], np.float32)
    return np.concatenate([t, halves]), a


def libm_values():
    m = C.CDLL("libm.so.6")
    m.tanf.restype = m.atanf.restype = C.c_float
    m.tanf.argtypes = m.atanf.argtypes = [C.c_float]
    ta, aa = libm_args()
    return (np.array([m.tanf(float(v)) for v in ta], np.float32), np.array([m.atanf(float(v)) for v in aa], np.float32))


def record(po, tmp):
    out = {}
    out["libm_tanf"], out["libm_atanf"] = libm_values()
    for name, text in cases():
        path = write_case(tmp, name, text)
        out[f"{name}__file"] = np.frombuffer(text.encode(), np.uint8).copy()
        r = po.RefUndistorterFile(path, "ref")
        leg = po.RefUndistorterFile(path, "ref_legacy_math")
        verdict = 2 if sscanf_count(text.split("\n")[0], 8) == 8 else po.ref_undistorter_for_file(path)
        if name in OPENCV_DISPATCH:
            assert verdict == 2
        n_invalid = -1 if r.remapX is None else int((r.remapX < 0).sum())
        out[f"{name}__info"] = np.array([r.valid, r.in_w, r.in_h, r.out_w, r.out_h, n_invalid, verdict], np.int64)
        out[f"{name}__K"] = np.array([r.K[0, 0], r.K[1, 1], r.K[0, 2], r.K[1, 2]], np.float32)
        if r.remapX is None:
            continue
        out[f"{name}__remap_sha"] = np.stack([sha(r.remapX), sha(r.remapY)])
        idx = sample_index(name, r.remapX.size)
        out[f"{name}__sample"] = np.stack([r.remapX.ravel()[idx], r.remapY.ravel()[idx]])
        shas, shapes, dpix, dmax = [], [], [], []
        for img in raw_images(r.in_w, r.in_h):
            a, b = r.undistort(img), leg.undistort(img)
            shas.append(sha(a))
            shapes.append(a.shape)
            dpix.append(int((a != b).sum()))
            dmax.append(int(np.abs(a.astype(np.int32) - b.astype(np.int32)).max()))
        out[f"{name}__img_sha"] = np.stack(shas)
        out[f"{name}__img_shape"] = np.array(shapes, np.int64)
        dx = int((r.remapX.view(np.int32) != leg.remapX.view(np.int32)).sum())
        dy = int((r.remapY.view(np.int32) != leg.remapY.view(np.int32)).sum())
        dk = int((np.asarray(r.K).view(np.int32) != np.asarray(leg.K).view(np.int32)).sum())
        out[f"{name}__legacy"] = np.array([dx, dy, dk] + dpix + dmax, np.int64)
        r.close()
        leg.close()
    return out


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import pyoracle
    from tests.golden.make_golden_ref_pin_globals import save_npz_reproducible
    pyoracle.build()
    if not pyoracle.ref_available():
        raise SystemExit("oracle/_ref is not built and the reference sources are absent: this fixture cannot be regenerated here")
    with tempfile.TemporaryDirectory() as tmp:
        res = record(pyoracle, tmp)
    save_npz_reproducible(OUT, res)
    print(f"{OUT}: {len(res)} arrays")
