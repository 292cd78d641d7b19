"""CPU checks of the gray conversion in front of the undistorter (cv_bridge::toCvCopy(img, MONO8), ROSImageStreamThread.cpp:117;
cvtColor(.., CV_RGB2GRAY), LiveSLAMWrapper.cpp:116-121): the tests' C restatement (tests/native/colour_input_oracle.c) against
what OpenCV 4.13 recorded in tests/golden/colour_input.npz -- the whole 2^24-colour table by its digest, the colours where OpenCV
2.4's 14-bit formula differs, small images of every encoding at odd widths, and the conversion followed by both undistorters --
and against cv2 itself where it can be imported.  The format numbers agree between include/lsdgpu.h, abi.py and the oracle."""
import hashlib
import os
import re

import numpy as np
import pytest

from tests import colour_input_oracle as co
from tests import undistort_opencv_oracle as uo
from tests.golden import make_golden_colour_input as mg

GOLD = np.load(mg.OUT)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def test_rgb_table_matches_opencv_digest_and_sample():
    table = co.rgb_table()
    assert hashlib.sha256(table.tobytes()).hexdigest() == co.RGB_TABLE_SHA256 == bytes(GOLD["rgb_sha256"]).hex()
    assert np.array_equal(table[GOLD["rgb_sample_idx"]], GOLD["rgb_sample_gray"])
    # the table through the image entry point: RGB and BGR orders, 3 and 4 channels
    idx = GOLD["rgb_sample_idx"]
    rgb = np.stack([(idx >> 16) & 255, (idx >> 8) & 255, idx & 255], -1).astype(np.uint8)[None]
    alpha = np.full(rgb.shape[:2] + (1,), 77, np.uint8)
    for enc, img in (("rgb8", rgb), ("bgr8", rgb[..., ::-1]), ("rgba8", np.concatenate([rgb, alpha], -1)),
                     ("bgra8", np.concatenate([rgb[..., ::-1], alpha], -1))):
        assert np.array_equal(co.to_gray(img, enc)[0], GOLD["rgb_sample_gray"]), enc


def test_opencv_2_4_formula_differs_by_one_level_on_the_recorded_colours():
    table = co.rgb_table().astype(np.int64)
    c = np.arange(1 << 24, dtype=np.int64)
    old = ((c >> 16) * 4899 + ((c >> 8) & 255) * 9617 + (c & 255) * 1868 + 8192) >> 14
    diff = np.nonzero(old != table)[0]
    assert len(diff) == 43864
    assert np.array_equal(diff, GOLD["rgb14_diff_idx"])
    assert np.abs(old[diff] - table[diff]).max() == 1


@pytest.mark.parametrize("enc", mg.ENCODINGS)
def test_small_images_at_odd_widths_match_opencv(enc):
    for w in mg.small_widths(enc):
        raw = GOLD[f"small__{enc}__{w}__raw"]
        assert np.array_equal(co.to_gray(raw, enc), GOLD[f"small__{enc}__{w}__gray"]), w


@pytest.mark.parametrize("enc", mg.ENCODINGS)
def test_conversion_then_both_undistorters_match_opencv(enc, oracle):
    pt = mg.ptam_undistorter()
    raw = co.random_raw(pt.in_w, pt.in_h, enc, mg.raw_seed(enc))
    assert _sha(pt.undistort(co.to_gray(raw, enc))) == bytes(GOLD[f"undist__ptam__{enc}"])
    calib, in_size, mode, out_size = mg.opencv_case()
    u = uo.UndistorterOpenCV(calib, in_size, mode, out_size)
    raw = co.random_raw(in_size[0], in_size[1], enc, mg.raw_seed(enc))
    assert _sha(u.undistort(co.to_gray(raw, enc))) == bytes(GOLD[f"undist__opencv__{enc}"])


@pytest.mark.parametrize("enc", mg.ENCODINGS)
def test_oracle_equals_cv2(enc):
    cv2 = pytest.importorskip("cv2")
    if not cv2.__version__.startswith("4.13"):
        pytest.skip(f"the conversion is pinned to OpenCV 4.13, not {cv2.__version__}")
    for w in (1, 2, 3, 7, 17, 640, 641):
        if enc.startswith("yuv") and w % 2:
            continue
        raw = co.random_raw(w, 5, enc, seed=w)
        assert np.array_equal(co.to_gray(raw, enc), co.cv2_gray(raw, enc)), w


def test_format_numbers_agree_with_the_header_and_abi():
    from lsd_slam_b200 import abi
    hdr = open(os.path.join(ROOT, "include", "lsdgpu.h")).read()
    enum = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"LSDGPU_PIX_([A-Z0-9_]+)\s*=\s*(\d+)", hdr)}
    assert enum == {k: v[0] for k, v in co.FORMATS.items()}
    assert abi.INPUT_FORMATS == co.FORMATS
