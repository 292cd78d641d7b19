"""PIN of UndistorterPTAM (util/Undistorter.cpp:38-411) to the reference's own code, on the CPU.

tests/golden/ref_pin_undistort.npz holds what the reference's class, compiled unmodified into oracle/_ref/liblsd_ref.so, computes
from the calibration files of tests/golden/make_golden_ref_pin_undistort.py: its verdict, sizes, K, remap-table digests and
undistort() digests on three raw images, getUndistorterForFile's verdict, and the distance of the legacy-math build.  Here the C
oracle (oracle/lsd_oracle_undistort.inc), the library's table builder (lsdgpu_undistorter_ptam_prepare) and the C++ adapter's
file constructor and getUndistorterForFile (through host_demo) must reproduce that record on every file; where oracle/_ref exists
the live reference must too.  The device remap is pinned to the same digests by tests/test_gpu_undistort_ptam.py."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi
from oracle import pyoracle as po
from tests.golden import make_golden_ref_pin_undistort as mg

GOLD = np.load(mg.OUT)
CASES = [name for name, _ in mg.cases()]
TEXT = dict(mg.cases())
# files the reference's UndistorterPTAM constructor accepts: the parsed APIs take their first five numbers
VALID = [n for n in CASES if GOLD[n + "__info"][0] == 1]


def _info(name):
    valid, iw, ih, ow, oh, n_invalid, verdict = (int(v) for v in GOLD[name + "__info"])
    return valid, (iw, ih), (ow, oh), n_invalid, verdict


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def _k4(K):
    K = np.asarray(K, np.float32).reshape(3, 3)
    return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float32)


def _same_bits(a, b):
    return np.asarray(a, np.float32).tobytes() == np.asarray(b, np.float32).tobytes()


def _check_tables(name, remapX, remapY, K):
    _, _, (ow, oh), n_invalid, _ = _info(name)
    assert remapX.shape == (oh, ow)
    assert _same_bits(_k4(K), GOLD[name + "__K"]), (name, _k4(K), GOLD[name + "__K"])
    assert int((remapX < 0).sum()) == n_invalid, name
    idx = mg.sample_index(name, remapX.size)
    got = np.stack([remapX.ravel()[idx], remapY.ravel()[idx]])
    want = GOLD[name + "__sample"]
    bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any(axis=0))
    assert bad.size == 0, f"{name}: {bad.size} of {idx.size} sampled entries differ, first at {idx[bad[0]]}: {got[:, bad[0]]} vs {want[:, bad[0]]}"
    assert _sha(remapX) == GOLD[name + "__remap_sha"][0].tobytes() and _sha(remapY) == GOLD[name + "__remap_sha"][1].tobytes(), name


def _check_images(name, undistort, in_size):
    for k, img in enumerate(mg.raw_images(*in_size)):
        out = undistort(img)
        assert out.shape == tuple(GOLD[name + "__img_shape"][k]) and _sha(out) == GOLD[name + "__img_sha"][k].tobytes(), (name, k)


def test_libm_is_the_recording_machines():
    """the record's tables come from this libm's tanf / atanf: a machine whose libm rounds them otherwise fails here, naming libm,
    and not below naming the library"""
    tanf, atanf = mg.libm_values()
    assert tanf.tobytes() == GOLD["libm_tanf"].tobytes() and atanf.tobytes() == GOLD["libm_atanf"].tobytes(), \
        "libm's tanf / atanf differ from the libm the UndistorterPTAM record was made with (glibc 2.39, x86-64)"


def test_record_covers_the_sweep():
    """the record is of this case list; it holds the rounding-resistant entries (:299-301), the NaN cases, truncated whites and
    the malformed files' verdicts"""
    assert sorted(k[:-len("__file")] for k in GOLD.files if k.endswith("__file")) == sorted(CASES)
    for name in CASES:
        assert GOLD[name + "__file"].tobytes() == TEXT[name].encode(), name
    assert len(CASES) >= 30
    for name in mg.ROUNDING_CASES:
        ic, in_size, oc, out_size = mg.parse(TEXT[name])
        u = po.UndistorterPTAM(ic, in_size, oc, out_size)
        _check_tables(name, u.remapX, u.remapY, u.K)
        assert (u.remapX == np.float32(0.01)).any() or (u.remapY == np.float32(0.01)).any(), name
        assert (u.remapX == np.float32(in_size[0] - 1.01)).any(), name
    for name in ("nan_full_cx0_cy0", "nan_crop_cx0"):
        _, _, (ow, oh), n_invalid, _ = _info(name)
        assert n_invalid == ow * oh and np.isnan(GOLD[name + "__K"]).sum() == 1, name
    white = GOLD["fov_crop_same__img_sha"][2].tobytes()
    assert white != _sha(np.full((480, 640), 255, np.uint8))            # truncation leaves 254s in a constant-255 image
    verdicts = {n: _info(n)[0:1] + (_info(n)[4],) for n in CASES if n.startswith("bad_") or n == "opencv8"}
    assert verdicts == {"bad_trailing_blank": (0, 0), "bad_crlf": (0, 0), "bad_missing_line4": (0, 0), "bad_four_numbers": (0, 0),
                        "bad_six_numbers": (1, 1), "opencv8": (1, 2)}, verdicts


@pytest.mark.parametrize("name", VALID)
def test_c_oracle_matches_reference_record(name):
    ic, in_size, oc, out_size = mg.parse(TEXT[name])
    u = po.UndistorterPTAM(ic, in_size, oc, out_size)
    assert u.status == (1 if in_size == out_size and ic[4] == 0 else 0)
    _check_tables(name, u.remapX, u.remapY, u.K)
    _check_images(name, u.undistort, in_size)


@pytest.mark.parametrize("name", VALID)
def test_library_table_builder_matches_reference_record(name):
    ic, in_size, oc, out_size = mg.parse(TEXT[name])
    u = abi.UndistorterPTAM(ic, in_size, oc, out_size)
    assert u.status == (1 if in_size == out_size and ic[4] == 0 else 0)
    _check_tables(name, u.remapX, u.remapY, u.K)
    if u.status == 0:
        assert abi.load().lsdgpu_undistorter_validate_tables(*in_size, *out_size, u.remapX.ctypes.data_as(abi._fp),
                                                              u.remapY.ctypes.data_as(abi._fp)) == 0


@pytest.fixture(scope="module")
def cfg_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("calib")
    for name, text in mg.cases():
        mg.write_case(str(d), name, text)
    return d


@pytest.mark.parametrize("name", CASES)
def test_live_reference_matches_record(name, cfg_dir):
    """the reference's class on the file (and, for valid files, on the parsed lines) gives the record; so does
    getUndistorterForFile's verdict, and the legacy-math build's distance"""
    if not po.ref_available():
        pytest.skip("oracle/_ref is not built here")
    path = os.path.join(str(cfg_dir), name + ".cfg")
    valid, in_size, out_size, n_invalid, verdict = _info(name)
    r = po.RefUndistorterFile(path)
    assert (r.valid, (r.in_w, r.in_h), (r.out_w, r.out_h)) == (bool(valid), in_size, out_size)
    assert _same_bits(_k4(r.K), GOLD[name + "__K"])
    if name not in mg.OPENCV_DISPATCH:
        assert po.ref_undistorter_for_file(path) == verdict
    if not valid:
        assert r.remapX is None
        return
    _check_tables(name, r.remapX, r.remapY, r.K)
    _check_images(name, r.undistort, in_size)
    ic, _, oc, _ = mg.parse(TEXT[name])
    p = po.UndistorterPTAM(ic, in_size, oc, out_size, fast="ref")
    _check_tables(name, p.remapX, p.remapY, p.K)
    _check_images(name, p.undistort, in_size)
    leg = po.RefUndistorterFile(path, "ref_legacy_math")
    dpix, dmax = [], []
    for img in mg.raw_images(*in_size):
        a, b = r.undistort(img).astype(np.int32), leg.undistort(img).astype(np.int32)
        dpix.append(int((a != b).sum()))
        dmax.append(int(np.abs(a - b).max()))
    got = [int((r.remapX.view(np.int32) != leg.remapX.view(np.int32)).sum()), int((r.remapY.view(np.int32) != leg.remapY.view(np.int32)).sum()),
           int((r.K.view(np.int32) != leg.K.view(np.int32)).sum())] + dpix + dmax
    assert got == GOLD[name + "__legacy"].tolist(), (name, got)


def test_legacy_math_distance():
    """the float overloads (liblsd_ref.so, the library) against tan / atan / sqrt on doubles (liblsd_ref_legacy_math.so): the
    distance DESIGN.md §5 states, as recorded"""
    leg = {n: GOLD[n + "__legacy"] for n in VALID}
    assert leg["fov_crop_same"][:3].tolist() == [56880, 264162, 2]                   # remapX, remapY entries, K values (fy, cy)
    assert leg["fov_crop_same"][3] == 691 and leg["fov_crop_1280"][:2].tolist() == [228536, 1053681]
    assert all(leg[n].sum() == 0 for n in ("w0_same", "w0_down", "w0_up", "w0_centred_same"))    # no tan / atan without distortion
    assert all(leg[n][:2].sum() > 0 for n in VALID if mg.parse(TEXT[n])[0][4] != 0 and _info(n)[3] < np.prod(_info(n)[2]))


@pytest.fixture(scope="module")
def demo():
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    return build.DEMO_OUT


def _run(demo, mode, path, tables):
    r = subprocess.run([demo, mode, path, tables], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip().splitlines()


@pytest.mark.parametrize("name", CASES)
def test_adapter_reads_files_as_the_reference(name, cfg_dir, demo, tmp_path):
    """lsd_slam::UndistorterPTAM(configFileName) and getUndistorterForFile of the C++ adapter give the reference's verdict and,
    for a file the reference accepts, its sizes, K and tables.  One recorded difference: the reference's PTAM constructor reads
    the first five numbers of an OpenCV-model line, the adapter's refuses the file (getUndistorterForFile agrees on both)."""
    path = os.path.join(str(cfg_dir), name + ".cfg")
    tables = str(tmp_path / "tables.bin")
    valid, in_size, out_size, _, verdict = _info(name)

    def check(l1, l2, at):
        assert [int(v) for v in l1[at:at + 4]] == [*in_size, *out_size], (name, l1)
        K = np.array([float(v) for v in l2.split()], np.float32)
        t = np.fromfile(tables, np.float32).reshape(2, out_size[1], out_size[0])
        _check_tables(name, t[0], t[1], K)

    lines = _run(demo, "--undistorter", path, tables)
    l1 = lines[0].split()
    if name in mg.OPENCV_DISPATCH:
        assert valid == 1 and l1[0] == "0"
    else:
        assert int(l1[0]) == valid, (name, l1)
        if valid:
            ic = mg.parse(TEXT[name])[0]
            assert int(l1[1]) == (1 if in_size == out_size and ic[4] == 0 else 0)
            check(l1, lines[1], 2)
    lines = _run(demo, "--undistorter-any", path, tables)
    l1 = lines[0].split()
    if verdict == 0:
        assert l1 == ["0"], (name, lines)
    elif verdict == 2:
        assert l1[:2] == ["1", "1"], (name, lines)
    else:
        assert l1[:2] == ["1", "0"], (name, lines)
        check(l1, lines[1], 2)
