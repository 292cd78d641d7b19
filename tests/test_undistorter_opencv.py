"""UndistorterOpenCV (util/Undistorter.cpp:449-567): the library's host-side table builder and the tests' C restatement against
what OpenCV 4.13 computes (tests/golden/opencv_undistort.npz, CPU), the C++ adapter's file parsing and model dispatch (CPU), and
-- on the GPU -- the device remap, the fused undistort + Frame construction, switching models on one context and a short
track + map run fed with distorted frames."""
import os
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import undistort_opencv_oracle as cvo
from tests.golden import make_golden_opencv_undistort as mg

GOLD = np.load(mg.OUT)
CASES = mg.cases()
IDS = [c[0] for c in CASES]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold(i):
    return {k: GOLD[k][i] for k in ("K_new", "K_out", "crc_map1", "crc_map2", "crc_remap")}


def test_fixture_lists_the_cases():
    assert list(GOLD["name"]) == IDS
    assert np.array_equal(GOLD["calib"], np.array([np.float32(c[1]) for c in CASES]))
    assert len(CASES) >= 27


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_library_tables_equal_opencv(i):
    name, calib, in_size, mode, out_size = CASES[i]
    g = _gold(i)
    u = abi.UndistorterOpenCV(calib, in_size, mode, out_size)
    assert u.status == 0
    assert u.K_new.ravel().tobytes() == g["K_new"].tobytes()
    assert u.getK().ravel().tobytes() == g["K_out"].tobytes()
    assert mg.crc(u.map1) == g["crc_map1"] and mg.crc(u.map2) == g["crc_map2"]
    if name == mg.SMALL:
        assert np.array_equal(u.map1, GOLD["small_map1"]) and np.array_equal(u.map2, GOLD["small_map2"])


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_oracle_tables_and_remap_equal_opencv(i):
    name, calib, in_size, mode, out_size = CASES[i]
    g = _gold(i)
    u = cvo.UndistorterOpenCV(calib, in_size, mode, out_size)
    assert u.status == 0
    assert u.K_new.ravel().tobytes() == g["K_new"].tobytes() and u.K.ravel().tobytes() == g["K_out"].tobytes()
    assert mg.crc(u.map1) == g["crc_map1"] and mg.crc(u.map2) == g["crc_map2"]
    for s, want in zip(mg.RAW_SEEDS, g["crc_remap"]):
        assert mg.crc(u.undistort(mg.raw_image(*in_size, s))) == want


def test_remap_border_and_weights():
    """the oracle's remap on hand-made maps: exact weights, constant-0 border per tap, map2 read modulo 1024"""
    raw = np.full((4, 4), 200, np.uint8)
    m1 = np.array([[[1, 1], [-1, 1], [3, 3], [9, 9], [1, 1]]], np.int16)
    m2 = np.array([[16 * 32 + 16, 16 * 32 + 16, 16 * 32 + 16, 0, 1024 + 16 * 32 + 16]], np.uint16)
    out = cvo.remap(raw, m1, m2)
    assert list(out[0]) == [200, 100, 50, 0, 200]


def test_invalid_modes_and_sizes_return_minus_2():
    import ctypes as C
    L = abi.load()
    ic = np.float32(mg.TUM_FR1)
    fp = ic.ctypes.data_as(C.POINTER(C.c_float))
    for mode, iw, ow in ((0, 640, 640), (-3, 640, 640), (1, 640, 640), (-1, 0, 640), (-2, 640, 0)):
        assert L.lsdgpu_undistorter_opencv_prepare(fp, iw, 480, mode, ow, 480, None, None, None, None) == -2
        assert cvo.lib().lsdo_cv_prepare(fp, iw, 480, mode, ow, 480, None, None, None, None) == -2
    assert L.lsdgpu_undistorter_opencv_prepare(fp, 640, 480, -1, 640, 480, None, None, None, None) == 0
    assert abi.UndistorterOpenCV(mg.TUM_FR1, (640, 480), "none", (640, 480)).status == -2
    with pytest.raises(abi.LsdGpuError):
        abi.UndistorterOpenCV(mg.TUM_FR1, (640, 480), "none", (640, 480)).install(None)


def test_live_cross_check_against_cv2():
    """the seeded calibrations (and a fresh draw of them) against the cv2 module itself, when it is importable"""
    cv2 = pytest.importorskip("cv2")
    for name, calib, in_size, mode, out_size in mg.random_cases() + mg.random_cases(8, seed=7):
        K_new, K_out, map1, map2 = mg.opencv_tables(cv2, calib, in_size, mode, out_size)
        u = abi.UndistorterOpenCV(calib, in_size, mode, out_size)
        assert u.K_new.tobytes() == K_new.tobytes(), name
        assert np.array_equal(u.map1, map1) and np.array_equal(u.map2, map2), name
        raw = mg.raw_image(*in_size, 5)
        assert np.array_equal(cvo.remap(raw, u.map1, u.map2), cv2.remap(raw, map1, map2, cv2.INTER_LINEAR)), name


def _demo(args):
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    r = subprocess.run([build.DEMO_OUT] + [str(a) for a in args], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip().splitlines()


def test_adapter_file_parser_and_dispatcher(tmp_path):
    """lsd_slam::UndistorterOpenCV(configFileName) and getUndistorterForFile of the C++ adapter -- host-only, no GPU"""
    cfg, tables = tmp_path / "cam.cfg", tmp_path / "tables.bin"
    for name in ("tum_fr1_crop", "euroc_full", "relative_crop", "example_crop"):
        i = IDS.index(name)
        _, calib, (iw, ih), mode, (ow, oh) = CASES[i]
        cfg.write_text(" ".join(repr(float(v)) for v in np.float32(calib)) + "\n%d %d\n%s\n%d %d\n" % (iw, ih, mode, ow, oh))
        l1, l2 = _demo(["--undistorter-any", cfg, tables])
        assert [int(v) for v in l1.split()] == [1, 1, iw, ih, ow, oh]
        assert np.array_equal(np.float32(l2.split()), GOLD["K_out"][i])
        t = np.fromfile(tables, np.uint8)
        assert mg.crc(t[:ow * oh * 4]) == GOLD["crc_map1"][i] and mg.crc(t[ow * oh * 4:]) == GOLD["crc_map2"][i]
        # the PTAM class still turns the file away
        assert _demo(["--undistorter", cfg, tables])[0].split()[0] == "0"
    # "none" / explicit output parameters: the reference's undistorter is invalid and the dispatcher returns null
    for l3 in ("none", "0.5 0.5 0.5 0.5 0"):
        cfg.write_text("517.3 516.5 318.6 255.3 0.2624 -0.9531 -0.0054 0.0026\n640 480\n%s\n640 480\n" % l3)
        assert _demo(["--undistorter-any", cfg, tables]) == ["0"]
    # a PTAM file goes to UndistorterPTAM: same output as --undistorter
    fov = [0.535719308086809, 0.669566858850269, 0.493248545285398, 0.500408664348414, 0.897966326944875]
    cfg.write_text(" ".join(repr(v) for v in fov) + "\n752 480\ncrop\n640 480\n")
    any_out = _demo(["--undistorter-any", cfg, tables])
    any_tables = tables.read_bytes()
    ptam_out = _demo(["--undistorter", cfg, tables])
    assert any_out[0].split() == ["1", "0", "752", "480", "640", "480"] and any_out[1] == ptam_out[1]
    assert any_tables == tables.read_bytes()


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _frame_bytes(ctx, fid):
    return [ctx.download(fid, abi.BUF_IMAGE, lvl).tobytes() for lvl in range(5)] + \
           [ctx.download(fid, abi.BUF_GRADIENTS, 0).tobytes(), ctx.download(fid, abi.BUF_MAXGRAD, 0).tobytes()]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_gpu_undistort_and_fused_frame_bit_exact(oracle, i):
    name, calib, in_size, mode, out_size = CASES[i]
    g = _gold(i)
    u = abi.UndistorterOpenCV(calib, in_size, mode, out_size)
    ow, oh = out_size
    ctx = abi.Context(ow, oh, u.getK(), max_frames=4)
    u.install(ctx)
    for s, want_crc in zip(mg.RAW_SEEDS, g["crc_remap"]):
        raw = mg.raw_image(*in_size, s)
        want = cvo.remap(raw, u.map1, u.map2)
        got = ctx.undistort(raw)
        assert mg.crc(got) == want_crc and np.array_equal(got, want)
    raw = mg.raw_image(*in_size, mg.RAW_SEEDS[0])
    want = cvo.remap(raw, u.map1, u.map2)
    ctx.upload_distorted(7, raw)
    of = oracle.Frame(7, want, u.getK())
    for lvl in range(5):
        assert np.array_equal(ctx.download(7, abi.BUF_IMAGE, lvl), of.image(lvl)), lvl
    assert np.array_equal(ctx.download(7, abi.BUF_GRADIENTS, 0)[..., :3], of.gradients(0)[..., :3])
    assert np.array_equal(ctx.download(7, abi.BUF_MAXGRAD, 0), of.maxGradients(0))
    ctx.upload(8, want)                                  # the plain path on the undistorted image gives the same frame
    assert _frame_bytes(ctx, 8) == _frame_bytes(ctx, 7)
    ctx.close()


@pytest.mark.gpu
def test_gpu_switching_models_matches_fresh_contexts():
    """PTAM -> OpenCV -> PTAM on one context: each install gives the bytes of a fresh context with that model"""
    fov = [0.535719308086809, 0.669566858850269, 0.493248545285398, 0.500408664348414, 0.897966326944875]
    ptam = abi.UndistorterPTAM(fov, (752, 480), "crop", (640, 480))
    ocv = abi.UndistorterOpenCV(mg.EUROC, (752, 480), "full", (640, 480))
    raw = mg.raw_image(752, 480, 1)

    def run(ctx, u):
        u.install(ctx)
        ctx.upload_distorted(0, raw)
        out = [ctx.undistort(raw).tobytes()] + _frame_bytes(ctx, 0)
        ctx.release(0)
        return out
    fresh = {}
    for key, u in (("ptam", ptam), ("ocv", ocv)):
        c = abi.Context(640, 480, ptam.getK(), max_frames=2)
        fresh[key] = run(c, u)
        c.close()
    assert fresh["ptam"] != fresh["ocv"]
    ctx = abi.Context(640, 480, ptam.getK(), max_frames=2)
    for key, u in (("ptam", ptam), ("ocv", ocv), ("ptam", ptam)):
        assert run(ctx, u) == fresh[key], key
    ctx.close()


def _distort_frames(seq, frames, calib, in_size, K_new, out_size):
    """raw images of a camera with the OpenCV model `calib` looking at the rendered scene, and the rendered depth resampled onto
    the undistorted (K_new) grid.  Approximate (nearest depth, bilinear image): both legs of the test see the same raw bytes."""
    iw, ih = in_size
    fx, fy, cx, cy, k1, k2, p1, p2 = [float(v) for v in np.float32(calib)]
    Ks = seq.K.astype(np.float64)
    v, u = np.mgrid[0:ih, 0:iw].astype(np.float64)
    xd, yd = (u - cx) / fx, (v - cy) / fy
    x, y = xd.copy(), yd.copy()
    for _ in range(10):                                   # undistortPoints' fixed-point iteration
        r2 = x * x + y * y
        icd = 1 / (1 + (k2 * r2 + k1) * r2)
        x = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) * icd
        y = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) * icd
    su, sv = Ks[0, 0] * x + Ks[0, 2], Ks[1, 1] * y + Ks[1, 2]
    h, w = seq.h, seq.w
    x0, y0 = np.clip(np.floor(su).astype(int), 0, w - 2), np.clip(np.floor(sv).astype(int), 0, h - 2)
    ax, ay = np.clip(su - x0, 0, 1), np.clip(sv - y0, 0, 1)
    raws = []
    for img in frames:
        f = img.astype(np.float64)
        val = (f[y0, x0] * (1 - ax) * (1 - ay) + f[y0, x0 + 1] * ax * (1 - ay) + f[y0 + 1, x0] * (1 - ax) * ay + f[y0 + 1, x0 + 1] * ax * ay)
        raws.append(np.clip(np.rint(val), 0, 255).astype(np.uint8))
    ow, oh = out_size
    q, p = np.mgrid[0:oh, 0:ow].astype(np.float64)
    du = np.rint(Ks[0, 0] * (p - K_new[0, 2]) / K_new[0, 0] + Ks[0, 2]).astype(int)
    dv = np.rint(Ks[1, 1] * (q - K_new[1, 2]) / K_new[1, 1] + Ks[1, 2]).astype(int)
    return raws, (np.clip(du, 0, w - 1), np.clip(dv, 0, h - 1))


@pytest.mark.gpu
def test_gpu_track_and_map_on_distorted_frames(seq_small, frames_small):
    """10 frames, GT-depth init: upload_distorted + se3_track + depth_update_keyframe gives the poses and depth maps of the same
    calls fed with host-undistorted frames"""
    seq = seq_small
    K = seq.K.astype(np.float64)
    calib = [K[0, 0] * 1.02, K[1, 1] * 1.02, K[0, 2] + 1.5, K[1, 2] - 1.0, -0.18, 0.05, 0.0007, -0.0004]
    in_size = out_size = (seq.w, seq.h)
    u = abi.UndistorterOpenCV(calib, in_size, "crop", out_size)
    imgs = [frames_small[k][0] for k in range(10)]
    raws, (du, dv) = _distort_frames(seq, imgs, calib, in_size, u.K_new, out_size)
    depth0 = frames_small[0][1][dv, du]
    legs = {}
    for leg in ("fused", "host"):
        ctx = abi.Context(seq.w, seq.h, u.getK(), max_frames=12)
        u.install(ctx)
        trk, dm = abi.SE3Tracker(ctx, mode=1), abi.DepthMap(ctx)
        poses, maps = [], []
        last = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
        for k, raw in enumerate(raws):
            if leg == "fused":
                ctx.upload_distorted(k, raw)
            else:
                ctx.upload(k, cvo.remap(raw, u.map1, u.map2))
            if k == 0:
                ctx.set_depth_gt(0, depth0)
                dm.initializeFromGTDepth(0)
                continue
            if k == 1 or ctx.depth_updated_flag(0):
                trk.importFrame(0)
            pose = trk.trackFrame(0, k, last)
            poses.append((pose.tobytes(), trk.trackingWasGood))
            dm.updateKeyframe([k])
            ctx.clear_good_mask(k)
            maps.append(dm.current().tobytes())
            last = pose
        legs[leg] = (poses, maps)
        ctx.close()
    assert legs["fused"][0] == legs["host"][0]
    assert legs["fused"][1] == legs["host"][1]
    assert sum(good for _, good in legs["fused"][0]) >= 5          # the run tracks: the distortion model is consistent
