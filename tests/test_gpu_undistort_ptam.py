"""UndistorterPTAM on the device at the calibrations of the reference pin (tests/golden/ref_pin_undistort.npz, recorded from the
reference's own util/Undistorter.cpp): undistort() and the fused undistort + Frame construction (k_undistort and
k_image_pyramid<PYR_PTAM>, both through undistortPixel) give the reference's images bit for bit, from host memory and from a
device image whose row pitch exceeds its width; the frame built on it equals oracle.Frame; and a 10-frame track-and-map run on
distorted frames agrees with the oracle fed the undistorted ones."""
import hashlib

import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests.golden import make_golden_ref_pin_undistort as mg

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GOLD = np.load(mg.OUT)
TEXT = dict(mg.cases())
LEVELS = 5


def _info(name):
    valid, iw, ih, ow, oh, n_invalid, verdict = (int(v) for v in GOLD[name + "__info"])
    return valid, (iw, ih), (ow, oh), n_invalid


# every recorded file the reference accepts whose output size a context takes (multiples of 16, SlamSystem.cpp:55)
DEVICE_CASES = [n for n, _ in mg.cases() if _info(n)[0] == 1 and _info(n)[2][0] % 16 == 0 and _info(n)[2][1] % 16 == 0]
FINITE_K = np.array([[277.5, 0, 319.5], [0, 291.5, 239.5], [0, 0, 1]], np.float32)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def _cuda(img, extra):
    """img as a uint8 CUDA tensor view whose row pitch is `extra` bytes larger than its width"""
    h, w = img.shape
    t = torch.zeros((h, w + extra), dtype=torch.uint8, device="cuda")
    t[:, :w] = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    return t[:, :w]


def _planes(ctx, fid):
    out = [ctx.download(fid, abi.BUF_IMAGE, lvl).tobytes() for lvl in range(LEVELS)]
    out += [ctx.download(fid, abi.BUF_GRADIENTS, lvl).tobytes() for lvl in range(LEVELS)]
    return out + [ctx.download(fid, abi.BUF_MAXGRAD, 0).tobytes()]


def test_device_cases_cover_the_sweep():
    assert len(DEVICE_CASES) >= 25
    assert {"nan_full_cx0_cy0", "nan_crop_cx0", "w0_same", "tiny64", "raw1241_crop", "fov_full_1280"} <= set(DEVICE_CASES)


@pytest.mark.parametrize("name", DEVICE_CASES)
def test_undistort_and_fused_frame_match_reference(name, oracle):
    _, in_size, out_size, n_invalid = _info(name)
    u = abi.UndistorterPTAM(*mg.parse(TEXT[name]))
    K = u.getK()
    if not np.isfinite(K).all():
        # the reference's K is NaN here (compared on the CPU by tests/test_ref_pin_undistort.py); its tables are all -1
        assert n_invalid == out_size[0] * out_size[1]
        K = FINITE_K
    ctx = abi.Context(*out_size, K, max_frames=4)
    try:
        u.install(ctx)
        for k, raw in enumerate(mg.raw_images(*in_size)):
            img = ctx.undistort(raw)
            assert img.shape == tuple(GOLD[name + "__img_shape"][k]) and _sha(img) == GOLD[name + "__img_sha"][k].tobytes(), (name, k)
            if n_invalid == img.size:
                assert not img.any()
            ctx.upload_distorted(0, raw)
            assert np.array_equal(ctx.download(0, abi.BUF_IMAGE, 0), img.astype(np.float32)), (name, k)
            of = oracle.Frame(0, img, K)
            for lvl in range(1, LEVELS):
                assert np.array_equal(ctx.download(0, abi.BUF_IMAGE, lvl), of.image(lvl)), (name, k, lvl)
                assert np.array_equal(ctx.download(0, abi.BUF_GRADIENTS, lvl)[..., :3], of.gradients(lvl)[..., :3]), (name, k, lvl)
            assert np.array_equal(ctx.download(0, abi.BUF_GRADIENTS, 0)[..., :3], of.gradients(0)[..., :3]), (name, k)
            assert np.array_equal(ctx.download(0, abi.BUF_MAXGRAD, 0), of.maxGradients(0)), (name, k)
            ctx.upload_distorted(1, _cuda(raw, 5 + k))
            assert _planes(ctx, 1) == _planes(ctx, 0), (name, k)
            ctx.release(0)
            ctx.release(1)
    finally:
        ctx.close()


def _distort_frames(seq, frames, calib, in_size):
    """raw images of an ATAN (FOV-model) camera `calib` (relative units, Undistorter.cpp:177-180) looking at the rendered scene:
    a raw pixel at distorted radius rd sees the undistorted direction of radius tan(rd * w) / (2 tan(w / 2)), projected with
    the scene's camera.  Approximate (bilinear); both legs of the test see the same raw bytes."""
    iw, ih = in_size
    c = [float(v) for v in np.float32(calib)]
    fx, fy, cx, cy, w = c[0] * iw, c[1] * ih, c[2] * iw - 0.5, c[3] * ih - 0.5, c[4]
    v, u = np.mgrid[0:ih, 0:iw].astype(np.float64)
    xd, yd = (u - cx) / fx, (v - cy) / fy
    rd = np.hypot(xd, yd)
    s = np.where(rd > 0, np.tan(rd * w) / (2 * np.tan(w / 2)) / np.maximum(rd, 1e-12), 1.0)
    Ks = seq.K.astype(np.float64)
    su, sv = Ks[0, 0] * xd * s + Ks[0, 2], Ks[1, 1] * yd * s + Ks[1, 2]
    h, wd = seq.h, seq.w
    x0, y0 = np.clip(np.floor(su).astype(int), 0, wd - 2), np.clip(np.floor(sv).astype(int), 0, h - 2)
    ax, ay = np.clip(su - x0, 0, 1), np.clip(sv - y0, 0, 1)
    raws = []
    for img in frames:
        f = img.astype(np.float64)
        val = f[y0, x0] * (1 - ax) * (1 - ay) + f[y0, x0 + 1] * ax * (1 - ay) + f[y0 + 1, x0] * (1 - ax) * ay + f[y0 + 1, x0 + 1] * ax * ay
        raws.append(np.clip(np.rint(val), 0, 255).astype(np.uint8))
    return raws


def test_track_and_map_on_distorted_frames(oracle, seq_small, frames_small):
    """10 frames, GT-depth init, through PYR_PTAM: upload_distorted + se3_track + depth_update_keyframe gives the poses and depth
    maps of the same calls fed with host-undistorted frames; and the host leg agrees with the oracle fed the same undistorted
    images and getK(): every pose to 1e-4 plus the reference's own summation noise on that step, every map bit for bit when the
    oracle maps with the device's pose, residual and good mask.  The output camera is the scene's own (an explicit output
    calibration), so the rendered depth is the undistorted frame's depth."""
    from tests.pin_cases import set_depth
    from tests.util import hyp_equal_report, pose_err
    seq = seq_small
    K = seq.K.astype(np.float64)
    w, h = seq.w, seq.h
    calib = [K[0, 0] / w * 1.04, K[1, 1] / h * 1.03, (K[0, 2] + 2.0) / w, (K[1, 2] - 1.5) / h, 0.7]
    out_calib = [K[0, 0] / w, K[1, 1] / h, (K[0, 2] + 0.5) / w, (K[1, 2] + 0.5) / h, 0]
    u = abi.UndistorterPTAM(calib, (w, h), out_calib, (w, h))
    ou = oracle.UndistorterPTAM(calib, (w, h), out_calib, (w, h))
    Ku = u.getK()
    assert u.status == 0 and np.abs(Ku - seq.K).max() < 1e-3 and (u.remapX >= 0).mean() > 0.9
    imgs = [frames_small[k][0] for k in range(10)]
    raws = _distort_frames(seq, imgs, calib, (w, h))
    depth0 = frames_small[0][1]
    legs = {}
    L = oracle.lib()
    for leg in ("fused", "host"):
        ctx = abi.Context(w, h, Ku, max_frames=12)
        u.install(ctx)
        trk, dm = abi.SE3Tracker(ctx, mode=1), abi.DepthMap(ctx)
        poses, maps = [], []
        last = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
        keep = []
        for k, raw in enumerate(raws):
            img = ou.undistort(raw)
            if leg == "fused":
                ctx.upload_distorted(k, raw)
            else:
                ctx.upload(k, img)
            if k == 0:
                ctx.set_depth_gt(0, depth0)
                dm.initializeFromGTDepth(0)
                if leg == "host":
                    okf = oracle.Frame(0, img, Ku)
                    okf.setDepthFromGroundTruth(depth0)
                    odm = oracle.DepthMap(w, h, Ku)
                    odm.initializeFromGTDepth(okf)
                    img0 = img
                continue
            if k == 1 or ctx.depth_updated_flag(0):
                trk.importFrame(0)
            pose = trk.trackFrame(0, k, last)
            poses.append((pose.tobytes(), trk.trackingWasGood))
            counters = ctx.get_counters(0)
            if leg == "host":
                L.lsdo_frame_set_depthHasBeenUpdatedFlag(okf.ptr, 0)
                oracle.set_globals(exactTrackingSums=1)
                try:
                    xkf = oracle.Frame(0, img0, Ku)
                    if k == 1:
                        xkf.setDepthFromGroundTruth(depth0)
                    else:
                        set_depth(xkf, odm.current())
                    rx = oracle.se3_track(xkf, oracle.Frame(k, img, Ku), last)
                finally:
                    oracle.set_globals()
                of = oracle.Frame(k, img, Ku)
                keep.append(of)
                r = oracle.se3_track(okf, of, last)
                assert bool(r.trackingWasGood) == trk.trackingWasGood and not r.diverged, k
                dt, ang = pose_err(pose, r.frameToRef_qt)
                nt, na = pose_err(r.frameToRef_qt, rx.frameToRef_qt)
                assert dt <= 1e-4 + nt and ang <= 1e-6 + na, (k, dt, nt, ang, na)
                qts, _, itr = ctx.get_pose(k)
                of.set_thisToParent(np.array(qts, np.float64), okf)
                L.lsdo_frame_set_initialTrackedResidual(of.ptr, float(itr))
                of.refPixelWasGood(create=True)[:] = ctx.download(k, abi.BUF_GOODMASK)
                L.lsdo_frame_set_counters(okf.ptr, int(counters[0]), int(counters[1]))
            dm.updateKeyframe([k])
            ctx.clear_good_mask(k)
            maps.append(dm.current().tobytes())
            if leg == "host":
                odm.updateKeyframe([of])
                L.lsdo_frame_clear_refPixelWasGood(of.ptr)
                rep = hyp_equal_report(dm.current(), odm.current())
                assert rep["n_valid"] > 3000 and all(v == 0 for key, v in rep.items() if key.endswith(("mismatch", "bitdiff"))), (k, rep)
            last = pose
        legs[leg] = (poses, maps)
        ctx.close()
    assert legs["fused"][0] == legs["host"][0]
    assert legs["fused"][1] == legs["host"][1]
    assert sum(good for _, good in legs["fused"][0]) >= 5          # the run tracks: the distortion model is consistent
