"""ctypes binding of the CPU ORACLE (oracle/lsd_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference`` legs import this.

Flavours (the ``fast`` argument everywhere): False = strict-IEEE C restatement (parity), True = its -O3 timing build,
"ref" = oracle/_ref/liblsd_ref.so and "ref_sse" = oracle/_ref/liblsd_ref_sse.so -- the reference's own sources compiled
unmodified (oracle/ref_build.py, oracle/ref_driver.cpp) behind the same C names; entry points the reference-compiled
library does not export are simply absent there.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 5


class Hyp(C.Structure):
    _fields_ = [("isValid", C.c_uint8), ("_pad", C.c_uint8 * 3), ("blacklisted", C.c_int32),
                ("nextStereoFrameMinID", C.c_float), ("validity_counter", C.c_int32),
                ("idepth", C.c_float), ("idepth_var", C.c_float),
                ("idepth_smoothed", C.c_float), ("idepth_var_smoothed", C.c_float)]


HYP_DTYPE = np.dtype([("isValid", np.uint8), ("_pad", np.uint8, 3), ("blacklisted", np.int32),
                      ("nextStereoFrameMinID", np.float32), ("validity_counter", np.int32),
                      ("idepth", np.float32), ("idepth_var", np.float32),
                      ("idepth_smoothed", np.float32), ("idepth_var_smoothed", np.float32)])
assert HYP_DTYPE.itemsize == 32 and C.sizeof(Hyp) == 32


POINT_DENSE = np.dtype([("idepth", np.float32), ("idepth_var", np.float32), ("color", np.uint8, (4,))])     # InputPointDense


class Globals(C.Structure):
    _fields_ = [("minUseGrad", C.c_float), ("cameraPixelNoise2", C.c_float), ("depthSmoothingFactor", C.c_float),
                ("allowNegativeIdepths", C.c_int), ("useSubpixelStereo", C.c_int),
                ("useAffineLightningEstimation", C.c_int), ("multiThreading", C.c_int), ("useSSE", C.c_int),
                ("exactAffineSums", C.c_int), ("exactTrackingSums", C.c_int), ("exactSim3Sums", C.c_int)]


class TrackSettings(C.Structure):
    _fields_ = [("lambdaSuccessFac", C.c_float), ("lambdaFailFac", C.c_float),
                ("lambdaInitial", C.c_float * LEVELS), ("stepSizeMin", C.c_float * LEVELS),
                ("convergenceEps", C.c_float * LEVELS), ("maxItsPerLvl", C.c_int * LEVELS),
                ("huber_d", C.c_float), ("var_weight", C.c_float)]


class TrackResult(C.Structure):
    _fields_ = [("frameToRef_qt", C.c_double * 7),
                ("pointUsage", C.c_float), ("lastGoodCount", C.c_float), ("lastBadCount", C.c_float),
                ("lastMeanRes", C.c_float), ("lastResidual", C.c_float),
                ("affineEstimation_a", C.c_float), ("affineEstimation_b", C.c_float),
                ("diverged", C.c_int), ("trackingWasGood", C.c_int),
                ("numCalcResidualCalls", C.c_int * LEVELS), ("numCalcWarpUpdateCalls", C.c_int * LEVELS),
                ("initialTrackedResidual", C.c_float)]


class EvalResult(C.Structure):
    _fields_ = [("A", C.c_float * 36), ("b", C.c_float * 6), ("lsError", C.c_float),
                ("meanWeightedRes", C.c_float), ("meanUnweightedRes", C.c_float), ("warpedSize", C.c_int),
                ("pointUsage", C.c_float), ("goodCount", C.c_float), ("badCount", C.c_float), ("meanRes", C.c_float),
                ("affine_a_lastIt", C.c_float), ("affine_b_lastIt", C.c_float),
                ("sxx", C.c_float), ("syy", C.c_float), ("sx", C.c_float), ("sy", C.c_float), ("sw", C.c_float)]


class Sim3Result(C.Structure):
    _fields_ = [("frameToRef_qts", C.c_double * 8), ("lastSim3Hessian", C.c_float * 49),
                ("lastResidual", C.c_float), ("lastDepthResidual", C.c_float), ("lastPhotometricResidual", C.c_float),
                ("pointUsage", C.c_float), ("affineEstimation_a", C.c_float), ("affineEstimation_b", C.c_float),
                ("diverged", C.c_int),
                ("numCalcResidualCalls", C.c_int * LEVELS), ("numCalcWarpUpdateCalls", C.c_int * LEVELS)]


class Sim3EvalResult(C.Structure):
    _fields_ = [("A", C.c_float * 49), ("b", C.c_float * 7), ("num_constraints", C.c_int),
                ("sumResD", C.c_float), ("sumResP", C.c_float), ("numTermsD", C.c_int), ("numTermsP", C.c_int),
                ("mean", C.c_float), ("meanD", C.c_float), ("meanP", C.c_float), ("warpedSize", C.c_int),
                ("pointUsage", C.c_float), ("affine_a_lastIt", C.c_float), ("affine_b_lastIt", C.c_float)]


def build(force: bool = False) -> None:
    """Compile the oracle with the committed Makefile (gcc only)."""
    if force or not (os.path.exists(os.path.join(_HERE, "liblsd_oracle.so"))
                     and os.path.exists(os.path.join(_HERE, "liblsd_oracle_fast.so"))):
        subprocess.run(["make", "-C", _HERE] + (["-B"] if force else []), check=True, capture_output=True)


def ref_available() -> bool:
    """oracle/_ref present (prebuilt, or buildable because /root/reference is here)?"""
    from oracle import ref_build
    return ref_build.built() or ref_build.available()


_libs: dict = {}
_REF_NAMES = {"ref": "liblsd_ref.so", "ref_sse": "liblsd_ref_sse.so", "ref_legacy_math": "liblsd_ref_legacy_math.so"}


def lib(fast=False):
    if isinstance(fast, str):
        name = os.path.join("_ref", _REF_NAMES[fast])
    else:
        name = "liblsd_oracle_fast.so" if fast else "liblsd_oracle.so"
    if name in _libs:
        return _libs[name]
    path = os.path.join(_HERE, name)
    if isinstance(fast, str):
        from oracle import ref_build
        if not ref_build.build():
            raise RuntimeError("oracle/_ref is not built and /root/reference is not available to build it")
    elif not os.path.exists(path):
        build()
    L = C.CDLL(path)
    fp, dp, ip, u8p, vp = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint8), C.c_void_p

    def sig(name, res, *args):
        try:
            f = getattr(L, name)
        except AttributeError:
            if isinstance(fast, str) or name.startswith("lsdo_ref_"):
                return                      # not exported by the reference-compiled library / only exported by it
            raise
        f.restype = res
        f.argtypes = list(args)

    sig("lsdo_default_globals", None, C.POINTER(Globals))
    sig("lsdo_set_globals", None, C.POINTER(Globals))
    sig("lsdo_get_globals", None, C.POINTER(Globals))
    sig("lsdo_default_track_settings", None, C.POINTER(TrackSettings))
    for s, t in (("d", dp), ("f", fp)):
        sig(f"lsdo_se3{s}_exp", None, t, t)
        sig(f"lsdo_se3{s}_mul", None, t, t, t)
        sig(f"lsdo_se3{s}_inverse", None, t, t)
        sig(f"lsdo_se3{s}_matrix", None, t, t, t)
    sig("lsdo_se3d_log", None, dp, dp)
    sig("lsdo_ldlt6_solve", C.c_int, fp, fp, fp)
    sig("lsdo_mat3_inverse", None, fp, fp)
    sig("lsdo_frame_create_u8", vp, C.c_int, C.c_int, C.c_int, fp, u8p)
    sig("lsdo_frame_destroy", None, vp)
    sig("lsdo_frame_id", C.c_int, vp)
    sig("lsdo_frame_width", C.c_int, vp, C.c_int)
    sig("lsdo_frame_height", C.c_int, vp, C.c_int)
    for n in ("image", "gradients", "maxGradients", "idepth", "idepthVar"):
        sig(f"lsdo_frame_{n}", fp, vp, C.c_int)
    sig("lsdo_frame_K", None, vp, C.c_int, fp, fp)
    sig("lsdo_frame_refPixelWasGood", u8p, vp)
    sig("lsdo_frame_refPixelWasGoodNoCreate", u8p, vp)
    sig("lsdo_frame_clear_refPixelWasGood", None, vp)
    sig("lsdo_frame_setDepthFromGroundTruth", None, vp, fp, C.c_float)
    sig("lsdo_frame_setDepth", None, vp, C.POINTER(Hyp))
    sig("lsdo_frame_numMappablePixels", C.c_int, vp)
    sig("lsdo_frame_meanIdepth", C.c_float, vp)
    sig("lsdo_frame_numPoints", C.c_int, vp)
    sig("lsdo_frame_depthHasBeenUpdatedFlag", C.c_int, vp)
    sig("lsdo_frame_set_depthHasBeenUpdatedFlag", None, vp, C.c_int)
    sig("lsdo_frame_initialTrackedResidual", C.c_float, vp)
    sig("lsdo_frame_set_initialTrackedResidual", None, vp, C.c_float)
    sig("lsdo_frame_get_thisToParent", None, vp, dp)
    sig("lsdo_frame_set_thisToParent", None, vp, dp, vp)
    sig("lsdo_frame_numFramesTrackedOnThis", C.c_int, vp)
    sig("lsdo_frame_numMappedOnThis", C.c_int, vp)
    sig("lsdo_frame_set_counters", None, vp, C.c_int, C.c_int)
    sig("lsdo_make_point_cloud", C.c_int, vp, C.c_int, fp, fp, fp, ip)
    sig("lsdo_frame_takeReActivationData", None, vp, C.POINTER(Hyp))
    sig("lsdo_frame_idepth_reAct", fp, vp)
    sig("lsdo_frame_idepthVar_reAct", fp, vp)
    sig("lsdo_frame_validity_reAct", u8p, vp)
    sig("lsdo_pack_pointcloud", None, vp, C.c_int, vp)
    sig("lsdo_se3_eval", C.c_int, vp, vp, C.c_int, fp, C.c_float, C.c_float, C.POINTER(TrackSettings), C.c_int, C.POINTER(EvalResult))
    sig("lsdo_se3_track", C.c_int, vp, vp, dp, C.POINTER(TrackSettings), C.POINTER(TrackResult))
    sig("lsdo_ldlt7_solve", C.c_int, fp, fp, fp)
    sig("lsdo_sim3d_exp", None, dp, dp)
    sig("lsdo_sim3d_mul", None, dp, dp, dp)
    sig("lsdo_sim3d_inverse", None, dp, dp)
    sig("lsdo_sim3_pose_constants", None, dp, fp, fp, fp)
    sig("lsdo_sim3_eval", C.c_int, vp, vp, C.c_int, dp, C.c_float, C.c_float, C.POINTER(TrackSettings), C.POINTER(Sim3EvalResult))
    sig("lsdo_sim3_track", C.c_int, vp, vp, dp, C.c_int, C.c_int, C.POINTER(TrackSettings), C.POINTER(Sim3Result))
    sig("lsdo_undistorter_ptam_prepare", C.c_int, fp, C.c_int, C.c_int, fp, C.c_int, C.c_int, fp, fp, fp)
    sig("lsdo_undistort", None, fp, fp, C.c_int, C.c_int, C.c_int, u8p, u8p)
    sig("lsdo_ref_undistorter_open", vp, C.c_char_p)
    sig("lsdo_ref_undistorter_close", None, vp)
    sig("lsdo_ref_undistorter_info", None, vp, ip, fp)
    sig("lsdo_ref_undistorter_tables", C.c_int, vp, fp, fp)
    sig("lsdo_ref_undistorter_undistort", C.c_int, vp, u8p, C.c_int, C.c_int, u8p, C.c_int)
    sig("lsdo_ref_undistorter_for_file", C.c_int, C.c_char_p)
    sig("lsdo_frame_setPermaRef", C.c_int, vp, fp, fp)
    sig("lsdo_checkPermaRefOverlap", C.c_float, C.c_int, C.c_int, fp, fp, C.c_int, dp)
    sig("lsdo_trackFrameOnPermaref", C.c_int, C.c_int, C.c_int, fp, fp, C.c_int, vp, dp, C.POINTER(TrackResult))
    sig("lsdo_ref_checkPermaRefOverlap", C.c_float, vp, dp)
    sig("lsdo_ref_trackFrameOnPermaref", C.c_int, vp, vp, dp, C.POINTER(TrackResult))
    sig("lsdo_depthmap_create", vp, C.c_int, C.c_int, fp)
    sig("lsdo_depthmap_destroy", None, vp)
    sig("lsdo_depthmap_reset", None, vp)
    sig("lsdo_depthmap_initializeFromGTDepth", None, vp, vp)
    sig("lsdo_depthmap_initializeRandomly", None, vp, vp)
    sig("lsdo_depthmap_setFromExistingKF", None, vp, vp, fp, fp, u8p)
    sig("lsdo_depthmap_updateKeyframe", None, vp, C.POINTER(vp), C.c_int)
    sig("lsdo_depthmap_createKeyFrame", None, vp, vp)
    sig("lsdo_depthmap_finalizeKeyFrame", None, vp)
    sig("lsdo_depthmap_current", C.POINTER(Hyp), vp)
    sig("lsdo_depthmap_set_current", None, vp, C.POINTER(Hyp))
    sig("lsdo_depthmap_integral", ip, vp)
    sig("lsdo_depthmap_observeDepth", None, vp, C.POINTER(vp), C.c_int)
    sig("lsdo_depthmap_regularizeFillHoles", None, vp)
    sig("lsdo_depthmap_regularize", None, vp, C.c_int, C.c_int)
    sig("lsdo_depthmap_propagateDepth", None, vp, vp)
    sig("lsdo_depthmap_last_timings", None, vp, fp)
    sig("lsdo_ref_prepareForStereoWith", None, vp, vp, dp, fp, fp)
    if not isinstance(fast, str):            # diagnostic counters of the C restatement only
        sig("lsdo_depth_branch_counts", None, C.POINTER(C.c_int64))
        sig("lsdo_depth_branch_counts_reset", None)
        sig("lsdo_sim3_branch_counts", None, C.POINTER(C.c_int64))
        sig("lsdo_sim3_branch_counts_reset", None)
    _libs[name] = L
    return L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def default_track_settings(fast=False, main_tracker: bool = True) -> TrackSettings:
    s = TrackSettings()
    lib(fast).lsdo_default_track_settings(C.byref(s))
    if main_tracker:                       # SlamSystem.cpp:80-81
        for lvl in range(4, LEVELS):
            s.maxItsPerLvl[lvl] = 0
    return s


# the diagnostic branch counters of the C restatement's depth map, in the order of lsd_oracle.h's LSDO_BR_* enum
BRANCHES = ("depth_x", "depth_y", "firstx_gate", "rescale_gate", "near_clamp", "epl_crop",
            "clip_left", "clip_right", "clip_top", "clip_bottom", "subpixel_pre", "subpixel_post", "subpixel_none",
            "prop_skip", "prop_invalidate", "prop_merge", "prop_merge_cap",
            "stereo_err_search", "stereo_err_interp", "stereo_unclear", "stereo_negative",
            "update_fail_invalidate", "update_inconsistent", "create_blacklist", "prop_mask", "prop_color",
            "reg_occlusion", "reg_validity", "fill_create", "epl_reject_grad", "epl_reject_angle")


def branch_counts(fast=False) -> dict:
    """how often each branch of doLineStereo, observeDepth and propagateDepth ran since the last reset, over every depth map of
    the process"""
    out = np.zeros(len(BRANCHES), np.int64)
    lib(fast).lsdo_depth_branch_counts(out.ctypes.data_as(C.POINTER(C.c_int64)))
    return dict(zip(BRANCHES, out.tolist()))


def branch_counts_reset(fast=False) -> None:
    lib(fast).lsdo_depth_branch_counts_reset()


# the same for the Sim3 tracker, the 7x7 solve and the permaRef overlap, in the order of lsd_oracle.h's LSDO_S3_* enum
SIM3_BRANCHES = ("sim3_outside", "sim3_no_depth", "sim3_usage_clamp", "sim3_affine_clamp", "sim3_huber", "ldlt7_solve",
                 "ldlt7_pivot", "perma_outside", "perma_usage_clamp")


def sim3_branch_counts(fast=False) -> dict:
    """how often each counted branch of the Sim3 tracker's scalar path and of checkPermaRefOverlap ran since the last reset"""
    out = np.zeros(len(SIM3_BRANCHES), np.int64)
    lib(fast).lsdo_sim3_branch_counts(out.ctypes.data_as(C.POINTER(C.c_int64)))
    return dict(zip(SIM3_BRANCHES, out.tolist()))


def sim3_branch_counts_reset(fast=False) -> None:
    lib(fast).lsdo_sim3_branch_counts_reset()


def set_globals(fast=False, **kw) -> Globals:
    g = Globals()
    lib(fast).lsdo_default_globals(C.byref(g))
    for k, v in kw.items():
        setattr(g, k, v)
    lib(fast).lsdo_set_globals(C.byref(g))
    return g


class Frame:
    """Mirror of lsd_slam::Frame for the oracle (DataStructures/Frame.h)."""

    def __init__(self, fid: int, image_u8: np.ndarray, K: np.ndarray, fast=False):
        self.L = lib(fast)
        self.h, self.w = image_u8.shape
        img = np.ascontiguousarray(image_u8, np.uint8)
        Kf = np.ascontiguousarray(K, np.float32).reshape(9)
        self.ptr = self.L.lsdo_frame_create_u8(fid, self.w, self.h, _fp(Kf), img.ctypes.data_as(C.POINTER(C.c_uint8)))
        self.id = fid
        self.fl = fast

    def __del__(self):
        if getattr(self, "ptr", None):
            self.L.lsdo_frame_destroy(self.ptr)
            self.ptr = None

    def size(self, level):
        return self.w >> level, self.h >> level

    def _arr(self, name, level, ch=1):
        w, h = self.size(level)
        p = getattr(self.L, f"lsdo_frame_{name}")(self.ptr, level)
        if not p:
            return None
        shape = (h, w, ch) if ch > 1 else (h, w)
        return np.ctypeslib.as_array(p, shape=shape)

    def image(self, level=0):
        return self._arr("image", level)

    def gradients(self, level=0):
        return self._arr("gradients", level, 4)

    def maxGradients(self, level=0):
        return self._arr("maxGradients", level)

    def idepth(self, level=0):
        return self._arr("idepth", level)

    def idepthVar(self, level=0):
        return self._arr("idepthVar", level)

    def reactivation_data(self):
        """copies of (idepth_reAct, idepthVar_reAct, validity_reAct) (Frame.cpp:107-145) or None before the first take"""
        p = self.L.lsdo_frame_idepthVar_reAct(self.ptr)
        if not p:
            return None
        sh = (self.h, self.w)
        return (np.ctypeslib.as_array(self.L.lsdo_frame_idepth_reAct(self.ptr), shape=sh).copy(),
                np.ctypeslib.as_array(p, shape=sh).copy(),
                np.ctypeslib.as_array(self.L.lsdo_frame_validity_reAct(self.ptr), shape=sh).copy())

    def pack_pointcloud(self, level=0) -> np.ndarray:
        """keyframeMsg.pointcloud as InputPointDense records (ROSOutput3DWrapper.cpp:91-110)"""
        w, h = self.size(level)
        out = np.zeros(w * h, POINT_DENSE)
        self.L.lsdo_pack_pointcloud(self.ptr, level, out.ctypes.data_as(C.c_void_p))
        return out

    def K(self, level=0):
        K = np.zeros(9, np.float32)
        Ki = np.zeros(9, np.float32)
        self.L.lsdo_frame_K(self.ptr, level, _fp(K), _fp(Ki))
        return K.reshape(3, 3), Ki.reshape(3, 3)

    def refPixelWasGood(self, create=True):
        p = (self.L.lsdo_frame_refPixelWasGood if create else self.L.lsdo_frame_refPixelWasGoodNoCreate)(self.ptr)
        if not p:
            return None
        w, h = self.size(1)
        return np.ctypeslib.as_array(p, shape=(h, w))

    def setDepthFromGroundTruth(self, depth: np.ndarray, cov_scale: float = 1.0):
        d = np.ascontiguousarray(depth, np.float32)
        self.L.lsdo_frame_setDepthFromGroundTruth(self.ptr, _fp(d), cov_scale)

    def thisToParent(self):
        o = np.zeros(8, np.float64)
        self.L.lsdo_frame_get_thisToParent(self.ptr, _dp(o))
        return o

    def set_thisToParent(self, qts, parent: "Frame"):
        o = np.ascontiguousarray(qts, np.float64)
        self.L.lsdo_frame_set_thisToParent(self.ptr, _dp(o), parent.ptr)

    def point_cloud(self, level):
        w, h = self.size(level)
        n = w * h
        pos = np.zeros((n, 3), np.float32)
        grad = np.zeros((n, 2), np.float32)
        cv = np.zeros((n, 2), np.float32)
        idx = np.zeros(n, np.int32)
        m = self.L.lsdo_make_point_cloud(self.ptr, level, _fp(pos), _fp(grad), _fp(cv), idx.ctypes.data_as(C.POINTER(C.c_int)))
        return pos[:m], grad[:m], cv[:m], idx[:m]


class PermaRef:
    """Frame::setPermaRef snapshot of a keyframe's level-4 point cloud (Frame.cpp:149-174).  The C restatement takes the
    snapshot's arrays; the reference-compiled library reads them from the keyframe, which this object therefore keeps."""

    def __init__(self, kf: Frame):
        w, h = kf.size(4)
        self.w0, self.h0 = kf.w, kf.h
        self.pos = np.zeros((w * h, 3), np.float32)
        self.colvar = np.zeros((w * h, 2), np.float32)
        self.n = kf.L.lsdo_frame_setPermaRef(kf.ptr, _fp(self.pos), _fp(self.colvar))
        self.K4 = kf.K(4)[0].copy()
        self.L = kf.L
        self.kf = kf
        self.ref = isinstance(kf.fl, str)

    def overlap(self, refToFrame_qt) -> float:
        q = np.ascontiguousarray(refToFrame_qt, np.float64)
        if self.ref:
            return float(self.L.lsdo_ref_checkPermaRefOverlap(self.kf.ptr, _dp(q)))
        K4 = np.ascontiguousarray(self.K4, np.float32).reshape(9)
        return float(self.L.lsdo_checkPermaRefOverlap(self.w0, self.h0, _fp(K4), _fp(self.pos), self.n, _dp(q)))

    def track(self, frame: Frame, refToFrame_qt) -> TrackResult:
        q = np.ascontiguousarray(refToFrame_qt, np.float64)
        r = TrackResult()
        if self.ref:
            self.L.lsdo_ref_trackFrameOnPermaref(self.kf.ptr, frame.ptr, _dp(q), C.byref(r))
        else:
            self.L.lsdo_trackFrameOnPermaref(self.w0, self.h0, _fp(self.pos), _fp(self.colvar), self.n, frame.ptr, _dp(q), C.byref(r))
        return r


class UndistorterPTAM:
    """util/Undistorter.cpp:91-411 with the calibration file's four lines already parsed.  out_calib: "crop", "full" or
    (fx, fy, cx, cy, 0) relative to the output size.  Under a reference flavour ("ref", "ref_legacy_math", ...) the reference's
    own class computes the tables from the same lines (oracle/ref_driver.cpp)."""

    def __init__(self, in_calib, in_size, out_calib, out_size, fast: bool = False):
        self.L = lib(fast)
        self.in_w, self.in_h = in_size
        self.out_w, self.out_h = out_size
        ic = np.ascontiguousarray(in_calib, np.float32)
        oc = np.zeros(5, np.float32)
        if isinstance(out_calib, str):
            oc[0] = {"crop": -1, "full": -2}[out_calib]
        else:
            oc[:] = out_calib
        self.remapX = np.zeros((self.out_h, self.out_w), np.float32)
        self.remapY = np.zeros((self.out_h, self.out_w), np.float32)
        self.K = np.zeros(9, np.float32)
        self.status = self.L.lsdo_undistorter_ptam_prepare(_fp(ic), self.in_w, self.in_h, _fp(oc), self.out_w, self.out_h,
                                                           _fp(self.remapX), _fp(self.remapY), _fp(self.K))
        self.K = self.K.reshape(3, 3)

    def undistort(self, image_u8: np.ndarray) -> np.ndarray:
        img = np.ascontiguousarray(image_u8, np.uint8)
        assert img.shape == (self.in_h, self.in_w)
        if self.status == 1:
            return img.copy()
        out = np.zeros((self.out_h, self.out_w), np.uint8)
        u8p = C.POINTER(C.c_uint8)
        self.L.lsdo_undistort(_fp(self.remapX), _fp(self.remapY), self.in_w, self.out_w, self.out_h, img.ctypes.data_as(u8p), out.ctypes.data_as(u8p))
        return out


class RefUndistorterFile:
    """lsd_slam::UndistorterPTAM(configFileName) of the reference itself (util/Undistorter.cpp:91-345), constructed from a
    calibration file in zero-filled storage by oracle/_ref (flavour "ref", "ref_legacy_math" or "ref_sse").  valid, the sizes,
    K as main_on_images.cpp:164-167 reads getK(), the tables (None when the reference built none) and undistort()."""

    def __init__(self, path: str, flavour: str = "ref"):
        self.L = lib(flavour)
        self.ptr = self.L.lsdo_ref_undistorter_open(os.fsencode(path))
        info = np.zeros(5, np.int32)
        K = np.zeros(9, np.float32)
        self.L.lsdo_ref_undistorter_info(self.ptr, info.ctypes.data_as(C.POINTER(C.c_int)), _fp(K))
        self.valid = bool(info[0])
        self.in_w, self.in_h, self.out_w, self.out_h = (int(v) for v in info[1:])
        self.K = K.reshape(3, 3)
        self.remapX = np.zeros((max(self.out_h, 0), max(self.out_w, 0)), np.float32)
        self.remapY = np.zeros_like(self.remapX)
        if not self.L.lsdo_ref_undistorter_tables(self.ptr, _fp(self.remapX), _fp(self.remapY)):
            self.remapX = self.remapY = None

    def undistort(self, image_u8: np.ndarray) -> np.ndarray:
        img = np.ascontiguousarray(image_u8, np.uint8)
        cap = max(img.size, self.out_w * self.out_h)
        out = np.zeros(cap, np.uint8)
        u8p = C.POINTER(C.c_uint8)
        shape = self.L.lsdo_ref_undistorter_undistort(self.ptr, img.ctypes.data_as(u8p), img.shape[1], img.shape[0],
                                                      out.ctypes.data_as(u8p), cap)
        assert shape >= 0
        return out[:(shape >> 16) * (shape & 0xFFFF)].reshape(shape >> 16, shape & 0xFFFF)

    def close(self):
        if self.ptr:
            self.L.lsdo_ref_undistorter_close(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ref_undistorter_for_file(path: str, flavour: str = "ref") -> int:
    """Undistorter::getUndistorterForFile (util/Undistorter.cpp:38-88) of the reference: 0 for its null result, 1 for an
    UndistorterPTAM.  Never pass a file with 8 numbers on its first line: that constructs UndistorterOpenCV, which oracle/_ref
    cannot run."""
    return int(lib(flavour).lsdo_ref_undistorter_for_file(os.fsencode(path)))


def se3_track(kf: Frame, frame: Frame, init_frameToRef_qt, settings: TrackSettings | None = None) -> TrackResult:
    s = settings or default_track_settings()
    r = TrackResult()
    q = np.ascontiguousarray(init_frameToRef_qt, np.float64)
    kf.L.lsdo_se3_track(kf.ptr, frame.ptr, _dp(q), C.byref(s), C.byref(r))
    return r


def sim3_track(ref_kf: Frame, frame: Frame, init_frameToRef_qts, start_level=4, final_level=1,
               settings: TrackSettings | None = None) -> Sim3Result:
    """Sim3Tracker::trackFrameSim3 (Sim3Tracker.cpp:149-382); `frame` must carry depth."""
    s = settings or default_track_settings(main_tracker=False)      # constraintTracker keeps the class defaults
    r = Sim3Result()
    q = np.ascontiguousarray(init_frameToRef_qts, np.float64)
    ref_kf.L.lsdo_sim3_track(ref_kf.ptr, frame.ptr, _dp(q), start_level, final_level, C.byref(s), C.byref(r))
    return r


def sim3_eval(ref_kf: Frame, frame: Frame, level: int, refToFrame_qts, a=1.0, b=0.0, settings=None) -> Sim3EvalResult:
    s = settings or default_track_settings(main_tracker=False)
    r = Sim3EvalResult()
    q = np.ascontiguousarray(refToFrame_qts, np.float64)
    ref_kf.L.lsdo_sim3_eval(ref_kf.ptr, frame.ptr, level, _dp(q), a, b, C.byref(s), C.byref(r))
    return r


def se3_eval(kf: Frame, frame: Frame, level: int, refToFrame_qt, a=1.0, b=0.0, settings=None, write_mask=False) -> EvalResult:
    s = settings or default_track_settings()
    r = EvalResult()
    q = np.ascontiguousarray(refToFrame_qt, np.float32)
    kf.L.lsdo_se3_eval(kf.ptr, frame.ptr, level, _fp(q), a, b, C.byref(s), int(write_mask), C.byref(r))
    return r


class DepthMap:
    """Mirror of lsd_slam::DepthMap for the oracle (DepthEstimation/DepthMap.h)."""

    def __init__(self, w, h, K, fast=False):
        self.L = lib(fast)
        self.w, self.h = w, h
        Kf = np.ascontiguousarray(K, np.float32).reshape(9)
        self.ptr = self.L.lsdo_depthmap_create(w, h, _fp(Kf))
        self._keep = []

    def __del__(self):
        if getattr(self, "ptr", None):
            self.L.lsdo_depthmap_destroy(self.ptr)
            self.ptr = None

    def initializeFromGTDepth(self, f: Frame):
        self._keep.append(f)
        self.L.lsdo_depthmap_initializeFromGTDepth(self.ptr, f.ptr)

    def initializeRandomly(self, f: Frame):
        self._keep.append(f)
        self.L.lsdo_depthmap_initializeRandomly(self.ptr, f.ptr)

    def setFromExistingKF(self, kf: Frame, idepth=None, idepthVar=None, validity=None):
        self._keep.append(kf)
        if idepth is None:                # the keyframe's own reactivation data, as DepthMap.cpp:926-928 reads them
            self.L.lsdo_depthmap_setFromExistingKF(self.ptr, kf.ptr, None, None, None)
            return
        a, b = np.ascontiguousarray(idepth, np.float32), np.ascontiguousarray(idepthVar, np.float32)
        c = np.ascontiguousarray(validity, np.uint8)
        self.L.lsdo_depthmap_setFromExistingKF(self.ptr, kf.ptr, _fp(a), _fp(b), c.ctypes.data_as(C.POINTER(C.c_uint8)))

    def _refs(self, refs):
        arr = (C.c_void_p * len(refs))(*[r.ptr for r in refs])
        return arr

    def updateKeyframe(self, refs):
        self.L.lsdo_depthmap_updateKeyframe(self.ptr, self._refs(refs), len(refs))

    def observeDepth(self, refs):
        self.L.lsdo_depthmap_observeDepth(self.ptr, self._refs(refs), len(refs))

    def regularizeFillHoles(self):
        self.L.lsdo_depthmap_regularizeFillHoles(self.ptr)

    def regularize(self, removeOcclusions, validityTH=24):
        self.L.lsdo_depthmap_regularize(self.ptr, int(removeOcclusions), validityTH)

    def propagateDepth(self, new_kf: Frame):
        self._keep.append(new_kf)
        self.L.lsdo_depthmap_propagateDepth(self.ptr, new_kf.ptr)

    def createKeyFrame(self, new_kf: Frame):
        self._keep.append(new_kf)
        self.L.lsdo_depthmap_createKeyFrame(self.ptr, new_kf.ptr)

    def finalizeKeyFrame(self):
        self.L.lsdo_depthmap_finalizeKeyFrame(self.ptr)

    def current(self) -> np.ndarray:
        p = self.L.lsdo_depthmap_current(self.ptr)
        buf = (C.c_uint8 * (32 * self.w * self.h)).from_address(C.addressof(p.contents))
        return np.frombuffer(buf, dtype=HYP_DTYPE).reshape(self.h, self.w)

    def set_current(self, hyp: np.ndarray):
        a = np.ascontiguousarray(hyp)
        self.L.lsdo_depthmap_set_current(self.ptr, a.ctypes.data_as(C.POINTER(Hyp)))

    def integral(self) -> np.ndarray:
        return np.ctypeslib.as_array(self.L.lsdo_depthmap_integral(self.ptr), shape=(self.h, self.w))

    def timings(self):
        o = np.zeros(8, np.float32)
        self.L.lsdo_depthmap_last_timings(self.ptr, _fp(o))
        return dict(zip(["update", "create", "finalize", "observe", "regularize", "propagate", "fillHoles", "setDepth"], o.tolist()))
