"""ctypes binding of the C ABI (include/lsdgpu.h -> liblsdgpu.so) plus thin Python mirrors of the reference's
public interface for the hot path (``SE3Tracker.trackFrame``, ``DepthMap.updateKeyframe`` /
``createKeyFrame`` -- Tracking/SE3Tracker.h:65-68, DepthEstimation/DepthMap.h:58,63).

This is the product path: it loads the CUDA library and nothing else.  There is NO CPU fallback -- a missing
or unloadable ``liblsdgpu.so`` raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import NamedTuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblsdgpu.so")
LEVELS = 5

EVAL_NSUMS = 40
ALLREDUCE_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_float), C.c_int)

BUF_IMAGE, BUF_GRADIENTS, BUF_MAXGRAD, BUF_IDEPTH, BUF_IDEPTH_VAR, BUF_GOODMASK = range(6)


class Hyp(C.Structure):
    _fields_ = [("isValid", C.c_uint8), ("_pad", C.c_uint8 * 3), ("blacklisted", C.c_int32),
                ("nextStereoFrameMinID", C.c_float), ("validity_counter", C.c_int32),
                ("idepth", C.c_float), ("idepth_var", C.c_float),
                ("idepth_smoothed", C.c_float), ("idepth_var_smoothed", C.c_float)]


HYP_DTYPE = np.dtype([("isValid", np.uint8), ("_pad", np.uint8, 3), ("blacklisted", np.int32),
                      ("nextStereoFrameMinID", np.float32), ("validity_counter", np.int32),
                      ("idepth", np.float32), ("idepth_var", np.float32),
                      ("idepth_smoothed", np.float32), ("idepth_var_smoothed", np.float32)])


POINT_DENSE = np.dtype([("idepth", np.float32), ("idepth_var", np.float32), ("color", np.uint8, (4,))])     # InputPointDense


class RefDesc(C.Structure):
    """lsdgpu_ref_desc (include/lsdgpu.h)"""
    _fields_ = [("frame_id", C.c_int32), ("tracked_on_kf", C.c_int32), ("refToKf_qts", C.c_double * 8)]


class Globals(C.Structure):
    _fields_ = [("minUseGrad", C.c_float), ("cameraPixelNoise2", C.c_float), ("depthSmoothingFactor", C.c_float),
                ("allowNegativeIdepths", C.c_int), ("useSubpixelStereo", C.c_int),
                ("useAffineLightningEstimation", C.c_int)]


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


class GroupStep(C.Structure):
    """lsdgpu_group_step (include/lsdgpu.h): one stream's frame in lsdgpu_track_and_map_group"""
    _fields_ = [("ctx", C.c_void_p), ("kf_id", C.c_int), ("frame_id", C.c_int), ("gray", C.POINTER(C.c_uint8)),
                ("stage_index", C.c_int), ("frameToRef_init_qt", C.c_double * 7), ("settings", C.POINTER(TrackSettings)),
                ("keyframe_change", C.c_int)]


GROUP_MAX_STEPS = 8


class MemoryUsage(NamedTuple):
    """Context.memory_usage: minimized frames whose record is in device memory, offloaded ones, and the records' layout bytes in
    each tier (an offloaded frame's device residue counts under device_bytes)"""
    n_device: int
    device_bytes: int
    n_host: int
    host_bytes: int


class RandState(C.Structure):
    """lsdgpu_rand_state (include/lsdgpu.h): glibc's random() state -- random_r's table and its rear index, in any of the five
    state types (0: the LCG; 1..4: tables of 7, 15, 31, 63 words; rand() after srand() uses type 3).  The stream
    ``DepthMap.initializeRandomly`` draws from (DepthMap.cpp:898)."""
    _fields_ = [("type", C.c_int32), ("rear", C.c_int32), ("r", C.c_uint32 * 63)]

    @classmethod
    def from_seed(cls, seed: int, type: int = 3) -> "RandState":
        """srandom_r(seed) for a buffer of the given type (srand(seed) for type 3)"""
        st = cls()
        if load().lsdgpu_rand_state_seed(int(type), C.c_uint(seed & 0xffffffff), C.byref(st)) != 0:
            raise ValueError(f"bad random state type {type}")
        return st

    def copy(self) -> "RandState":
        st = RandState()
        C.memmove(C.byref(st), C.byref(self), C.sizeof(RandState))
        return st

    def advance(self, n: int, values: bool = True):
        """n calls of random(): returns them (int32) when ``values``, otherwise jumps ahead; the state moves on in place"""
        out = np.zeros(n, np.int32) if values else None
        p = out.ctypes.data_as(C.POINTER(C.c_int32)) if values else None
        if load().lsdgpu_rand_state_advance(C.byref(self), C.c_int64(n), p) != 0:
            raise ValueError("bad random state or count")
        return out

    def __eq__(self, other) -> bool:
        return isinstance(other, RandState) and bytes(self) == bytes(other)


# every symbol include/lsdgpu.h declares: (name, restype, argtypes)
_vp, _fp, _dp, _ip, _u8p = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint8)
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


class CloudFilter(C.Structure):
    """lsdgpu_cloud_filter: the viewer's filter settings, lsd_slam_viewer/src/settings.cpp:36-40"""
    _fields_ = [("scaledDepthVarTH", C.c_float), ("absDepthVarTH", C.c_float), ("minNearSupport", C.c_int), ("sparsifyFactor", C.c_int)]


CLOUD_PLY, CLOUD_VERTEX = 0, 1
CLOUD_ERR_CAPACITY = -4
# LSDGPU_CLOUD_PLY: flushPC's record (KeyFrameDisplay.cpp:328-333); LSDGPU_CLOUD_VERTEX: MyVertex (KeyFrameDisplay.h:33-37)
CLOUD_PLY_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4")])
CLOUD_VERTEX_DTYPE = np.dtype([("point", "<f4", (3,)), ("color", "u1", (4,))])


def default_cloud_filter(**kw) -> CloudFilter:
    f = CloudFilter()
    load().lsdgpu_default_cloud_filter(C.byref(f))
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def write_ply(path, points: np.ndarray) -> None:
    """Writes points (CLOUD_PLY_DTYPE, e.g. from Context.export_pointcloud) as the viewer's pc.ply: the header of
    KeyFrameGraphDisplay.cpp:74-82, then the 16-byte records.  The viewer's copy loop `while(!f3.eof()) f2.put(f3.get())`
    (:84-85) appends one stray 0xFF byte after the last record; this writer does not, so its file is the viewer's minus that byte."""
    pts = np.ascontiguousarray(points, CLOUD_PLY_DTYPE)
    with open(path, "wb") as f:
        f.write(b"ply\nformat binary_little_endian 1.0\n")
        f.write(b"element vertex %d\n" % len(pts))
        f.write(b"property float x\nproperty float y\nproperty float z\nproperty float intensity\nend_header\n")
        f.write(pts.tobytes())


SYMBOLS = [
    ("lsdgpu_create", C.c_int, [C.c_int, C.c_int, C.c_int, _fp, C.c_int, C.POINTER(_vp)]),
    ("lsdgpu_destroy", None, [_vp]),
    ("lsdgpu_last_error", C.c_char_p, [_vp]),
    ("lsdgpu_abi_version", C.c_int, []),
    ("lsdgpu_set_globals", C.c_int, [_vp, C.POINTER(Globals)]),
    ("lsdgpu_get_globals", C.c_int, [_vp, C.POINTER(Globals)]),
    ("lsdgpu_default_globals", None, [C.POINTER(Globals)]),
    ("lsdgpu_default_track_settings", None, [C.POINTER(TrackSettings)]),
    ("lsdgpu_synchronize", C.c_int, [_vp]),
    ("lsdgpu_launch_count", C.c_longlong, [_vp]),
    ("lsdgpu_timer_begin", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_timer_end", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_timer_elapsed_ms", C.c_int, [_vp, C.c_int, _fp]),
    ("lsdgpu_track_kernel_stats", C.c_int, [_vp, C.c_int, _dp, C.POINTER(C.c_longlong), _dp]),
    ("lsdgpu_frame_upload_u8", C.c_int, [_vp, C.c_int, _u8p]),
    ("lsdgpu_frame_release", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_stage_reserve", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_stage_put", C.c_int, [_vp, C.c_int, _u8p]),
    ("lsdgpu_frame_from_stage", C.c_int, [_vp, C.c_int, C.c_int]),
    ("lsdgpu_frame_download", C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp]),
    ("lsdgpu_frame_set_depth_gt", C.c_int, [_vp, C.c_int, _fp, C.c_float]),
    ("lsdgpu_frame_set_idepth", C.c_int, [_vp, C.c_int, _fp, _fp]),
    ("lsdgpu_frame_set_pose", C.c_int, [_vp, C.c_int, _dp, C.c_int, C.c_float]),
    ("lsdgpu_frame_get_pose", C.c_int, [_vp, C.c_int, _dp, _ip, _fp]),
    ("lsdgpu_frame_get_counters", C.c_int, [_vp, C.c_int, _ip, _ip]),
    ("lsdgpu_frame_set_counters", C.c_int, [_vp, C.c_int, C.c_int, C.c_int]),
    ("lsdgpu_frame_get_depth_stats", C.c_int, [_vp, C.c_int, _fp, _ip, _ip]),
    ("lsdgpu_frame_clear_good_mask", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_frame_minimize", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_frame_activate", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_frame_offload", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_frame_memory_usage", C.c_int, [_vp, _ip, C.POINTER(C.c_size_t), _ip, C.POINTER(C.c_size_t)]),
    ("lsdgpu_ref_import", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_se3_eval", C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _fp, C.c_float, C.c_float, C.POINTER(TrackSettings), C.c_int, C.POINTER(EvalResult)]),
    ("lsdgpu_se3_track", C.c_int, [_vp, C.c_int, C.c_int, _dp, C.POINTER(TrackSettings), C.c_int, C.POINTER(TrackResult)]),
    ("lsdgpu_track_and_map", C.c_int, [_vp, C.c_int, C.c_int, _u8p, C.c_int, _dp, C.POINTER(TrackSettings), C.c_int, C.c_int, C.POINTER(TrackResult), _dp]),
    ("lsdgpu_track_and_map_group", C.c_int, [C.c_int, C.POINTER(GroupStep), C.POINTER(TrackResult), _dp]),
    ("lsdgpu_undistorter_ptam_prepare", C.c_int, [_fp, C.c_int, C.c_int, _fp, C.c_int, C.c_int, _fp, _fp, _fp]),
    ("lsdgpu_undistorter_validate_tables", C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _fp, _fp]),
    ("lsdgpu_set_undistorter", C.c_int, [_vp, C.c_int, C.c_int, _fp, _fp]),
    ("lsdgpu_undistorter_opencv_prepare", C.c_int, [_fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int16),
                                                    C.POINTER(C.c_uint16), _dp, _fp]),
    ("lsdgpu_set_undistorter_opencv", C.c_int, [_vp, C.c_int, C.c_int, C.POINTER(C.c_int16), C.POINTER(C.c_uint16)]),
    ("lsdgpu_undistort_u8", C.c_int, [_vp, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8)]),
    ("lsdgpu_frame_upload_distorted_u8", C.c_int, [_vp, C.c_int, C.POINTER(C.c_uint8)]),
    ("lsdgpu_keyframe_pack_pointcloud", C.c_int, [_vp, C.c_int, C.c_int, _vp]),
    ("lsdgpu_default_cloud_filter", None, [C.c_void_p]),
    ("lsdgpu_cloud_reserve", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_map_export_pointcloud", C.c_int, [_vp, C.c_int, _ip, _fp, C.c_int, C.c_void_p, C.c_int, _vp, C.c_int64,
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    ("lsdgpu_cloud_last_kernel_ms", C.c_int, [_vp, _fp]),
    ("lsdgpu_frame_upload_device_u8", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_frame_upload_distorted_device_u8", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_stage_put_device", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_set_input_format", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_stage_put_raw", C.c_int, [_vp, C.c_int, C.POINTER(C.c_uint8)]),
    ("lsdgpu_stage_put_raw_device", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_frame_download_device", C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_map_export_pointcloud_device", C.c_int, [_vp, C.c_int, _ip, _fp, C.c_int, C.c_void_p, C.c_int, _vp, C.c_int64,
                                                      C.POINTER(C.c_int64), C.POINTER(C.c_int32), _vp]),
    ("lsdgpu_frame_set_depth_gt_device", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, C.c_float, _vp]),
    ("lsdgpu_frame_set_idepth_device", C.c_int, [_vp, C.c_int, _vp, _vp, C.c_size_t, _vp]),
    ("lsdgpu_depth_set_hypotheses_device", C.c_int, [_vp, C.c_int, _vp, C.c_int, C.c_int, _vp]),
    ("lsdgpu_depth_download_device", C.c_int, [_vp, _vp, C.c_size_t, _vp]),
    ("lsdgpu_keyframe_pack_pointcloud_device", C.c_int, [_vp, C.c_int, C.c_int, _vp, C.c_size_t, _vp]),
    ("lsdgpu_frame_take_reactivation_data", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_frame_download_reactivation_data", C.c_int, [_vp, C.c_int, _fp, _fp, C.POINTER(C.c_uint8)]),
    ("lsdgpu_depth_set_from_existing_kf", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_sim3_eval", C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _dp, C.c_float, C.c_float, C.POINTER(TrackSettings), C.POINTER(Sim3EvalResult)]),
    ("lsdgpu_sim3_track", C.c_int, [_vp, C.c_int, C.c_int, _dp, C.c_int, C.c_int, C.POINTER(TrackSettings), C.POINTER(Sim3Result)]),
    ("lsdgpu_sim3_track_batch", C.c_int, [_vp, C.c_int, _ip, _ip, _dp, C.c_int, C.c_int, C.POINTER(TrackSettings), C.POINTER(Sim3Result)]),
    ("lsdgpu_frame_set_perma_ref", C.c_int, [_vp, C.c_int, _ip]),
    ("lsdgpu_perma_overlap_batch", C.c_int, [_vp, C.c_int, _ip, _dp, _fp]),
    ("lsdgpu_perma_track_batch", C.c_int, [_vp, C.c_int, _ip, C.c_int, _dp, C.POINTER(TrackResult)]),
    ("lsdgpu_se3_track_sharded", C.c_int, [_vp, C.c_int, C.c_int, _dp, C.POINTER(TrackSettings), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(TrackResult)]),
    ("lsdgpu_depth_reset", C.c_int, [_vp]),
    ("lsdgpu_depth_is_valid", C.c_int, [_vp]),
    ("lsdgpu_depth_invalidate", C.c_int, [_vp]),
    ("lsdgpu_depth_init_from_gt", C.c_int, [_vp, C.c_int]),
    ("lsdgpu_depth_set_hypotheses", C.c_int, [_vp, C.c_int, C.POINTER(Hyp), C.c_int, C.c_int]),
    ("lsdgpu_rand_state_seed", C.c_int, [C.c_int, C.c_uint, C.POINTER(RandState)]),
    ("lsdgpu_rand_state_advance", C.c_int, [C.POINTER(RandState), C.c_int64, C.POINTER(C.c_int32)]),
    ("lsdgpu_depth_init_random", C.c_int, [_vp, C.c_int, C.POINTER(RandState), C.POINTER(C.c_int64)]),
    ("lsdgpu_depth_update_keyframe", C.c_int, [_vp, _ip, C.c_int]),
    ("lsdgpu_depth_update_keyframe_refs", C.c_int, [_vp, C.c_void_p, C.c_int]),
    ("lsdgpu_peer_export", C.c_int, [_vp, C.c_void_p]),
    ("lsdgpu_peer_attach", C.c_int, [_vp, C.c_int, C.c_int, C.c_void_p]),
    ("lsdgpu_peer_detach", C.c_int, [_vp]),
    ("lsdgpu_depth_create_keyframe", C.c_int, [_vp, C.c_int, _dp]),
    ("lsdgpu_seq_sum_f32", C.c_int, [_vp, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    ("lsdgpu_depth_finalize_keyframe", C.c_int, [_vp]),
    ("lsdgpu_depth_active_keyframe", C.c_int, [_vp]),
    ("lsdgpu_depth_download", C.c_int, [_vp, C.POINTER(Hyp)]),
    ("lsdgpu_depth_download_integral", C.c_int, [_vp, C.POINTER(C.c_int32)]),
    ("lsdgpu_depth_observe", C.c_int, [_vp, _ip, C.c_int]),
    ("lsdgpu_depth_regularize_fill_holes", C.c_int, [_vp]),
    ("lsdgpu_depth_regularize", C.c_int, [_vp, C.c_int, C.c_int]),
    ("lsdgpu_depth_propagate", C.c_int, [_vp, C.c_int]),
]

_lib = None


def load():
    """Load liblsdgpu.so (loudly: raises if the extension is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    global LIB_PATH
    if os.environ.get("LSDGPU_LIB"):                 # A/B runs of two builds of the library (scripts/ab_track.py, profiling)
        LIB_PATH = os.path.abspath(os.environ["LSDGPU_LIB"])
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with `python -m lsd_slam_b200.build` "
                           "(the product path has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args
    _lib = L
    return L


class LsdGpuError(RuntimeError):
    pass


def _is_tensor(x) -> bool:
    """x is a torch.Tensor; decided without importing torch, so that numpy callers never load it"""
    return type(x).__module__.split(".")[0] == "torch"


def _tensor_dtype(t, dtype: str, what: str):
    import torch
    if t.dtype != getattr(torch, dtype):
        raise ValueError(f"{what}: needs torch.{dtype}, not {t.dtype}")


def _cuda_stream(t, device: int, what: str) -> int:
    """checks that t is a CUDA tensor on the context's device -> the handle of that device's current stream (0 = the legacy default
    stream), on which the *_device entry points order their work"""
    import torch
    if not t.is_cuda:
        raise ValueError(f"{what}: needs a CUDA tensor, not one on {t.device}")
    if t.device.index != device:
        raise ValueError(f"{what}: the tensor is on {t.device}, the context on cuda:{device}")
    return torch.cuda.current_stream(t.device).cuda_stream


def _device_image(t, device: int, w: int, h: int, what: str, dtype: str = "uint8"):
    """a 2-D CUDA tensor of h x w (uint8, or `dtype`) whose rows are contiguous -> (pointer, row pitch in bytes, stream)"""
    _tensor_dtype(t, dtype, what)
    if t.dim() != 2 or tuple(t.shape) != (h, w):
        raise ValueError(f"{what}: needs shape ({h}, {w}), not {tuple(t.shape)}")
    if t.stride(1) != 1 or t.stride(0) < w:
        raise ValueError(f"{what}: needs contiguous rows (stride(1) == 1, stride(0) >= {w}), not strides {t.stride()}")
    return t.data_ptr(), t.stride(0) * t.element_size(), _cuda_stream(t, device, what)


def _device_out(t, dtype: str, n: int, device: int, what: str) -> int:
    """a contiguous CUDA tensor of `dtype` with at least n elements -> the stream its device work is ordered on"""
    _tensor_dtype(t, dtype, what)
    if not t.is_contiguous() or t.numel() < n:
        raise ValueError(f"{what}: needs a contiguous tensor of at least {n} elements")
    return _cuda_stream(t, device, what)


HYP_FIELDS = [(name, HYP_DTYPE.fields[name][1], HYP_DTYPE.fields[name][0]) for name in HYP_DTYPE.names if name != "_pad"]


def hyp_fields(t) -> dict:
    """the eight DepthMapPixelHypothesis fields of a (h, w, 32) uint8 tensor of hypotheses (``DepthMap.current(out=...)``, the input
    of ``DepthMap.setHypotheses``) as (h, w) strided views of it, without copies: isValid uint8, blacklisted and validity_counter
    int32, the others float32.  Writes to a view write the hypotheses."""
    import torch
    _tensor_dtype(t, "uint8", "hyp_fields")
    if t.dim() != 3 or t.shape[2] != HYP_DTYPE.itemsize or not t.is_contiguous():
        raise ValueError(f"hyp_fields: needs a contiguous (h, w, {HYP_DTYPE.itemsize}) uint8 tensor, not {tuple(t.shape)}")
    out = {}
    for name, offset, dt in HYP_FIELDS:
        if dt == np.uint8:
            out[name] = t[:, :, offset]
        else:
            words = t.view(torch.int32 if dt == np.int32 else torch.float32)       # (h, w, 8)
            out[name] = words[:, :, offset // 4]
    return out


# the camera's raw pixel formats (LSDGPU_PIX_*), by ROS image encoding: (format, bytes per pixel).  Context.set_input_format selects
# one; the device converts each raw pixel as OpenCV 4.13's cv::cvtColor(.., COLOR_RGB2GRAY / BGR2GRAY / YUV2GRAY_UYVY / _YUY2) does.
INPUT_FORMATS = {"mono8": (0, 1), "rgb8": (1, 3), "bgr8": (2, 3), "rgba8": (3, 4), "bgra8": (4, 4), "yuv422": (5, 2),
                 "yuv422_yuy2": (6, 2)}


class UndistorterPTAM:
    """Mirror of lsd_slam::UndistorterPTAM (util/Undistorter.h:96-160) with the calibration file's lines already parsed.
    out_calib: "crop", "full" or (fx, fy, cx, cy, 0).  Host-only; `install(ctx)` puts the tables on the device."""

    def __init__(self, in_calib, in_size, out_calib, out_size):
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
        K = np.zeros(9, np.float32)
        self.status = load().lsdgpu_undistorter_ptam_prepare(ic.ctypes.data_as(_fp), self.in_w, self.in_h, oc.ctypes.data_as(_fp),
                                                             self.out_w, self.out_h, self.remapX.ctypes.data_as(_fp),
                                                             self.remapY.ctypes.data_as(_fp), K.ctypes.data_as(_fp))
        if self.status < 0:
            raise LsdGpuError("UndistorterPTAM: invalid calibration")
        self.K = K.reshape(3, 3)

    def getK(self) -> np.ndarray:
        return self.K

    def install(self, ctx: "Context"):
        assert (ctx.w, ctx.h) == (self.out_w, self.out_h)
        if self.status == 1:
            ctx._ck(ctx.L.lsdgpu_set_undistorter(ctx.ptr, self.in_w, self.in_h, None, None))
        else:
            ctx._ck(ctx.L.lsdgpu_set_undistorter(ctx.ptr, self.in_w, self.in_h, self.remapX.ctypes.data_as(_fp), self.remapY.ctypes.data_as(_fp)))
        ctx.raw_size = (self.in_w, self.in_h)


class UndistorterOpenCV:
    """Mirror of lsd_slam::UndistorterOpenCV (util/Undistorter.h:164-233) with the calibration file's lines already parsed:
    in_calib = fx fy cx cy k1 k2 p1 p2, out_mode "crop" or "full".  Host-only (lsdgpu_undistorter_opencv_prepare): map1 (h, w, 2)
    int16 and map2 (h, w) uint16 are cv::initUndistortRectifyMap(.., CV_16SC2), K_new (float64) cv::getOptimalNewCameraMatrix,
    K (float32) the matrix getK() hands to SlamSystem.  `status` is 0, or -2 for an invalid calibration (an output mode other
    than crop / full included); install(ctx) then raises."""

    MODES = {"crop": -1, "full": -2}

    def __init__(self, in_calib, in_size, out_mode, out_size):
        self.in_w, self.in_h = in_size
        self.out_w, self.out_h = out_size
        ic = np.ascontiguousarray(in_calib, np.float32)
        assert ic.shape == (8,)
        self.map1 = np.zeros((self.out_h, self.out_w, 2), np.int16)
        self.map2 = np.zeros((self.out_h, self.out_w), np.uint16)
        K_new = np.zeros(9, np.float64)
        K = np.zeros(9, np.float32)
        self.status = load().lsdgpu_undistorter_opencv_prepare(
            ic.ctypes.data_as(_fp), self.in_w, self.in_h, self.MODES.get(out_mode, 0), self.out_w, self.out_h,
            self.map1.ctypes.data_as(C.POINTER(C.c_int16)), self.map2.ctypes.data_as(C.POINTER(C.c_uint16)),
            K_new.ctypes.data_as(_dp), K.ctypes.data_as(_fp))
        self.K_new = K_new.reshape(3, 3)
        self.K = K.reshape(3, 3)

    def getK(self) -> np.ndarray:
        return self.K

    def install(self, ctx: "Context"):
        if self.status != 0:
            raise LsdGpuError("UndistorterOpenCV: invalid calibration")
        assert (ctx.w, ctx.h) == (self.out_w, self.out_h)
        ctx._ck(ctx.L.lsdgpu_set_undistorter_opencv(ctx.ptr, self.in_w, self.in_h, self.map1.ctypes.data_as(C.POINTER(C.c_int16)),
                                                    self.map2.ctypes.data_as(C.POINTER(C.c_uint16))))
        ctx.raw_size = (self.in_w, self.in_h)


def default_track_settings(main_tracker: bool = True) -> TrackSettings:
    s = TrackSettings()
    load().lsdgpu_default_track_settings(C.byref(s))
    if main_tracker:                      # SlamSystem.cpp:80-81
        for lvl in range(4, LEVELS):
            s.maxItsPerLvl[lvl] = 0
    return s


class Context:
    """One device context = the device state of one SlamSystem (frames + one tracker + one depth map)."""

    input_format = "mono8"                    # ROS encoding of the installed undistorter's raw images (set_input_format)

    def __init__(self, w: int, h: int, K: np.ndarray, device: int = 0, max_frames: int = 8, **globals_kw):
        self.L = load()
        self.w, self.h = w, h
        self.device = device
        self.raw_size = None                  # (in_width, in_height) of the installed undistorter
        self.K = np.ascontiguousarray(K, np.float32).reshape(3, 3)
        p = _vp()
        rc = self.L.lsdgpu_create(device, w, h, self.K.ctypes.data_as(_fp), max_frames, C.byref(p))
        self.ptr = p
        if rc != 0:
            msg = self.L.lsdgpu_last_error(p).decode() if p else "lsdgpu_create failed"
            if p:
                self.L.lsdgpu_destroy(p)
            self.ptr = None
            raise LsdGpuError(f"lsdgpu_create({w}x{h}) -> {rc}: {msg}")
        if globals_kw:
            self.set_globals(**globals_kw)

    def close(self):
        if getattr(self, "ptr", None):
            self.L.lsdgpu_destroy(self.ptr)
            self.ptr = None

    def __del__(self):
        self.close()

    def _ck(self, rc):
        if rc != 0:
            raise LsdGpuError(f"rc={rc}: {self.L.lsdgpu_last_error(self.ptr).decode()}")

    def set_globals(self, **kw):
        g = Globals()
        self.L.lsdgpu_default_globals(C.byref(g))
        for k, v in kw.items():
            setattr(g, k, v)
        self._ck(self.L.lsdgpu_set_globals(self.ptr, C.byref(g)))

    def get_globals(self) -> dict:
        """the run-time settings the context's next calls use (lsdgpu_get_globals), by field name"""
        g = Globals()
        self._ck(self.L.lsdgpu_get_globals(self.ptr, C.byref(g)))
        return {name: getattr(g, name) for name, _ in Globals._fields_}

    def synchronize(self):
        self._ck(self.L.lsdgpu_synchronize(self.ptr))

    def launch_count(self) -> int:
        return int(self.L.lsdgpu_launch_count(self.ptr))

    def timer_begin(self, slot=0):
        self._ck(self.L.lsdgpu_timer_begin(self.ptr, slot))

    def timer_end(self, slot=0) -> None:
        self._ck(self.L.lsdgpu_timer_end(self.ptr, slot))

    def timer_ms(self, slot=0) -> float:
        ms = C.c_float()
        self._ck(self.L.lsdgpu_timer_elapsed_ms(self.ptr, slot, C.byref(ms)))
        return ms.value

    def track_kernel_stats(self, reset=0):
        ms, n, b = C.c_double(), C.c_longlong(), C.c_double()
        self._ck(self.L.lsdgpu_track_kernel_stats(self.ptr, reset, C.byref(ms), C.byref(n), C.byref(b)))
        return ms.value, n.value, b.value

    # ---- Frame ----
    def upload(self, fid: int, image_u8):
        """Frame::Frame from a host image (numpy), or from a 2-D uint8 CUDA tensor with contiguous rows (its row stride is the
        pitch), ordered on the tensor's current stream (lsdgpu_frame_upload_device_u8)"""
        if _is_tensor(image_u8):
            ptr, pitch, stream = _device_image(image_u8, self.device, self.w, self.h, "upload")
            self._ck(self.L.lsdgpu_frame_upload_device_u8(self.ptr, fid, ptr, pitch, stream))
            return
        img = np.ascontiguousarray(image_u8, np.uint8)
        assert img.shape == (self.h, self.w)
        self._ck(self.L.lsdgpu_frame_upload_u8(self.ptr, fid, img.ctypes.data_as(_u8p)))

    def stage_reserve(self, n: int):
        self._ck(self.L.lsdgpu_stage_reserve(self.ptr, n))

    def stage_put(self, index: int, image_u8):
        """one frame into prefetch-ring entry `index`: a host image (numpy), or a CUDA tensor as `upload` takes it
        (lsdgpu_stage_put_device, which does not wait for the device)"""
        if _is_tensor(image_u8):
            ptr, pitch, stream = _device_image(image_u8, self.device, self.w, self.h, "stage_put")
            self._ck(self.L.lsdgpu_stage_put_device(self.ptr, index, ptr, pitch, stream))
            return
        img = np.ascontiguousarray(image_u8, np.uint8)
        self._ck(self.L.lsdgpu_stage_put(self.ptr, index, img.ctypes.data_as(_u8p)))

    def frame_from_stage(self, fid: int, index: int):
        self._ck(self.L.lsdgpu_frame_from_stage(self.ptr, fid, index))

    def release(self, fid: int):
        self._ck(self.L.lsdgpu_frame_release(self.ptr, fid))

    def minimize(self, fid: int):
        """Frame::minimizeInMemory (lsdgpu_frame_minimize): the frame gives its slot back and keeps level 0, the reactivation
        data, the permaRef and its metadata in a record; its good mask is cleared"""
        self._ck(self.L.lsdgpu_frame_minimize(self.ptr, fid))

    def activate(self, fid: int):
        """FrameMemory::activateFrame + Frame::require (lsdgpu_frame_activate): a minimized frame takes a free slot again"""
        self._ck(self.L.lsdgpu_frame_activate(self.ptr, fid))

    def offload(self, fid: int):
        """moves a minimized frame's record to host memory, keeping its depth statistics and permaRef on the device
        (lsdgpu_frame_offload); the frame serves the same calls as before, and activate brings it back into a slot"""
        self._ck(self.L.lsdgpu_frame_offload(self.ptr, fid))

    def memory_usage(self) -> "MemoryUsage":
        """the minimized frames in each tier and their records' layout bytes (lsdgpu_frame_memory_usage)"""
        nd, nh, db, hb = C.c_int(), C.c_int(), C.c_size_t(), C.c_size_t()
        self._ck(self.L.lsdgpu_frame_memory_usage(self.ptr, C.byref(nd), C.byref(db), C.byref(nh), C.byref(hb)))
        return MemoryUsage(nd.value, db.value, nh.value, hb.value)

    def download(self, fid: int, what: int, level: int = 0, out=None):
        """one plane of a frame as a numpy array, or -- out = a contiguous CUDA tensor (float32; uint8 for BUF_GOODMASK) of at
        least the plane's size -- copied on the device into out, ordered on its current stream; returns a view of out
        (lsdgpu_frame_download_device)"""
        w, h = self.w >> level, self.h >> level
        if what == BUF_GRADIENTS:
            shape, dtype = (h, w, 4), np.float32
        elif what == BUF_GOODMASK:
            shape, dtype = (self.h >> 1, self.w >> 1), np.uint8
        else:
            shape, dtype = (h, w), np.float32
        if out is not None:
            _tensor_dtype(out, "uint8" if dtype == np.uint8 else "float32", "download(out=)")
            n = int(np.prod(shape))
            if not out.is_contiguous() or out.numel() < n:
                raise ValueError(f"download(out=): needs a contiguous tensor of at least {n} elements")
            stream = _cuda_stream(out, self.device, "download(out=)")
            self._ck(self.L.lsdgpu_frame_download_device(self.ptr, fid, what, level, out.data_ptr(), out.numel() * out.element_size(), stream))
            return out.reshape(-1)[:n].view(shape)
        out = np.empty(shape, dtype)
        self._ck(self.L.lsdgpu_frame_download(self.ptr, fid, what, level, out.ctypes.data_as(_vp)))
        return out

    def set_depth_gt(self, fid: int, depth, cov_scale: float = 1.0):
        """Frame::setDepthFromGroundTruth from metric depth: a host array (numpy), or a 2-D float32 CUDA tensor of (h, w) with
        contiguous rows, read on the device in order on its current stream (lsdgpu_frame_set_depth_gt_device)"""
        if _is_tensor(depth):
            ptr, pitch, stream = _device_image(depth, self.device, self.w, self.h, "set_depth_gt", "float32")
            self._ck(self.L.lsdgpu_frame_set_depth_gt_device(self.ptr, fid, ptr, pitch, cov_scale, stream))
            return
        d = np.ascontiguousarray(depth, np.float32)
        self._ck(self.L.lsdgpu_frame_set_depth_gt(self.ptr, fid, d.ctypes.data_as(_fp), cov_scale))

    def set_idepth(self, fid: int, idepth, var):
        """level-0 idepth and idepthVar of a frame: host arrays, or two float32 CUDA tensors as set_depth_gt takes them, with the
        same row stride (lsdgpu_frame_set_idepth_device)"""
        if _is_tensor(idepth) or _is_tensor(var):
            if not (_is_tensor(idepth) and _is_tensor(var)):
                raise ValueError("set_idepth: idepth and var must both be CUDA tensors or both host arrays")
            pa, pitch, stream = _device_image(idepth, self.device, self.w, self.h, "set_idepth", "float32")
            pb, pitch_b, _ = _device_image(var, self.device, self.w, self.h, "set_idepth", "float32")
            if pitch_b != pitch:
                raise ValueError(f"set_idepth: idepth and var need the same row stride, not {idepth.stride(0)} and {var.stride(0)}")
            self._ck(self.L.lsdgpu_frame_set_idepth_device(self.ptr, fid, pa, pb, pitch, stream))
            return
        a = np.ascontiguousarray(idepth, np.float32)
        b = np.ascontiguousarray(var, np.float32)
        self._ck(self.L.lsdgpu_frame_set_idepth(self.ptr, fid, a.ctypes.data_as(_fp), b.ctypes.data_as(_fp)))

    def set_pose(self, fid: int, qts, parent_id: int, initialTrackedResidual: float = 0.0):
        q = np.ascontiguousarray(qts, np.float64)
        self._ck(self.L.lsdgpu_frame_set_pose(self.ptr, fid, q.ctypes.data_as(_dp), parent_id, initialTrackedResidual))

    def get_pose(self, fid: int):
        q = np.zeros(8, np.float64)
        pid, itr = C.c_int(), C.c_float()
        self._ck(self.L.lsdgpu_frame_get_pose(self.ptr, fid, q.ctypes.data_as(_dp), C.byref(pid), C.byref(itr)))
        return q, pid.value, itr.value

    PEER_HANDLE_BYTES = 64

    def peer_export(self) -> bytes:
        """CUDA IPC handle of this context's arena (lsdgpu_peer_export)"""
        buf = C.create_string_buffer(self.PEER_HANDLE_BYTES)
        self._ck(self.L.lsdgpu_peer_export(self.ptr, buf))
        return buf.raw

    def peer_attach(self, rank: int, handles: list):
        """map the arenas of all ranks (handles in rank order) and shard the device-resident tracker over them"""
        blob = b"".join(handles)
        assert len(blob) == self.PEER_HANDLE_BYTES * len(handles)
        self._ck(self.L.lsdgpu_peer_attach(self.ptr, rank, len(handles), C.c_char_p(blob) if len(handles) > 1 else None))

    def peer_detach(self):
        self._ck(self.L.lsdgpu_peer_detach(self.ptr))

    def seq_sum_f32(self, x, valid=None):
        """the sequential fp32 `sum += x[i]` of DepthMap.cpp:1286-1293 through the kernels createKeyFrame uses"""
        x = np.ascontiguousarray(x, np.float32).ravel()
        v = None if valid is None else np.ascontiguousarray(valid, np.uint8).ravel()
        s, c = C.c_float(), C.c_int()
        self._ck(self.L.lsdgpu_seq_sum_f32(self.ptr, x.ctypes.data, None if v is None else v.ctypes.data, x.size, C.byref(s), C.byref(c)))
        return np.float32(s.value), c.value

    def get_counters(self, fid: int):
        a, b = C.c_int(), C.c_int()
        self._ck(self.L.lsdgpu_frame_get_counters(self.ptr, fid, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_counters(self, fid: int, tracked: int, mapped: int):
        self._ck(self.L.lsdgpu_frame_set_counters(self.ptr, fid, tracked, mapped))

    def depth_stats(self, fid: int):
        m, n, f = C.c_float(), C.c_int(), C.c_int()
        self._ck(self.L.lsdgpu_frame_get_depth_stats(self.ptr, fid, C.byref(m), C.byref(n), C.byref(f)))
        return m.value, n.value, bool(f.value)

    def depth_updated_flag(self, fid: int) -> bool:
        """Frame::depthHasBeenUpdatedFlag only (no device sync, unlike depth_stats)."""
        f = C.c_int()
        self._ck(self.L.lsdgpu_frame_get_depth_stats(self.ptr, fid, None, None, C.byref(f)))
        return bool(f.value)

    def set_input_format(self, encoding: str):
        """the ROS image encoding of the installed undistorter's raw images (lsdgpu_set_input_format): "mono8" (the default),
        "rgb8", "bgr8", "rgba8", "bgra8", "yuv422" (UYVY) or "yuv422_yuy2".  undistort, upload_distorted and stage_put_raw then take
        (h, w, 3 | 4 | 2) images and convert them to gray as cv_bridge / cv::cvtColor does (ROSImageStreamThread.cpp:117)"""
        if encoding not in INPUT_FORMATS:
            raise ValueError(f"set_input_format: unknown encoding {encoding!r}, not one of {sorted(INPUT_FORMATS)}")
        self._ck(self.L.lsdgpu_set_input_format(self.ptr, INPUT_FORMATS[encoding][0]))
        self.input_format = encoding

    def _raw_shape(self, what: str) -> tuple:
        """the array shape of one raw image in the input format: (h, w) for mono8, (h, w, bytes per pixel) otherwise"""
        if self.raw_size is None:
            raise ValueError(f"{what}: no undistorter installed")
        (w, h), bpp = self.raw_size, INPUT_FORMATS[self.input_format][1]
        return (h, w) if bpp == 1 else (h, w, bpp)

    def _host_raw(self, raw, what: str) -> np.ndarray:
        raw = np.ascontiguousarray(raw, np.uint8)
        shape = self._raw_shape(what)
        if raw.shape != shape:
            raise ValueError(f"{what}: a {self.input_format} image needs shape {shape}, not {raw.shape}")
        return raw

    def _device_raw(self, t, what: str):
        """a CUDA uint8 tensor of the raw shape whose pixels are contiguous within each row -> (pointer, row pitch in bytes, stream)"""
        _tensor_dtype(t, "uint8", what)
        shape = self._raw_shape(what)
        if tuple(t.shape) != shape:
            raise ValueError(f"{what}: a {self.input_format} tensor needs shape {shape}, not {tuple(t.shape)}")
        row = shape[1] * (shape[2] if len(shape) == 3 else 1)
        if t.stride(1) != (shape[2] if len(shape) == 3 else 1) or (len(shape) == 3 and t.stride(2) != 1) or t.stride(0) < row:
            raise ValueError(f"{what}: needs contiguous rows (stride(0) >= {row} bytes), not strides {t.stride()}")
        return t.data_ptr(), t.stride(0), _cuda_stream(t, self.device, what)

    def stage_put_raw(self, index: int, raw):
        """camera image in, prefetch-ring entry out: converts (input format), undistorts and writes the gray result into ring entry
        `index` (lsdgpu_stage_put_raw); a CUDA tensor is read on the device, ordered on its current stream, without waiting for the
        device (lsdgpu_stage_put_raw_device)"""
        if _is_tensor(raw):
            ptr, pitch, stream = self._device_raw(raw, "stage_put_raw")
            self._ck(self.L.lsdgpu_stage_put_raw_device(self.ptr, index, ptr, pitch, stream))
            return
        img = self._host_raw(raw, "stage_put_raw")
        self._ck(self.L.lsdgpu_stage_put_raw(self.ptr, index, img.ctypes.data_as(C.POINTER(C.c_uint8))))

    def undistort(self, raw_u8: np.ndarray) -> np.ndarray:
        """UndistorterPTAM::undistort (Undistorter.cpp:355-411) or UndistorterOpenCV::undistort (:564-567), whichever is installed,
        of a raw image in the input format (converted to gray first)"""
        raw = np.ascontiguousarray(raw_u8, np.uint8) if self.input_format == "mono8" else self._host_raw(raw_u8, "undistort")
        out = np.zeros((self.h, self.w), np.uint8)
        self._ck(self.L.lsdgpu_undistort_u8(self.ptr, raw.ctypes.data_as(C.POINTER(C.c_uint8)), out.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out

    def upload_distorted(self, fid: int, raw_u8):
        """undistort (either model) + Frame construction fused (one H2D copy of the raw image, remap feeds the pyramid kernel).
        raw_u8 may be a CUDA tensor as `upload` takes it, of the undistorter's input size (lsdgpu_frame_upload_distorted_device_u8).
        In another input format than mono8 (set_input_format) the image is (h, w, bytes per pixel), converted to gray on the device."""
        if _is_tensor(raw_u8):
            if self.raw_size is None:
                raise ValueError("upload_distorted: no undistorter installed")
            if self.input_format == "mono8":
                ptr, pitch, stream = _device_image(raw_u8, self.device, *self.raw_size, "upload_distorted")
            else:
                ptr, pitch, stream = self._device_raw(raw_u8, "upload_distorted")
            self._ck(self.L.lsdgpu_frame_upload_distorted_device_u8(self.ptr, fid, ptr, pitch, stream))
            return
        raw = np.ascontiguousarray(raw_u8, np.uint8) if self.input_format == "mono8" else self._host_raw(raw_u8, "upload_distorted")
        self._ck(self.L.lsdgpu_frame_upload_distorted_u8(self.ptr, fid, raw.ctypes.data_as(C.POINTER(C.c_uint8))))

    def pack_pointcloud(self, kf_id: int, level: int = 0, out=None):
        """keyframeMsg.pointcloud of ROSOutput3DWrapper::publishKeyframe (ROSOutput3DWrapper.cpp:91-110), packed on the device.
        out = a contiguous uint8 CUDA tensor of at least 12 bytes per record: the records are written there, ordered on its
        current stream (lsdgpu_keyframe_pack_pointcloud_device); returns a (n, 12) view of out"""
        n = (self.w >> level) * (self.h >> level)
        if out is not None:
            stream = _device_out(out, "uint8", n * POINT_DENSE.itemsize, self.device, "pack_pointcloud(out=)")
            self._ck(self.L.lsdgpu_keyframe_pack_pointcloud_device(self.ptr, kf_id, level, out.data_ptr(), out.numel(), stream))
            return out.reshape(-1)[:n * POINT_DENSE.itemsize].view(n, POINT_DENSE.itemsize)
        out = np.zeros(n, POINT_DENSE)
        self._ck(self.L.lsdgpu_keyframe_pack_pointcloud(self.ptr, kf_id, level, out.ctypes.data_as(_vp)))
        return out

    def cloud_reserve(self, max_keyframes_per_launch: int):
        """device buffers of export_pointcloud (lsdgpu_cloud_reserve): larger exports run in batches of this many keyframes"""
        self._ck(self.L.lsdgpu_cloud_reserve(self.ptr, int(max_keyframes_per_launch)))

    def export_pointcloud(self, kf_ids, camToWorld, level: int = 0, filter=None, layout: int = CLOUD_PLY, capacity=None, out=None):
        """the viewer's point cloud of keyframes kf_ids (KeyFrameDisplay::refreshPC + flushPC, KeyFrameDisplay.cpp:106-222,
        :269-339), filtered and transformed on the device: camToWorld = (n, 7) float32 Sim3f data (keyframeMsg.camToWorld).
        filter: CloudFilter, dict of its fields, or None (the viewer's defaults).  Returns (points, counts): points in keyframe
        order (CLOUD_PLY_DTYPE world points + intensity, or CLOUD_VERTEX_DTYPE camera points + colour), counts = (n, 2) int32
        totalPoints, displayedPoints.  Needs cloud_reserve first.  capacity=None sizes the output for every interior pixel;
        out = a caller's array of the layout's dtype to fill instead (its length is the capacity; the points are a view of it).
        out = a contiguous float32 CUDA tensor of shape (capacity, 4): the points are written there on the device, ordered on its
        current stream, in one launch and without a reservation (lsdgpu_map_export_pointcloud_device); points = a view of out."""
        ids = np.ascontiguousarray(kf_ids, np.int32).reshape(-1)
        n = len(ids)
        c2w = np.ascontiguousarray(camToWorld, np.float32).reshape(n, 7)
        if filter is None or isinstance(filter, dict):
            filter = default_cloud_filter(**(filter or {}))
        if out is not None and _is_tensor(out):
            _tensor_dtype(out, "float32", "export_pointcloud(out=)")
            if out.dim() != 2 or out.shape[1] != 4 or not out.is_contiguous():
                raise ValueError(f"export_pointcloud(out=): needs a contiguous (capacity, 4) tensor, not {tuple(out.shape)}")
            stream = _cuda_stream(out, self.device, "export_pointcloud(out=)")
            counts = np.zeros((n, 2), np.int32)
            npts = C.c_int64(0)
            self._ck(self.L.lsdgpu_map_export_pointcloud_device(self.ptr, n, ids.ctypes.data_as(_ip), c2w.ctypes.data_as(_fp), level,
                                                                C.byref(filter), layout, out.data_ptr(), out.shape[0], C.byref(npts),
                                                                counts.ctypes.data_as(C.POINTER(C.c_int32)), stream))
            return out[:npts.value], counts
        wl, hl = self.w >> level, self.h >> level
        if out is None:
            if capacity is None:
                capacity = n * max(wl - 2, 0) * max(hl - 2, 0)
            out = np.empty(max(int(capacity), 1), CLOUD_VERTEX_DTYPE if layout == CLOUD_VERTEX else CLOUD_PLY_DTYPE)
        else:
            assert out.flags.c_contiguous and out.dtype.itemsize == 16
            capacity = len(out)
        counts = np.zeros((n, 2), np.int32)
        npts = C.c_int64(0)
        rc = self.L.lsdgpu_map_export_pointcloud(self.ptr, n, ids.ctypes.data_as(_ip), c2w.ctypes.data_as(_fp), level, C.byref(filter),
                                                 layout, out.ctypes.data_as(_vp), int(capacity), C.byref(npts),
                                                 counts.ctypes.data_as(C.POINTER(C.c_int32)))
        self._ck(rc)
        return out[:npts.value], counts

    def count_pointcloud(self, kf_ids, camToWorld, level: int = 0, filter=None):
        """(number of points, counts) of export_pointcloud without the points (out = NULL)"""
        ids = np.ascontiguousarray(kf_ids, np.int32).reshape(-1)
        c2w = np.ascontiguousarray(camToWorld, np.float32).reshape(len(ids), 7)
        if filter is None or isinstance(filter, dict):
            filter = default_cloud_filter(**(filter or {}))
        counts = np.zeros((len(ids), 2), np.int32)
        npts = C.c_int64(0)
        self._ck(self.L.lsdgpu_map_export_pointcloud(self.ptr, len(ids), ids.ctypes.data_as(_ip), c2w.ctypes.data_as(_fp), level,
                                                     C.byref(filter), CLOUD_PLY, None, 0, C.byref(npts),
                                                     counts.ctypes.data_as(C.POINTER(C.c_int32))))
        return npts.value, counts

    def cloud_kernel_ms(self) -> float:
        """device time of the last export's kernels (lsdgpu_cloud_last_kernel_ms)"""
        ms = C.c_float(0)
        self._ck(self.L.lsdgpu_cloud_last_kernel_ms(self.ptr, C.byref(ms)))
        return ms.value

    def take_reactivation_data(self, kf_id: int):
        self._ck(self.L.lsdgpu_frame_take_reactivation_data(self.ptr, kf_id))

    def reactivation_data(self, kf_id: int):
        """(idepth_reAct, idepthVar_reAct, validity_reAct) of Frame::takeReActivationData (Frame.cpp:107-145)"""
        a, b = np.zeros((self.h, self.w), np.float32), np.zeros((self.h, self.w), np.float32)
        c = np.zeros((self.h, self.w), np.uint8)
        self._ck(self.L.lsdgpu_frame_download_reactivation_data(self.ptr, kf_id, a.ctypes.data_as(_fp), b.ctypes.data_as(_fp),
                                                                c.ctypes.data_as(C.POINTER(C.c_uint8))))
        return a, b, c

    def clear_good_mask(self, fid: int):
        self._ck(self.L.lsdgpu_frame_clear_good_mask(self.ptr, fid))


class SE3Tracker:
    """Mirror of lsd_slam::SE3Tracker (Tracking/SE3Tracker.h): ``trackFrame`` + the public result fields."""

    def __init__(self, ctx: Context, mode: int = 1):
        self.ctx = ctx
        self.mode = mode
        self.settings = default_track_settings()
        self.pointUsage = 0.0
        self.lastGoodCount = self.lastBadCount = 0.0
        self.lastMeanRes = self.lastResidual = 0.0
        self.affineEstimation_a, self.affineEstimation_b = 1.0, 0.0
        self.diverged = False
        self.trackingWasGood = False
        self.last = None

    def importFrame(self, kf_id: int):
        """TrackingReference::importFrame + depthHasBeenUpdatedFlag=false (SlamSystem.cpp:907-912)."""
        self.ctx._ck(self.ctx.L.lsdgpu_ref_import(self.ctx.ptr, kf_id))

    def trackFrame(self, kf_id: int, frame_id: int, frameToReference_initialEstimate) -> np.ndarray:
        q = np.ascontiguousarray(frameToReference_initialEstimate, np.float64)
        r = TrackResult()
        self.ctx._ck(self.ctx.L.lsdgpu_se3_track(self.ctx.ptr, kf_id, frame_id, q.ctypes.data_as(_dp),
                                                 C.byref(self.settings), self.mode, C.byref(r)))
        self.last = r
        self.pointUsage, self.lastGoodCount, self.lastBadCount = r.pointUsage, r.lastGoodCount, r.lastBadCount
        self.lastMeanRes, self.lastResidual = r.lastMeanRes, r.lastResidual
        self.affineEstimation_a, self.affineEstimation_b = r.affineEstimation_a, r.affineEstimation_b
        self.diverged, self.trackingWasGood = bool(r.diverged), bool(r.trackingWasGood)
        return np.array(r.frameToRef_qt, np.float64)

    # ---- permaRef tracking (SURVEY 8f row 2), batched over candidate keyframes ----
    def setPermaRef(self, kf_id: int) -> int:
        n = C.c_int()
        self.ctx._ck(self.ctx.L.lsdgpu_frame_set_perma_ref(self.ctx.ptr, kf_id, C.byref(n)))
        return n.value

    def checkPermaRefOverlap(self, kf_ids, refToFrame_qts) -> np.ndarray:
        ids = np.ascontiguousarray(kf_ids, np.int32)
        q = np.ascontiguousarray(refToFrame_qts, np.float64).reshape(len(ids), 7)
        out = np.zeros(len(ids), np.float32)
        self.ctx._ck(self.ctx.L.lsdgpu_perma_overlap_batch(self.ctx.ptr, len(ids), ids.ctypes.data_as(_ip), q.ctypes.data_as(_dp), out.ctypes.data_as(_fp)))
        return out

    def trackFrameOnPermaref(self, kf_ids, frame_id: int, refToFrame_qts):
        ids = np.ascontiguousarray(kf_ids, np.int32)
        q = np.ascontiguousarray(refToFrame_qts, np.float64).reshape(len(ids), 7)
        res = (TrackResult * len(ids))()
        self.ctx._ck(self.ctx.L.lsdgpu_perma_track_batch(self.ctx.ptr, len(ids), ids.ctypes.data_as(_ip), frame_id, q.ctypes.data_as(_dp), res))
        return list(res)

    def eval(self, kf_id: int, frame_id: int, level: int, refToFrame_qt, a=1.0, b=0.0, write_mask=False) -> EvalResult:
        q = np.ascontiguousarray(refToFrame_qt, np.float32)
        r = EvalResult()
        self.ctx._ck(self.ctx.L.lsdgpu_se3_eval(self.ctx.ptr, kf_id, frame_id, level, q.ctypes.data_as(_fp), a, b,
                                                C.byref(self.settings), int(write_mask), C.byref(r)))
        return r


class Sim3Tracker:
    """Mirror of lsd_slam::Sim3Tracker (Tracking/Sim3Tracker.h:59-160); members as the reference names them."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.settings = default_track_settings(main_tracker=False)     # DenseDepthTrackerSettings(), Sim3Tracker.cpp:57
        self.diverged = False
        self.pointUsage = 0.0
        self.lastResidual = self.lastDepthResidual = self.lastPhotometricResidual = 0.0
        self.affineEstimation_a, self.affineEstimation_b = 1.0, 0.0
        self.lastSim3Hessian = np.zeros((7, 7), np.float32)
        self.last: Sim3Result | None = None

    def trackFrameSim3(self, reference_kf_id: int, frame_id: int, frameToReference_initialEstimate, startLevel: int, finalLevel: int) -> np.ndarray:
        """-> frameToReference as qts[8] (unit quaternion, translation, scale)"""
        q = np.ascontiguousarray(frameToReference_initialEstimate, np.float64)
        r = Sim3Result()
        self.ctx._ck(self.ctx.L.lsdgpu_sim3_track(self.ctx.ptr, reference_kf_id, frame_id, q.ctypes.data_as(_dp), startLevel, finalLevel,
                                                  C.byref(self.settings), C.byref(r)))
        self._take(r)
        return np.array(r.frameToRef_qts)

    def trackFrameSim3Batch(self, reference_kf_ids, frame_ids, inits, startLevel: int, finalLevel: int):
        """n independent trackings in one launch -> list of Sim3Result"""
        a = np.ascontiguousarray(reference_kf_ids, np.int32)
        b = np.ascontiguousarray(frame_ids, np.int32)
        q = np.ascontiguousarray(inits, np.float64).reshape(len(a), 8)
        res = (Sim3Result * len(a))()
        self.ctx._ck(self.ctx.L.lsdgpu_sim3_track_batch(self.ctx.ptr, len(a), a.ctypes.data_as(_ip), b.ctypes.data_as(_ip), q.ctypes.data_as(_dp),
                                                        startLevel, finalLevel, C.byref(self.settings), res))
        return list(res)

    def eval(self, reference_kf_id: int, frame_id: int, level: int, refToFrame_qts, a=1.0, b=0.0) -> Sim3EvalResult:
        q = np.ascontiguousarray(refToFrame_qts, np.float64)
        r = Sim3EvalResult()
        self.ctx._ck(self.ctx.L.lsdgpu_sim3_eval(self.ctx.ptr, reference_kf_id, frame_id, level, q.ctypes.data_as(_dp), a, b,
                                                 C.byref(self.settings), C.byref(r)))
        return r

    def _take(self, r: Sim3Result):
        self.last = r
        self.diverged = bool(r.diverged)
        self.pointUsage = r.pointUsage
        self.lastResidual, self.lastDepthResidual, self.lastPhotometricResidual = r.lastResidual, r.lastDepthResidual, r.lastPhotometricResidual
        self.affineEstimation_a, self.affineEstimation_b = r.affineEstimation_a, r.affineEstimation_b
        self.lastSim3Hessian = np.array(r.lastSim3Hessian, np.float32).reshape(7, 7)


class DepthMap:
    """Mirror of lsd_slam::DepthMap (DepthEstimation/DepthMap.h)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def _ids(self, ids):
        a = np.ascontiguousarray(ids, np.int32)
        return a, a.ctypes.data_as(_ip), len(a)

    def reset(self):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_reset(self.ctx.ptr))

    def isValid(self) -> bool:
        return bool(self.ctx.L.lsdgpu_depth_is_valid(self.ctx.ptr))

    def invalidate(self):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_invalidate(self.ctx.ptr))

    def activeKeyFrame(self) -> int:
        return self.ctx.L.lsdgpu_depth_active_keyframe(self.ctx.ptr)

    def initializeFromGTDepth(self, kf_id: int):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_init_from_gt(self.ctx.ptr, kf_id))

    def initializeRandomly(self, kf_id: int, state: RandState) -> RandState:
        """DepthMap::initializeRandomly (DepthMap.cpp:883-916) on the device, drawing from ``state`` as the reference draws from
        rand(); returns the state after the last draw (``state`` itself is left as it was).  The number of draws is kept in
        ``last_draws``."""
        st = state.copy()
        n = C.c_int64(0)
        self.ctx._ck(self.ctx.L.lsdgpu_depth_init_random(self.ctx.ptr, kf_id, C.byref(st), C.byref(n)))
        self.last_draws = n.value
        return st

    def setHypotheses(self, kf_id: int, hyp, reactivated=False, do_set_depth=True):
        """the hypotheses of keyframe kf_id: a HYP_DTYPE host array of (h, w), or a contiguous uint8 CUDA tensor of its w * h * 32
        bytes (16-byte aligned, e.g. from current(out=...)), read on the device in order on its current stream
        (lsdgpu_depth_set_hypotheses_device)"""
        if _is_tensor(hyp):
            n = self.ctx.w * self.ctx.h * HYP_DTYPE.itemsize
            stream = _device_out(hyp, "uint8", n, self.ctx.device, "setHypotheses")
            if hyp.numel() != n:
                raise ValueError(f"setHypotheses: needs {n} bytes of hypotheses, not {hyp.numel()}")
            self.ctx._ck(self.ctx.L.lsdgpu_depth_set_hypotheses_device(self.ctx.ptr, kf_id, hyp.data_ptr(), int(reactivated),
                                                                       int(do_set_depth), stream))
            return
        a = np.ascontiguousarray(hyp)
        assert a.dtype == HYP_DTYPE
        self.ctx._ck(self.ctx.L.lsdgpu_depth_set_hypotheses(self.ctx.ptr, kf_id, a.ctypes.data_as(C.POINTER(Hyp)),
                                                            int(reactivated), int(do_set_depth)))

    def setFromExistingKF(self, kf_id: int):
        """DepthMap::setFromExistingKF (DepthMap.cpp:920-962) from the keyframe's device-resident reactivation data"""
        self.ctx._ck(self.ctx.L.lsdgpu_depth_set_from_existing_kf(self.ctx.ptr, kf_id))

    def updateKeyframe(self, referenceFrames):
        """DepthMap::updateKeyframe (DepthMap.cpp:1072-1213).  An item is a frame id (tracked on the active keyframe) or a pair
        (frame id, refToKf_qts) for a frame tracked on another keyframe -- refToKf = activeKeyFrame->getScaledCamToWorld().inverse()
        * frame->getScaledCamToWorld() (:1099), which the owner of the pose graph computes."""
        items = list(referenceFrames)
        if all(isinstance(it, (int, np.integer)) for it in items):
            a, p, n = self._ids(items)
            self.ctx._ck(self.ctx.L.lsdgpu_depth_update_keyframe(self.ctx.ptr, p, n))
            return
        descs = (RefDesc * len(items))()
        for d, it in zip(descs, items):
            if isinstance(it, (int, np.integer)):
                d.frame_id, d.tracked_on_kf = int(it), 1
            else:
                d.frame_id, d.tracked_on_kf = int(it[0]), 0
                d.refToKf_qts[:] = [float(v) for v in it[1]]
        self.ctx._ck(self.ctx.L.lsdgpu_depth_update_keyframe_refs(self.ctx.ptr, descs, len(items)))

    def createKeyFrame(self, new_kf_id: int) -> np.ndarray:
        q = np.zeros(8, np.float64)
        self.ctx._ck(self.ctx.L.lsdgpu_depth_create_keyframe(self.ctx.ptr, new_kf_id, q.ctypes.data_as(_dp)))
        return q

    def finalizeKeyFrame(self):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_finalize_keyframe(self.ctx.ptr))

    def observeDepth(self, referenceFrames):
        a, p, n = self._ids(referenceFrames)
        self.ctx._ck(self.ctx.L.lsdgpu_depth_observe(self.ctx.ptr, p, n))

    def regularizeFillHoles(self):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_regularize_fill_holes(self.ctx.ptr))

    def regularize(self, removeOcclusions: bool, validityTH: int = 24):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_regularize(self.ctx.ptr, int(removeOcclusions), validityTH))

    def propagateDepth(self, new_kf_id: int):
        self.ctx._ck(self.ctx.L.lsdgpu_depth_propagate(self.ctx.ptr, new_kf_id))

    def current(self, out=None):
        """currentDepthMap as a HYP_DTYPE host array of (h, w), or -- out = a contiguous uint8 CUDA tensor of at least w * h * 32
        bytes, 16-byte aligned -- written into out on the device, ordered on its current stream; returns a (h, w, 32) view of out
        (lsdgpu_depth_download_device), whose fields hyp_fields() gives"""
        if out is not None:
            h, w, rec = self.ctx.h, self.ctx.w, HYP_DTYPE.itemsize
            stream = _device_out(out, "uint8", h * w * rec, self.ctx.device, "current(out=)")
            self.ctx._ck(self.ctx.L.lsdgpu_depth_download_device(self.ctx.ptr, out.data_ptr(), out.numel(), stream))
            return out.reshape(-1)[:h * w * rec].view(h, w, rec)
        out = np.zeros((self.ctx.h, self.ctx.w), HYP_DTYPE)
        self.ctx._ck(self.ctx.L.lsdgpu_depth_download(self.ctx.ptr, out.ctypes.data_as(C.POINTER(Hyp))))
        return out

    def integral(self) -> np.ndarray:
        out = np.zeros((self.ctx.h, self.ctx.w), np.int32)
        self.ctx._ck(self.ctx.L.lsdgpu_depth_download_integral(self.ctx.ptr, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out
