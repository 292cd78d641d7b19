"""Sequential track + map loop over one image stream -- the part of SlamSystem that sits directly above the hot
path, in ``dataset_slam _hz:=0`` (blockUntilMapped) order:

    SlamSystem::trackFrame        SlamSystem.cpp:890-1040   new Frame -> importFrame if the KF depth changed
                                                            (:907-912) -> tracker->trackFrame (:932)
    SlamSystem::doMappingIteration SlamSystem.cpp:739-828   updateKeyframe (:794 -> :542-614), or on a keyframe
                                                            change finalizeKeyFrame (:400) + createKeyFrame (:473)

Keyframe SELECTION (SlamSystem.cpp:998-1020), the pose graph and loop closures are out of scope: a new keyframe
is forced every ``kf_every`` frames (SURVEY 8d).  This driver only issues C-ABI calls; it is what bench.py
times and what the full-loop parity tests run.  ``fused_call=True`` issues the whole frame as ONE ABI call
(``lsdgpu_track_and_map``, same call sequence inside the library); ``False`` issues the individual calls.

The stream keeps the ids of its keyframes and their camToWorld, chained from the thisToParent Sim3 that createKeyFrame returns
(odometry: no pose graph), so that ``ctx.export_pointcloud(stream.keyframe_ids, stream.keyframe_cam_to_world_f7())`` is the
viewer's map of the run.  With ``keep_keyframes=True`` finished keyframes stay resident (the context needs a frame slot for each).

``GpuStreamGroup`` steps K such streams (one context each, same GPU) with ONE call per frame
(``lsdgpu_track_and_map_group``): the trackings of the K frames share one launch, each stream on its own slice of the SMs.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi

IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
IDENT_QTS = np.array([0, 0, 0, 1, 0, 0, 0, 1], np.float64)


def _quat_mul(a, b):
    """Hamilton product of (x, y, z, w) quaternions"""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def _quat_rot(q, v):
    u = np.cross(q[:3], v)
    u = u + u
    return v + q[3] * u + np.cross(q[:3], u)


def sim3_mul_qts(a, b) -> np.ndarray:
    """a * b for Sim3 as qts[8] (unit quaternion x,y,z,w, translation, scale), in double"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    q = _quat_mul(a[:4], b[:4])
    q /= np.sqrt(q @ q)
    t = a[7] * _quat_rot(a[:4], b[4:7]) + a[4:7]
    return np.concatenate([q, t, [a[7] * b[7]]])


def qts_to_sim3f(qts) -> np.ndarray:
    """the ABI's Sim3 qts[8] as the 7 floats of keyframeMsg.camToWorld: Sophus::Sim3f::data() of getScaledCamToWorld().cast<float>()
    (the quaternion scaled by the scale, then the translation; ROSOutput3DWrapper.cpp:85-88)"""
    qts = np.asarray(qts, np.float64)
    return np.concatenate([qts[:4] * qts[7], qts[4:7]]).astype(np.float32)


class GpuStream:
    def __init__(self, ctx: abi.Context, mode: int = 1, kf_every: int = 20, fused_call: bool = True, kf_phase: int = 0,
                 keep_keyframes: bool = False):
        self.ctx = ctx
        self.keep_keyframes = keep_keyframes
        self.keyframe_ids: list[int] = []          # every keyframe of the run, oldest first
        self.keyframe_cam_to_world: list[np.ndarray] = []   # their camToWorld as qts[8], the first keyframe at the origin
        self.kf_phase = kf_phase          # shifts the forced keyframe changes: frame n changes keyframe when (n + kf_phase) % kf_every == 0
        self.tracker = abi.SE3Tracker(ctx, mode=mode)
        self.map = abi.DepthMap(ctx)
        self.kf_every = kf_every
        self.fused_call = fused_call
        self.kf_id = None
        self.last_pose = IDENT.copy()
        self.n_tracked = 0
        self.prev_ids: list[int] = []
        self.poses: list[np.ndarray] = []
        self._res = abi.TrackResult()
        self._qts = np.zeros(8, np.float64)

    def init_gt(self, fid: int, image_u8: np.ndarray, depth: np.ndarray):
        """SlamSystem::gtDepthInit, SlamSystem.cpp:831-854"""
        self.ctx.upload(fid, image_u8)
        self.ctx.set_depth_gt(fid, depth)
        self.map.initializeFromGTDepth(fid)
        self.kf_id = fid
        self.last_pose = IDENT.copy()
        self.keyframe_ids, self.keyframe_cam_to_world = [fid], [IDENT_QTS.copy()]

    def keyframe_cam_to_world_f7(self) -> np.ndarray:
        """(n, 7) float32 camToWorld of keyframe_ids, as keyframeMsg carries them"""
        return np.stack([qts_to_sim3f(q) for q in self.keyframe_cam_to_world])

    def _track_and_map_fused(self, fid, image_u8, stage_index, kf_change):
        ctx, trk = self.ctx, self.tracker
        img = None
        if image_u8 is not None:
            img = np.ascontiguousarray(image_u8, np.uint8).ctypes.data_as(C.POINTER(C.c_uint8))
        q = np.ascontiguousarray(self.last_pose, np.float64)
        r = self._res
        ctx._ck(ctx.L.lsdgpu_track_and_map(ctx.ptr, self.kf_id, fid, img, -1 if stage_index is None else stage_index,
                                           q.ctypes.data_as(C.POINTER(C.c_double)), C.byref(trk.settings), trk.mode,
                                           int(kf_change), C.byref(r), self._qts.ctypes.data_as(C.POINTER(C.c_double))))
        return self._take_result(r)

    def _take_result(self, r: abi.TrackResult) -> np.ndarray:
        """the tracker's public fields after a fused call (SE3Tracker.h:82-93); returns frameToRef"""
        trk = self.tracker
        trk.last = r
        trk.pointUsage, trk.lastGoodCount, trk.lastBadCount = r.pointUsage, r.lastGoodCount, r.lastBadCount
        trk.lastMeanRes, trk.lastResidual = r.lastMeanRes, r.lastResidual
        trk.affineEstimation_a, trk.affineEstimation_b = r.affineEstimation_a, r.affineEstimation_b
        trk.diverged, trk.trackingWasGood = bool(r.diverged), bool(r.trackingWasGood)
        return np.array(r.frameToRef_qt, np.float64)

    def next_is_keyframe_change(self) -> bool:
        return bool(self.kf_every) and (self.n_tracked + 1 + self.kf_phase) % self.kf_every == 0

    def step(self, fid: int, image_u8: np.ndarray | None = None, stage_index: int | None = None) -> np.ndarray:
        """one frame: Frame construction (host image, or a pre-staged device image), trackFrame, mapping"""
        ctx = self.ctx
        kf_change = self.next_is_keyframe_change()
        if self.fused_call:
            pose = self._track_and_map_fused(fid, image_u8, stage_index, kf_change)
        else:
            if stage_index is not None:
                ctx.frame_from_stage(fid, stage_index)
            else:
                ctx.upload(fid, image_u8)
            if ctx.depth_updated_flag(self.kf_id):
                self.tracker.importFrame(self.kf_id)
            pose = self.tracker.trackFrame(self.kf_id, fid, self.last_pose)
        self.n_tracked += 1
        if self.tracker.diverged:
            raise RuntimeError(f"tracking diverged on frame {fid}")
        if not self.fused_call:
            if kf_change:
                self.map.finalizeKeyFrame()
                self._qts[:] = self.map.createKeyFrame(fid)
            else:
                self.map.updateKeyframe([fid])
                ctx.clear_good_mask(fid)             # SlamSystem.cpp:573
        self._advance(fid, pose, kf_change, self._qts)
        return pose

    def _advance(self, fid: int, pose: np.ndarray, kf_change: bool, new_kf_qts=None):
        """bookkeeping after a mapped frame: the keyframe, the next initial pose and the frames that can be released"""
        ctx = self.ctx
        if kf_change:
            old_kf, self.kf_id = self.kf_id, fid
            self.last_pose = IDENT.copy()
            if self.keyframe_ids:               # the new keyframe's thisToParent (createKeyFrame) chained onto its parent
                self.keyframe_ids.append(fid)
                self.keyframe_cam_to_world.append(sim3_mul_qts(self.keyframe_cam_to_world[-1], new_kf_qts))
            for i in self.prev_ids + ([] if self.keep_keyframes else [old_kf]):
                ctx.release(i)
            self.prev_ids = []
        else:
            self.last_pose = pose
            self.prev_ids.append(fid)
            while len(self.prev_ids) > 1:
                ctx.release(self.prev_ids.pop(0))
        self.poses.append(pose)


class GpuStreamGroup:
    """K independent streams (GpuStream, one context each, all on one GPU, same size) advanced by one frame each with ONE C-ABI
    call (lsdgpu_track_and_map_group).  Same keyframe policy and release bookkeeping as GpuStream.step, per stream; the result
    of every stream is bit-identical to stepping the streams one after the other with GpuStream.step."""

    def __init__(self, streams: list[GpuStream]):
        n = len(streams)
        if not 1 <= n <= abi.GROUP_MAX_STEPS:
            raise ValueError(f"a group holds 1..{abi.GROUP_MAX_STEPS} streams, not {n}")
        if any(s.tracker.mode != 1 for s in streams):
            raise ValueError("grouped tracking is the device-resident tracker (mode 1)")
        self.streams = streams
        self.L = streams[0].ctx.L
        self._steps = (abi.GroupStep * n)()
        self._res = (abi.TrackResult * n)()
        self._qts = np.zeros((n, 8), np.float64)

    def step(self, fids, images=None, stage_indices=None) -> list[np.ndarray]:
        """one frame per stream: fids[s] is stream s's new frame id, from images[s] (host u8) or ring entry stage_indices[s]"""
        n = len(self.streams)
        kf_changes = [s.next_is_keyframe_change() for s in self.streams]
        keep = []                                  # the host images must live until the call returns
        for i, (gs, st) in enumerate(zip(self.streams, self._steps)):
            st.ctx = gs.ctx.ptr
            st.kf_id, st.frame_id = gs.kf_id, fids[i]
            if images is not None:
                img = np.ascontiguousarray(images[i], np.uint8)
                keep.append(img)
                st.gray, st.stage_index = img.ctypes.data_as(C.POINTER(C.c_uint8)), -1
            else:
                st.gray, st.stage_index = None, stage_indices[i]
            st.frameToRef_init_qt[:] = [float(x) for x in gs.last_pose]
            st.settings = C.pointer(gs.tracker.settings)
            st.keyframe_change = int(kf_changes[i])
        rc = self.L.lsdgpu_track_and_map_group(n, self._steps, self._res, self._qts.ctypes.data_as(C.POINTER(C.c_double)))
        if rc != 0:
            raise abi.LsdGpuError(f"rc={rc}: {self.L.lsdgpu_last_error(self.streams[0].ctx.ptr).decode()}")
        poses, diverged = [], []
        for i, gs in enumerate(self.streams):
            pose = gs._take_result(abi.TrackResult.from_buffer_copy(self._res[i]))
            gs.n_tracked += 1
            if gs.tracker.diverged:
                diverged.append(fids[i])
                continue
            gs._advance(fids[i], pose, kf_changes[i], self._qts[i])
            poses.append(pose)
        if diverged:
            raise RuntimeError(f"tracking diverged on frame(s) {diverged}")
        return poses
