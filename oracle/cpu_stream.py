"""oracle/cpu_stream.py -- TEST INFRASTRUCTURE: the sequential track + map loop of lsd_slam_b200/stream.py on the CPU.

Drives the oracle (or the reference-compiled library oracle/_ref, flavour "ref" / "ref_sse") through exactly the call
sequence GpuStream issues through the C ABI -- SlamSystem's order in `dataset_slam _hz:=0` mode (SlamSystem.cpp:890-1040,
739-828), forced keyframe change every `kf_every` tracked frames -- so that bench.py's CPU arm and the full-loop parity
tests run the same loop on both sides.  Only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this.
"""
from __future__ import annotations

import time

import numpy as np

from . import pyoracle as po

IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


class CpuStream:
    def __init__(self, seq, flavour=False, kf_every: int = 20, settings=None, keep_keyframes: bool = False):
        """keep_keyframes: hold every finished keyframe's Frame in `finished` (with the depth finalizeKeyFrame left in it),
        as the keyframe graph does, instead of dropping it once the next keyframe is made"""
        self.seq, self.fl, self.kf_every, self.keep_keyframes = seq, flavour, kf_every, keep_keyframes
        self.finished: list = []
        self.L = po.lib(flavour)
        self.st = settings or po.default_track_settings(flavour)
        self.kf = None
        self.dm = None
        self.last = IDENT.copy()
        self.n_tracked = 0
        self.keep: list = []
        self.poses: list[np.ndarray] = []
        self.results: list = []
        self.kf_changes: list[int] = []

    def init_gt(self, fid, image_u8, depth):
        """SlamSystem::gtDepthInit, SlamSystem.cpp:831-854"""
        self.kf = po.Frame(fid, image_u8, self.seq.K, fast=self.fl)
        self.kf.setDepthFromGroundTruth(depth)
        self.dm = po.DepthMap(self.seq.w, self.seq.h, self.seq.K, fast=self.fl)
        self.dm.initializeFromGTDepth(self.kf)
        self.keep = [self.kf]
        self.last = IDENT.copy()

    def step(self, fid, image_u8):
        """one frame; returns (frameToReference pose, wall seconds of the three reference calls + Frame construction)"""
        L, kf = self.L, self.kf
        t0 = time.perf_counter()
        f = po.Frame(fid, image_u8, self.seq.K, fast=self.fl)                 # Frame::Frame(uchar*) (u8 -> f32)
        if L.lsdo_frame_depthHasBeenUpdatedFlag(kf.ptr):
            L.lsdo_frame_set_depthHasBeenUpdatedFlag(kf.ptr, 0)              # importFrame, SlamSystem.cpp:907-912
        r = po.se3_track(kf, f, self.last, self.st)
        self.n_tracked += 1
        pose = np.array(r.frameToRef_qt)
        if r.diverged:
            raise RuntimeError(f"CPU arm: tracking diverged on frame {fid}")
        kf_change = bool(self.kf_every) and self.n_tracked % self.kf_every == 0
        if kf_change:
            self.dm.finalizeKeyFrame()
            self.dm.createKeyFrame(f)
            if self.keep_keyframes:
                self.finished.append(self.kf)
            self.kf = f
            self.last = IDENT.copy()
            self.kf_changes.append(fid)
        else:
            self.dm.updateKeyframe([f])
            L.lsdo_frame_clear_refPixelWasGood(f.ptr)                        # SlamSystem.cpp:573
            self.last = pose
        dt = time.perf_counter() - t0
        self.keep.append(f)
        while len(self.keep) > 3:                                            # the keyframe and its parent chain stay alive
            i = 0
            while self.keep[i] is self.kf:
                i += 1
            self.keep.pop(i)
        self.poses.append(pose)
        self.results.append(r)
        return pose, dt
