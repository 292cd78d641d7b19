"""oracle/replay.py -- TEST INFRASTRUCTURE: single-step parity of the CUDA path FROM THE DEVICE'S OWN STATE.

Why single steps.  LSD-SLAM's mapper decides when a pixel is observed next from the low-order bits of a float
(`inc += ((int)(result_eplLength*10000)%2)`, DepthMap.cpp:457; SURVEY App. A-16).  Two runs of THE REFERENCE ITSELF whose
tracked poses differ by 1e-6 relative therefore drift apart: after 19 mapped frames at 640x480 only 98 % of the pixels
still agree to 1e-3 (max 7e-3, <= 0.4 sigma of their own variance; measured with the oracle, DESIGN.md section 5).  A
parallel reduction cannot reproduce the CPU's sequential float sums bit for bit, so a closed-loop comparison over many
frames measures that sensitivity, not the kernels.  `north_star` asks for parity "for identical inputs": this module takes
the device's state before a step (hypotheses, keyframe, counters, initial pose), replays the SAME step on the CPU oracle,
and compares
  * the tracked pose and the LM call counters: <= 1e-4 relative, plus the reference's OWN summation noise on that step (the
    distance between the oracle and its diagnostic twin that accumulates the same fp32 terms exactly -- up to 1.7e-4 on the
    bench streams: the sequential fp32 sums of SE3Tracker.cpp carry ~1e-5 relative error into a 6x6 system whose weak
    directions amplify it), and
  * the device's refPixelWasGood mask against the oracle's own (`mask_mismatch`: pixels that differ), and
  * with the device's pose, residual and good-mask handed to the oracle, the depth map after the step BIT FOR BIT
    (keyframe changes included: the sequential fp32 sum behind the rescale factor, DepthMap.cpp:1286-1294, is reproduced
    exactly by csrc/seqsum.cuh).
Only tests/ and bench.py's parity leg import this.
"""
from __future__ import annotations

import numpy as np

from . import pyoracle as po


def pose_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    dt = float(np.linalg.norm(a[4:7] - b[4:7]) / max(np.linalg.norm(b[4:7]), 1e-12))
    ang = float(2 * np.arccos(min(1.0, abs(float(np.dot(a[:4], b[:4]))))))
    return dt, ang


class Snapshot:
    """what the step about to run will read: taken from the GPU stream BEFORE the step"""

    def __init__(self, gs, images):
        ctx = gs.ctx
        self.kf_id = gs.kf_id
        self.kf_image = images[gs.kf_id]
        self.hyp = gs.map.current().copy()
        self.counters = ctx.get_counters(gs.kf_id)          # (numFramesTrackedOnThis, numMappedOnThis)
        self.last_pose = np.array(gs.last_pose, np.float64)
        self.kf_change = bool(gs.kf_every) and (gs.n_tracked + 1) % gs.kf_every == 0


FLOAT_FIELDS = ("idepth", "idepth_var", "idepth_smoothed", "idepth_var_smoothed", "nextStereoFrameMinID")


def map_report(a, b):
    """flags on every pixel, the other fields on valid pixels: mismatch counts (bit patterns) and max relative error"""
    va, vb = a["isValid"] != 0, b["isValid"] != 0
    rep = {"valid_mismatch": int((va != vb).sum()), "blacklist_mismatch": int((a["blacklisted"] != b["blacklisted"]).sum())}
    both = va & vb
    rep["n_valid"] = int(both.sum())
    rep["validity_mismatch"] = int((a["validity_counter"][both] != b["validity_counter"][both]).sum())
    for f in FLOAT_FIELDS:
        x, y = a[f][both], b[f][both]
        rep[f + "_bitdiff"] = int((x.view(np.uint32) != y.view(np.uint32)).sum())
        rep[f + "_maxrel"] = float(np.max(np.abs(x - y) / np.maximum(np.abs(y), 1e-12))) if x.size else 0.0
    return rep


def oracle_keyframe(seq, snap: Snapshot):
    """the oracle's keyframe and depth map in the device's pre-step state of `snap` (C restatement, current settings)"""
    L = po.lib(False)
    hyp_c = np.ascontiguousarray(snap.hyp)
    kf = po.Frame(snap.kf_id, snap.kf_image, seq.K, fast=False)
    kf.setDepthFromGroundTruth(np.ones((seq.h, seq.w), np.float32))    # only to attach the frame as the active keyframe
    dm = po.DepthMap(seq.w, seq.h, seq.K, fast=False)
    dm.initializeFromGTDepth(kf)
    dm.set_current(snap.hyp)
    L.lsdo_frame_setDepth(kf.ptr, hyp_c.ctypes.data_as(po.C.POINTER(po.Hyp)))   # Frame::setDepth(currentDepthMap), DepthMap.cpp:1153 / 1311
    L.lsdo_frame_set_counters(kf.ptr, int(snap.counters[0]), int(snap.counters[1]))
    L.lsdo_frame_set_depthHasBeenUpdatedFlag(kf.ptr, 0)
    return kf, dm


def start_outcomes(seq, snap: Snapshot, fid: int, image_u8, n=20, eps=1e-6, seed=0):
    """the oracle's trackFrame of the step of `snap` from its start pose with the translation moved by eps (relative) in n seeded
    directions (a start near the identity by eps * 1e-2 absolute) -> list of (pose, numCalcResidualCalls, numCalcWarpUpdateCalls).  Where the tracking cost has several minima
    close together (a texture that repeats along the motion), starts closer than the fp32 resolution of a pose can end in
    different minima: these are the outcomes the reference arithmetic itself reaches from the step's state"""
    rng = np.random.default_rng(seed)
    outs = []
    for _ in range(n):
        q = np.array(snap.last_pose, np.float64)
        d = rng.normal(size=3)
        q[4:7] += d / np.linalg.norm(d) * eps * max(np.linalg.norm(q[4:7]), 1e-2)       # an identity start moves by 1e-2 eps
        kf, _dm = oracle_keyframe(seq, snap)
        r = po.se3_track(kf, po.Frame(fid, image_u8, seq.K, fast=False), q, po.default_track_settings(False))
        outs.append((np.array(r.frameToRef_qt, np.float64), list(r.numCalcResidualCalls), list(r.numCalcWarpUpdateCalls)))
    return outs


def replay_step(seq, snap: Snapshot, fid: int, image_u8, gs, settings=None, globals_kw=None):
    """Replay on the oracle the step GpuStream `gs` has JUST executed for frame `fid` from state `snap`, under the run-time settings
    of util/settings.cpp:80-88 the context holds (or `globals_kw` instead, e.g. to show that other values give another result).
    Returns a dict with the pose error, counter equality and the map comparison; "globals" is the settings the oracle used."""
    from lsd_slam_b200 import abi
    ctx = gs.ctx
    fl = False
    g = ctx.get_globals() if globals_kw is None else dict(globals_kw)
    po.set_globals(fl, **g)
    L = po.lib(fl)
    st = settings or po.default_track_settings(fl)

    def make_kf():
        return oracle_keyframe(seq, snap)

    # the reference's OWN summation noise on this step: the same tracking with every sum accumulated exactly (diagnostic twin of
    # the oracle, lsdo_globals.exactTrackingSums) -- what the sequential fp32 sums of SE3Tracker.cpp approximate
    po.set_globals(fl, exactTrackingSums=1, **g)
    xkf, _xdm = make_kf()
    xf = po.Frame(fid, image_u8, seq.K, fast=fl)
    pose_x = np.array(po.se3_track(xkf, xf, snap.last_pose, st).frameToRef_qt, np.float64)
    po.set_globals(fl, **g)
    okf, odm = make_kf()
    of = po.Frame(fid, image_u8, seq.K, fast=fl)
    r = po.se3_track(okf, of, snap.last_pose, st)
    res = gs.tracker.last
    pose_g = np.array(res.frameToRef_qt, np.float64)
    pose_o = np.array(r.frameToRef_qt, np.float64)
    out = {"frame": fid, "kf_change": snap.kf_change, "globals": g}
    out["pose_rel"], out["rot_rad"] = pose_err(pose_g, pose_o)
    out["ref_noise_rel"], out["ref_noise_rot"] = pose_err(pose_o, pose_x)      # reference (fp32 sequential sums) vs exact sums
    out["pose_rel_exact"], _ = pose_err(pose_g, pose_x)                        # device vs exact sums
    out["pose"], out["residual_calls"] = pose_g, list(res.numCalcResidualCalls)
    out["counts_equal"] = (list(res.numCalcResidualCalls) == list(r.numCalcResidualCalls)
                           and list(res.numCalcWarpUpdateCalls) == list(r.numCalcWarpUpdateCalls))
    out["stats"] = {"lastResidual": (res.lastResidual, r.lastResidual), "pointUsage": (res.pointUsage, r.pointUsage),
                    "good": (res.lastGoodCount, r.lastGoodCount), "bad": (res.lastBadCount, r.lastBadCount)}
    # mapping from IDENTICAL inputs: the device's pose, residual, mask and counters
    if snap.kf_change:
        qts_g = np.concatenate([pose_g, [1.0]])
        itr_g = res.initialTrackedResidual
        mask_g = ctx.download(fid, abi.BUF_GOODMASK)        # still there: createKeyFrame does not clear it
    else:
        qts_g, _, itr_g = ctx.get_pose(fid)
        mask_g = None                                       # cleared after mapping (SlamSystem.cpp:573): taken by the caller before
    out["_need_mask"] = mask_g is None
    out["_objs"] = (okf, odm, of, qts_g, itr_g, mask_g, r)
    return out


def finish_replay(seq, snap: Snapshot, out, gs, mask_before_clear=None, rescale_tol=0.0):
    """second half of replay_step: map the frame on the oracle with the device's pose / residual / mask and compare maps"""
    okf, odm, of, qts_g, itr_g, mask_g, r = out.pop("_objs")
    out.pop("_need_mask")
    L = po.lib(False)
    if mask_g is None:
        mask_g = mask_before_clear
    qts = np.array(qts_g, np.float64)
    if snap.kf_change:
        qts[7] = 1.0
    of.set_thisToParent(qts, okf)
    L.lsdo_frame_set_initialTrackedResidual(of.ptr, float(itr_g))
    if mask_g is not None:
        # the device's refPixelWasGood against the oracle's own tracking of the step (pixels that differ), before it is replaced
        out["mask_mismatch"] = int((of.refPixelWasGood(create=True) != mask_g).sum())
        of.refPixelWasGood(create=True)[:] = mask_g
    tracked_after, mapped_after = gs.ctx.get_counters(snap.kf_id) if not snap.kf_change else (None, None)
    if snap.kf_change:
        odm.finalizeKeyFrame()
        odm.createKeyFrame(of)
        rep = map_report(gs.map.current(), odm.current())
        sc_o = of.thisToParent()[7]
        sc_g = gs.ctx.get_pose(of.id)[0][7]
        out["rescale_rel"] = float(abs(sc_g - sc_o) / sc_o)
        # the rescale factor is the reference's sequential fp32 sum (DepthMap.cpp:1286-1294); the device reproduces that sum bit
        # for bit (csrc/seqsum.cuh), so the new keyframe's map is compared like every other step: bit patterns
        ok = (rep["valid_mismatch"] == 0 and rep["blacklist_mismatch"] == 0 and rep["validity_mismatch"] == 0
              and all(rep[f + "_bitdiff"] == 0 for f in FLOAT_FIELDS) and out["rescale_rel"] <= rescale_tol)
    else:
        # the device counted this frame as tracked iff trackingWasGood; the oracle's own tracking did the same on okf
        L.lsdo_frame_set_counters(okf.ptr, int(tracked_after), int(mapped_after) - 1)
        odm.updateKeyframe([of])
        rep = map_report(gs.map.current(), odm.current())
        ok = (rep["valid_mismatch"] == 0 and rep["blacklist_mismatch"] == 0 and rep["validity_mismatch"] == 0
              and all(rep[f + "_bitdiff"] == 0 for f in FLOAT_FIELDS))
    out["map"] = rep
    out["map_ok"] = bool(ok)
    return out


def run_with_replay(seq, frames, n_frames, kf_every=20, sample=None, mode=1, device=0, max_frames=8, globals_kw=None,
                    before_step=None, keep_snapshots=False):
    """GpuStream over frames 1..n_frames-1 with the oracle replaying the steps in `sample` (None = every step).
    Returns the list of per-step reports.  The stream itself never sees the oracle (it continues from ITS OWN state).
    globals_kw: the context's run-time settings (default: the reference's); before_step(k, ctx) runs before step k, e.g. to change
    them between two frames as a dynamic-reconfigure callback does.  keep_snapshots: each report also holds its step's state
    ("snap") and image ("image"), for start_outcomes.  The oracle is back at the default settings afterwards."""
    from lsd_slam_b200 import abi
    from lsd_slam_b200.stream import GpuStream
    images = {k: frames[k][0] for k in range(n_frames)}
    ctx = abi.Context(seq.w, seq.h, seq.K, device=device, max_frames=max_frames, **(globals_kw or {}))
    gs = GpuStream(ctx, mode=mode, kf_every=kf_every, fused_call=False)
    gs.init_gt(0, frames[0][0], frames[0][1])
    reports = []
    for k in range(1, n_frames):
        if before_step is not None:
            before_step(k, ctx)
        if sample is not None and k not in sample:
            gs.step(k, frames[k][0])
            continue
        snap = Snapshot(gs, images)
        # the unfused stream lets us read the good-mask between tracking and its clearing at the end of the step
        mask_holder = {}
        orig_clear = ctx.clear_good_mask

        def clear_and_keep(fid, _orig=orig_clear, _h=mask_holder):
            _h["mask"] = ctx.download(fid, abi.BUF_GOODMASK)
            return _orig(fid)
        ctx.clear_good_mask = clear_and_keep
        try:
            gs.step(k, frames[k][0])
        finally:
            ctx.clear_good_mask = orig_clear
        out = replay_step(seq, snap, k, frames[k][0], gs)
        out = finish_replay(seq, snap, out, gs, mask_before_clear=mask_holder.get("mask"))
        if keep_snapshots:
            out["snap"], out["image"] = snap, frames[k][0]
        reports.append(out)
    ctx.close()
    po.set_globals(False)
    return reports
