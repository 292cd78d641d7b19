"""lsdgpu_track_and_map_group: K streams advanced by one call, their trackings in one launch, must equal K single
lsdgpu_track_and_map calls issued one after the other -- bit for bit in the tracking results, the frame poses and counters,
the refPixelWasGood masks, the new keyframes' thisToParent and the depth maps."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup

pytestmark = pytest.mark.gpu
KF_EVERY = 20
LOOK_AWAY = np.array([0, 0.7071067811865476, 0, 0.7071067811865476, 0, 0, 0], np.float64)   # 90 deg about y: no point stays in view

_frames_cache = {}


def _frames(w, h, s, n):
    """stream s: its own synthetic sequence (seed 1234 + 1000 s, as scripts/bench_streams.py)"""
    key = (w, h, s)
    seq, fr = _frames_cache.get(key, (None, []))
    if seq is None:
        seq = synth.Sequence(w, h, seed=1234 + 1000 * s)
    while len(fr) < n:
        fr.append(seq.render(len(fr)))
    _frames_cache[key] = (seq, fr)
    return seq, fr


def _make_streams(w, h, phases, n_frames):
    streams, frames = [], []
    for s, ph in enumerate(phases):
        seq, fr = _frames(w, h, s, n_frames)
        ctx = abi.Context(w, h, seq.K, max_frames=8)
        gs = GpuStream(ctx, mode=1, kf_every=KF_EVERY, kf_phase=ph)
        gs.init_gt(0, fr[0][0], fr[0][1])
        streams.append(gs)
        frames.append(fr)
    return streams, frames


def _observe(gs, fid, qts):
    ctx = gs.ctx
    pose, parent, itr = ctx.get_pose(fid)
    return {"result": bytes(gs.tracker.last), "pose": pose.tobytes(), "parent": parent, "itr": np.float32(itr).tobytes(),
            "new_kf_qts": None if qts is None else np.asarray(qts).tobytes(),
            "counters": (ctx.get_counters(fid), ctx.get_counters(gs.kf_id)),
            "mask": ctx.download(fid, abi.BUF_GOODMASK).tobytes(),
            "depth": gs.map.current().tobytes()}


def _run(w, h, phases, n_steps, grouped, before_step=None):
    """grouped(k): step k is one group call (True) or one single call per stream (False).  before_step(k, streams) may change
    the streams' state first.  Returns per step and stream what _observe saw, and whether the step diverged."""
    streams, frames = _make_streams(w, h, phases, n_steps + 1)
    group = GpuStreamGroup(streams)
    log = []
    try:
        for k in range(1, n_steps + 1):
            if before_step:
                before_step(k, streams)
            kf = [gs.next_is_keyframe_change() for gs in streams]
            if grouped(k):
                try:
                    group.step([k] * len(streams), images=[f[k][0] for f in frames])
                except RuntimeError:
                    pass
                qts = [group._qts[i].copy() if kf[i] else None for i in range(len(streams))]
            else:
                qts = []
                for i, (gs, f) in enumerate(zip(streams, frames)):
                    try:
                        gs.step(k, f[k][0])
                    except RuntimeError:
                        pass
                    qts.append(gs._qts.copy() if kf[i] else None)
            log.append([dict(_observe(gs, k, q), diverged=bool(gs.tracker.diverged), kf=kf[i])
                        for i, (gs, q) in enumerate(zip(streams, qts))])
    finally:
        for gs in streams:
            gs.ctx.close()
    return log


def _assert_same(a, b):
    assert len(a) == len(b)
    for k, (sa, sb) in enumerate(zip(a, b), start=1):
        for s, (oa, ob) in enumerate(zip(sa, sb)):
            for key in oa:
                assert oa[key] == ob[key], f"step {k}, stream {s}: {key} differs"


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_group_equals_single_calls_640x480(n):
    """25 frames, one keyframe change per stream, in a different step for every stream: groups mix update and create"""
    phases = [2 * s for s in range(n)]              # keyframe changes at steps 20, 18, 16, ...
    single = _run(640, 480, phases, 25, lambda k: False)
    group = _run(640, 480, phases, 25, lambda k: True)
    changes = [[k for k, step in enumerate(single, start=1) if step[s]["kf"]] for s in range(n)]
    assert all(len(c) == 1 for c in changes) and len({c[0] for c in changes}) == n
    assert not any(o["diverged"] for step in single for o in step)
    _assert_same(group, single)


def test_group_equals_single_calls_1280x1024_n8():
    """at 1280x1024 a CTA of an 8-stream group stands in for up to 9 virtual CTAs of ~5 level-1 slots per warp each: more
    good-mask flags per thread than one 32-bit word holds"""
    phases = [15 + s % 5 for s in range(8)]         # keyframe changes at steps 5, 4, 3, 2, 1, 5, 4, 3
    single = _run(1280, 1024, phases, 5, lambda k: False)
    group = _run(1280, 1024, phases, 5, lambda k: True)
    assert all(sum(step[s]["kf"] for step in single) == 1 for s in range(8))
    _assert_same(group, single)


def test_group_and_single_calls_alternated():
    """group and single calls on the same contexts: the barrier bookkeeping of either launch stays right after the other"""
    phases = [10, 12, 14]                            # keyframe changes at steps 10, 8, 6
    single = _run(640, 480, phases, 12, lambda k: False)
    mixed = _run(640, 480, phases, 12, lambda k: k % 2 == 0)
    _assert_same(mixed, single)


def test_group_divergence_skips_only_that_streams_mapping():
    """one stream starts from a pose that puts every point out of view (SE3Tracker.cpp:324-329): it diverges, its map stays as it
    was, and the other streams track and map exactly as with single calls"""
    def look_away(k, streams):
        if k == 3:
            streams[1].last_pose = LOOK_AWAY.copy()
    phases = [0, 0, 0]
    single = _run(640, 480, phases, 3, lambda k: False, look_away)
    group = _run(640, 480, phases, 3, lambda k: True, look_away)
    assert [o["diverged"] for o in group[2]] == [False, True, False]
    assert group[2][1]["depth"] == group[1][1]["depth"]       # the diverged stream's map did not change
    _assert_same(group, single)


def _ctx(w, h, seed=1234):
    seq = synth.Sequence(w, h, seed=seed)
    img, depth = seq.render(0)
    ctx = abi.Context(w, h, seq.K, max_frames=8)
    ctx.upload(0, img)
    ctx.set_depth_gt(0, depth)
    abi.DepthMap(ctx).initializeFromGTDepth(0)
    return ctx, seq


def _call(steps_spec, img):
    n = len(steps_spec)
    steps = (abi.GroupStep * max(n, 1))()
    keep = np.ascontiguousarray(img, np.uint8)
    settings = abi.default_track_settings()
    for st, (ctx, kf_id, fid) in zip(steps, steps_spec):
        st.ctx, st.kf_id, st.frame_id = ctx.ptr, kf_id, fid
        st.gray, st.stage_index = keep.ctypes.data_as(C.POINTER(C.c_uint8)), -1
        st.frameToRef_init_qt[:] = [0, 0, 0, 1, 0, 0, 0]
        st.settings = C.pointer(settings)
    res = (abi.TrackResult * max(n, 1))()
    return abi.load().lsdgpu_track_and_map_group(n, steps, res, None)


def test_group_rejects_bad_input():
    a, seq = _ctx(320, 240)
    b, _ = _ctx(320, 240, 2234)
    c, _ = _ctx(320, 240, 3234)
    big, _ = _ctx(640, 480)
    img = seq.render(1)[0]
    try:
        def rejected(spec, step, what):
            assert _call(spec, img) != 0
            for ctx in {id(x[0]): x[0] for x in spec}.values():
                msg = abi.load().lsdgpu_last_error(ctx.ptr).decode()
                assert what in msg and (step is None or f"step {step}" in msg), msg
        assert _call([], img) != 0                                             # n = 0
        rejected([(a, 0, 5)] * 9, None, "1..8")                                # n = 9
        rejected([(a, 0, 5), (b, 0, 5), (a, 0, 6)], 2, "same context")
        rejected([(a, 0, 5), (big, 0, 5)], 1, "size")
        rejected([(a, 0, 5), (b, 0, 5), (c, 77, 5)], 2, "unknown frame id")
        # nothing was done: no frame 5 exists anywhere
        for ctx in (a, b, c, big):
            with pytest.raises(abi.LsdGpuError):
                ctx.get_pose(5)
        # and a valid group still works afterwards
        assert _call([(a, 0, 5), (b, 0, 5), (c, 0, 5)], img) == 0
    finally:
        for ctx in (a, b, c, big):
            ctx.close()


def test_group_rejects_contexts_on_different_devices():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    a, seq = _ctx(320, 240)
    seq1 = synth.Sequence(320, 240, seed=1234)
    img, depth = seq1.render(0)
    d1 = abi.Context(320, 240, seq1.K, device=1, max_frames=8)
    try:
        d1.upload(0, img)
        d1.set_depth_gt(0, depth)
        abi.DepthMap(d1).initializeFromGTDepth(0)
        assert _call([(a, 0, 5), (d1, 0, 5)], seq.render(1)[0]) != 0
        assert "step 1" in abi.load().lsdgpu_last_error(a.ptr).decode()
    finally:
        a.close()
        d1.close()
