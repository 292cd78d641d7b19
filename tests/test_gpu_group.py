"""lsdgpu_track_and_map_group: K streams advanced by one call, their trackings in one launch, must equal K single
lsdgpu_track_and_map calls issued one after the other -- bit for bit in the tracking results, the frame poses and counters,
the refPixelWasGood masks, the new keyframes' thisToParent and the depth maps."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from tests.device_cases import run_streams
from tests.util import assert_same

pytestmark = pytest.mark.gpu
LOOK_AWAY = np.array([0, 0.7071067811865476, 0, 0.7071067811865476, 0, 0, 0], np.float64)   # 90 deg about y: no point stays in view

@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_group_equals_single_calls_640x480(n):
    """25 frames, one keyframe change per stream, in a different step for every stream: groups mix update and create"""
    phases = [2 * s for s in range(n)]              # keyframe changes at steps 20, 18, 16, ...
    single = run_streams(640, 480, phases, 25, lambda k: False)
    group = run_streams(640, 480, phases, 25, lambda k: True)
    changes = [[k for k, step in enumerate(single, start=1) if step[s]["kf"]] for s in range(n)]
    assert all(len(c) == 1 for c in changes) and len({c[0] for c in changes}) == n
    assert not any(o["diverged"] for step in single for o in step)
    assert_same(group, single)


def test_group_equals_single_calls_1280x1024_n8():
    """at 1280x1024 a CTA of an 8-stream group stands in for up to 9 virtual CTAs of ~5 level-1 slots per warp each: more
    good-mask flags per thread than one 32-bit word holds"""
    phases = [15 + s % 5 for s in range(8)]         # keyframe changes at steps 5, 4, 3, 2, 1, 5, 4, 3
    single = run_streams(1280, 1024, phases, 5, lambda k: False)
    group = run_streams(1280, 1024, phases, 5, lambda k: True)
    assert all(sum(step[s]["kf"] for step in single) == 1 for s in range(8))
    assert_same(group, single)


def test_group_and_single_calls_alternated():
    """group and single calls on the same contexts: the barrier bookkeeping of either launch stays right after the other"""
    phases = [10, 12, 14]                            # keyframe changes at steps 10, 8, 6
    single = run_streams(640, 480, phases, 12, lambda k: False)
    mixed = run_streams(640, 480, phases, 12, lambda k: k % 2 == 0)
    assert_same(mixed, single)


def test_group_divergence_skips_only_that_streams_mapping():
    """one stream starts from a pose that puts every point out of view (SE3Tracker.cpp:324-329): it diverges, its map stays as it
    was, and the other streams track and map exactly as with single calls"""
    def look_away(k, streams):
        if k == 3:
            streams[1].last_pose = LOOK_AWAY.copy()
    phases = [0, 0, 0]
    single = run_streams(640, 480, phases, 3, lambda k: False, look_away)
    group = run_streams(640, 480, phases, 3, lambda k: True, look_away)
    assert [o["diverged"] for o in group[2]] == [False, True, False]
    assert group[2][1]["depth"] == group[1][1]["depth"]       # the diverged stream's map did not change
    assert_same(group, single)


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
