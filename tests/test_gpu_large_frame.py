"""A frame large enough that every tracker thread owns many level-1 chunk slots.

k_track_persistent deals the level-1 chunks out as slots k = warp, warp + 16, ... of every CTA, and the last candidate's good flags
of a pass go to the context's level-1 plane, one byte per point, to be committed at the end of the launch.  A single-stream
launch and a group launch run the same virtual grid, so one stream stepped with lsdgpu_track_and_map_group (n = 1) and one
stepped with lsdgpu_track_and_map must agree bit for bit, also when a thread walks dozens of slots.

4112 is a width that is not a multiple of 32, above the 2048 columns where k_cloud_export switches to one row per tile and above
the 4096 where its dynamic shared memory exceeds 48 KB.  The height is chosen from the device's SM count."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream, GpuStreamGroup
from oracle.replay import run_with_replay
from tests.util import assert_step_ok, oracle_cloud, same_cloud

pytestmark = pytest.mark.gpu

W = 4112
MIN_SLOTS_PER_THREAD = 35   # level-1 chunk slots of every thread (640x480 gives one or two)
STEPS = 3

_cache = {}


def _setup():
    """the height whose level-1 interior gives every warp of a one-CTA-per-SM grid at least MIN_SLOTS_PER_THREAD slots (16 warps per
    CTA, at most 160 CTAs)"""
    if not _cache:
        import torch
        grid = min(torch.cuda.get_device_properties(0).multi_processor_count, 160)

        def per_warp(h):
            chunks = -(-(W // 2 - 2) * (h // 2 - 2) // 32)
            return (-(-chunks // grid)) // 16
        h = next(h for h in range(16, 16384, 16) if per_warp(h) >= MIN_SLOTS_PER_THREAD)
        seq = synth.Sequence(W, h, seed=1234)
        _cache.update(seq=seq, frames=[seq.render(k) for k in range(STEPS + 1)])
    return _cache["seq"], _cache["frames"]


def test_group_of_one_equals_single_call_bit_for_bit():
    """every step changes keyframe (kf_every=1): createKeyFrame leaves the tracked frame's refPixelWasGood in place, where the
    mapping of an update step would clear it, so the mask each tracking committed is compared"""
    seq, frames = _setup()
    logs = []
    for grouped in (False, True):
        ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=4)
        try:
            gs = GpuStream(ctx, mode=1, kf_every=1)
            gs.init_gt(0, *frames[0])
            group = GpuStreamGroup([gs])
            log = []
            for k in range(1, STEPS + 1):
                pose = group.step([k], images=[frames[k][0]])[0] if grouped else gs.step(k, frames[k][0])
                assert not gs.tracker.diverged and gs.tracker.trackingWasGood
                mask = ctx.download(k, abi.BUF_GOODMASK)
                assert (mask == 0).sum() > 1000 and (mask == 1).sum() > 1000, k        # a tracked mask, not the all-true default
                log.append({"pose": pose.tobytes(), "result": bytes(gs.tracker.last), "new_kf_qts": (group._qts[0] if grouped else gs._qts).tobytes(),
                            "mask": mask, "depth": gs.map.current().tobytes()})
            logs.append(log)
        finally:
            ctx.close()
    for k, (a, b) in enumerate(zip(*logs), start=1):
        n_diff = int((a["mask"] != b["mask"]).sum())
        assert n_diff == 0, f"step {k}: {n_diff} refPixelWasGood bytes differ"
        assert a["pose"] == b["pose"] and a["result"] == b["result"] and a["new_kf_qts"] == b["new_kf_qts"], k
        assert a["depth"] == b["depth"], k


def test_one_step_replayed_on_the_oracle():
    """a sanity check of the large frame against the reference: the pose within 1e-4 plus the reference's own summation noise,
    the depth map bit for bit, and the mask close to the oracle's own (the device's pose is not the oracle's to the last bit, so
    flags at a threshold may differ); the exact check of the flags is the group comparison above"""
    seq, frames = _setup()
    (r,) = run_with_replay(seq, frames, 2, kf_every=0, max_frames=4)
    assert_step_ok(r)
    assert r["counts_equal"]
    assert r["mask_mismatch"] <= 1e-3 * (seq.w // 2) * (seq.h // 2), r["mask_mismatch"]


def test_level0_cloud_matches_oracle():
    seq, frames = _setup()
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=2)
    try:
        ctx.upload(0, frames[0][0])
        ctx.set_depth_gt(0, frames[0][1])
        ctx.cloud_reserve(1)
        c2w = np.array([[0.1, -0.2, 0.05, 0.97, 0.3, -0.1, 0.2]], np.float32)
        for layout in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
            pts, counts = ctx.export_pointcloud([0], c2w, level=0, layout=layout)
            ref, ref_counts = oracle_cloud(ctx, [0], c2w, 0, None, layout)
            assert (counts == ref_counts).all()
            same_cloud(pts, ref)
            assert len(pts) > 100000
    finally:
        ctx.close()
