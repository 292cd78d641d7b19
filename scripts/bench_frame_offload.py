#!/usr/bin/env python
"""Offloaded frames: lsdgpu_frame_offload and activation from the host tier (the reference's minimized frames in host RAM).

  python scripts/bench_frame_offload.py [--sizes 640x480,1280x1024] [--calls 200] [--cloud-kfs 64] [--frames 200] [--json FILE]

Per size, on a mapped keyframe with reactivation data and a permaRef:
  offload, activate    device time of one call (CUDA events on the context's stream around it), median over --calls rounds after
                       20 warm-up rounds; activation from the host tier against activation from the device tier
  bus rates            host body bytes over the offload time (the kernel's writes into host memory) and over the activation's
                       extra time against the device tier (its reads), next to a plain pinned cudaMemcpyAsync H2D and D2H of the
                       same bytes (CUDA events, median of --calls copies)
  cloud export         lsdgpu_map_export_pointcloud at level 0 over --cloud-kfs keyframes (GT depth), all in the device tier,
                       then all in the host tier: device time of its kernels (median of 20) and identical points asserted;
                       between the two, the wall time per offload of those keyframes (host clock and device synchronise
                       around all of them), where every offload allocates fresh host memory because no body is freed
  stream fps           a --frames GT stream (keyframe every 20 frames, keyframes kept, max_active_keyframes=2 in 6 slots) with
                       max_device_records=0 against the same stream with every keyframe resident; identical poses asserted
Card name and power limit are read in the same run.  Prints one JSON line per size.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench import ClockSampler  # noqa: E402
from bench_frame_memory import KF_EVERY, _render_image, a256, run_stream  # noqa: E402


def body_bytes(w, h):
    """the host body of a keyframe with depth and reactivation data (csrc/records.cu recordParts)"""
    n0 = w * h
    return 5 * a256(n0 * 4) + a256(n0)


def copy_ms(torch, nbytes, calls):
    """median device time of a pinned H2D and D2H cudaMemcpyAsync of nbytes"""
    host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {}
    for name, dst, src in (("h2d", dev, host), ("d2h", host, dev)):
        t = []
        for i in range(20 + calls):
            b.record()
            dst.copy_(src, non_blocking=True)
            e.record()
            e.synchronize()
            if i >= 20:
                t.append(b.elapsed_time(e))
        out[name] = float(np.median(t))
    return out


def bench_size(w, h, calls, n_cloud, n_frames):
    import torch
    from lsd_slam_b200 import abi, synth
    from lsd_slam_b200.stream import GpuStream
    seq = synth.Sequence(w, h, seed=1234)
    with ProcessPoolExecutor(min(32, os.cpu_count() or 1)) as ex:       # the renderer is numpy on the CPU
        images = list(ex.map(_render_image, [(w, h, k) for k in range(n_frames)]))
    depth0 = seq.render(0)[1]

    # offload and activation from either tier, on a mapped keyframe
    ctx = abi.Context(w, h, seq.K, max_frames=16)
    gs = GpuStream(ctx, mode=1, kf_every=10, keep_keyframes=True)
    gs.init_gt(0, images[0], depth0)
    for k in range(1, 12):
        gs.step(k, images[k])
    n_perma = gs.tracker.setPermaRef(0)
    want = [ctx.download(0, abi.BUF_GRADIENTS, lvl).tobytes() for lvl in range(5)]

    def timed(slot, f):
        ctx.timer_begin(slot)
        f(0)
        ctx.timer_end(slot)
        return ctx.timer_ms(slot)

    t_off, t_act_host, t_act_dev = [], [], []
    for i in range(20 + calls):
        ctx.minimize(0)
        off = timed(0, ctx.offload)
        act_host = timed(1, ctx.activate)
        ctx.minimize(0)
        act_dev = timed(2, ctx.activate)
        if i >= 20:
            t_off.append(off)
            t_act_host.append(act_host)
            t_act_dev.append(act_dev)
    assert [ctx.download(0, abi.BUF_GRADIENTS, lvl).tobytes() for lvl in range(5)] == want
    ctx.minimize(0)
    ctx.offload(0)
    usage = ctx.memory_usage()
    ctx.close()
    body = body_bytes(w, h)
    assert usage.host_bytes == body, (usage, body)
    off_ms, act_host_ms, act_dev_ms = (float(np.median(t)) for t in (t_off, t_act_host, t_act_dev))
    copies = copy_ms(torch, body, calls)

    # the cloud export over n_cloud keyframes in either tier
    ctx = abi.Context(w, h, seq.K, max_frames=2)
    for k in range(n_cloud):
        ctx.upload(k, images[k % len(images)])
        ctx.set_depth_gt(k, seq.render(k % 8)[1])
        ctx.minimize(k)
    ids = list(range(n_cloud))
    c2w = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], np.float32), (n_cloud, 1))
    c2w[:, 4] = np.arange(n_cloud, dtype=np.float32) * 0.01
    ctx.cloud_reserve(n_cloud)

    def export():
        t, pts = [], None
        for i in range(25):
            pts, _ = ctx.export_pointcloud(ids, c2w, level=0)
            if i >= 5:
                t.append(ctx.cloud_kernel_ms())
        return float(np.median(t)), pts.tobytes()

    cloud_dev_ms, pts_dev = export()
    ctx.synchronize()
    t0 = time.perf_counter()
    for k in ids:                                        # every body stays live: each offload grows the host pool
        ctx.offload(k)
    ctx.synchronize()
    offload_fresh_ms = (time.perf_counter() - t0) * 1e3 / n_cloud
    assert ctx.memory_usage().n_host == n_cloud
    cloud_host_ms, pts_host = export()
    ctx.close()

    full = run_stream(abi, GpuStream, seq, images, depth0, max_frames=n_frames // KF_EVERY + 4)
    host = run_stream(abi, GpuStream, seq, images, depth0, max_frames=6, max_active_keyframes=2, max_device_records=0)
    return {
        "size": f"{w}x{h}", "perma_points": n_perma, "body_bytes": body, "residue_bytes": usage.device_bytes, "calls": calls,
        "offload_us_median": off_ms * 1e3, "activate_host_us_median": act_host_ms * 1e3, "activate_device_us_median": act_dev_ms * 1e3,
        "offload_write_gbps": body / (off_ms * 1e-3) / 1e9,
        "activate_read_gbps": body / ((act_host_ms - act_dev_ms) * 1e-3) / 1e9 if act_host_ms > act_dev_ms else None,
        "memcpy_h2d_us": copies["h2d"] * 1e3, "memcpy_d2h_us": copies["d2h"] * 1e3,
        "memcpy_h2d_gbps": body / (copies["h2d"] * 1e-3) / 1e9, "memcpy_d2h_gbps": body / (copies["d2h"] * 1e-3) / 1e9,
        "offload_fresh_wall_ms": offload_fresh_ms, "cloud_keyframes": n_cloud, "cloud_points": len(pts_dev) // 16,
        "cloud_kernel_ms_device_tier": cloud_dev_ms, "cloud_kernel_ms_host_tier": cloud_host_ms,
        "cloud_identical": pts_dev == pts_host,
        "stream_frames": n_frames, "stream_fps_resident": full["fps"], "stream_fps_host_records": host["fps"],
        "keyframes": host["keyframes"], "poses_identical": bool(np.array_equal(full["poses"], host["poses"])),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--cloud-kfs", type=int, default=64)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for s in a.sizes.split(","):
        w, h = (int(x) for x in s.split("x"))
        r = bench_size(w, h, a.calls, a.cloud_kfs, a.frames)
        r.update({"gpu": sampler.gpu_name, "power_limit_w": sampler.power_limit_w, "max_sm_mhz": sampler.max_mhz})
        print(json.dumps(r), flush=True)
        rows.append(r)
    sampler.stop()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
