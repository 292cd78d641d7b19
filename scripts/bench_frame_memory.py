#!/usr/bin/env python
"""Minimized frames: lsdgpu_frame_minimize / lsdgpu_frame_activate (Frame::minimizeInMemory, FrameMemory::activateFrame).

  python scripts/bench_frame_memory.py [--sizes 640x480,1280x1024] [--calls 200] [--frames 200] [--json FILE]

Per size:
  minimize / activate  device time of one call (CUDA events on the context's stream around it), median over --calls round trips
                       of a mapped keyframe (reactivation data, permaRef) after 20 warm-up round trips
  bytes                a frame slot and a minimized record from the layout (each buffer 256-byte aligned), and measured as
                       cudaMemGetInfo deltas: two contexts that differ by 8 slots, and 8 records of minimized keyframes
  stream fps           a 200-frame GT stream (keyframe every 20 frames, keyframes kept) in a context with enough slots, and
                       with max_active_keyframes=2 in a context of 6 slots; wall clock of the frames after the first 10
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

from bench import ClockSampler  # noqa: E402

KF_EVERY = 20


def a256(n):
    return (n + 255) // 256 * 256


def slot_bytes(w, h):
    """the arena's per-slot buffers (csrc/context.cu carveArena)"""
    n0 = w * h
    b = sum(a256((n0 >> (2 * l)) * s) for l in range(5) for s in (4, 16, 4, 4))
    b += a256(n0 * 4) + a256(n0 // 4) + a256(64) + a256((n0 >> 8) * 16) + a256((n0 >> 8) * 4) + 2 * a256(n0 * 4) + a256(n0)
    return b


def record_bytes(w, h, n_perma):
    """a minimized keyframe with depth, reactivation data and a permaRef (csrc/records.cu recordParts)"""
    n0 = w * h
    return a256(24) + 3 * a256(n0 * 4) + 2 * a256(n0 * 4) + a256(n0) + a256(n_perma * 16) + a256(n_perma * 4)


def _render_image(args):
    from lsd_slam_b200 import synth
    w, h, k = args
    return synth.Sequence(w, h, seed=1234).render(k)[0]


def run_stream(abi, GpuStream, seq, images, depth0, max_frames, **kw):
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=max_frames)
    gs = GpuStream(ctx, mode=1, kf_every=KF_EVERY, keep_keyframes=True, **kw)
    gs.init_gt(0, images[0], depth0)
    for k in range(1, 11):
        gs.step(k, images[k])
    ctx.synchronize()
    t0 = time.perf_counter()
    for k in range(11, len(images)):
        gs.step(k, images[k])
    ctx.synchronize()
    dt = time.perf_counter() - t0
    out = {"fps": (len(images) - 11) / dt, "keyframes": len(gs.keyframe_ids), "max_frames": max_frames,
           "poses": np.array(gs.poses)}
    ctx.close()
    return out


def bench_size(w, h, calls, n_frames):
    import torch
    from lsd_slam_b200 import abi, synth
    from lsd_slam_b200.stream import GpuStream
    seq = synth.Sequence(w, h, seed=1234)
    with ProcessPoolExecutor(min(32, os.cpu_count() or 1)) as ex:       # the renderer is numpy on the CPU
        images = list(ex.map(_render_image, [(w, h, k) for k in range(n_frames)]))
    depth0 = seq.render(0)[1]

    # device time of minimize / activate on a mapped keyframe
    ctx = abi.Context(w, h, seq.K, max_frames=16)
    gs = GpuStream(ctx, mode=1, kf_every=10, keep_keyframes=True)
    gs.init_gt(0, images[0], depth0)
    for k in range(1, 90):
        gs.step(k, images[k])
    n_perma = gs.tracker.setPermaRef(0)
    t_min, t_act = [], []
    for i in range(20 + calls):
        ctx.timer_begin(0)
        ctx.minimize(0)
        ctx.timer_end(0)
        m = ctx.timer_ms(0)
        ctx.timer_begin(1)
        ctx.activate(0)
        ctx.timer_end(1)
        a = ctx.timer_ms(1)
        if i >= 20:
            t_min.append(m)
            t_act.append(a)
    # record bytes measured: minimize the 8 finished keyframes 0..70
    ctx.synchronize()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(0, 80, 10):
        ctx.minimize(k)
    ctx.synchronize()
    rec_meas = (free0 - torch.cuda.mem_get_info()[0]) / 8
    ctx.close()

    # slot bytes measured: two contexts that differ by 8 slots
    torch.cuda.synchronize()
    f0 = torch.cuda.mem_get_info()[0]
    c1 = abi.Context(w, h, seq.K, max_frames=8)
    f1 = torch.cuda.mem_get_info()[0]
    c1.close()
    c2 = abi.Context(w, h, seq.K, max_frames=16)
    f2 = torch.cuda.mem_get_info()[0]
    c2.close()
    slot_meas = ((f0 - f2) - (f0 - f1)) / 8

    full = run_stream(abi, GpuStream, seq, images, depth0, max_frames=n_frames // KF_EVERY + 4)
    mini = run_stream(abi, GpuStream, seq, images, depth0, max_frames=6, max_active_keyframes=2)
    return {
        "size": f"{w}x{h}",
        "minimize_us_median": float(np.median(t_min) * 1e3), "activate_us_median": float(np.median(t_act) * 1e3), "calls": calls,
        "slot_bytes_layout": slot_bytes(w, h), "slot_bytes_measured": slot_meas,
        "record_bytes_layout": record_bytes(w, h, n_perma), "record_bytes_measured": rec_meas, "perma_points": n_perma,
        "stream_frames": n_frames,
        "stream_fps_resident": full["fps"], "resident_max_frames": full["max_frames"],
        "stream_fps_minimized": mini["fps"], "minimized_max_frames": mini["max_frames"], "keyframes": mini["keyframes"],
        "poses_identical": bool(np.array_equal(full["poses"], mini["poses"])),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for s in a.sizes.split(","):
        w, h = (int(x) for x in s.split("x"))
        r = bench_size(w, h, a.calls, a.frames)
        r.update({"gpu": sampler.gpu_name, "power_limit_w": sampler.power_limit_w, "max_sm_mhz": sampler.max_mhz})
        print(json.dumps(r), flush=True)
        rows.append(r)
    sampler.stop()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
