#!/usr/bin/env python
"""K independent streams on ONE GPU: lsdgpu_track_and_map_group against K single lsdgpu_track_and_map calls.

  python scripts/bench_streams.py --streams K [--steps 60 --warmup 5 --width 640 --height 480] [--no-parity]

K contexts (seeds 1234 + 1000 s, the seeds bench.py gives the ranks of a multi-GPU run), frames parked in HBM.  Two legs are
timed in the same run, step by step in alternation: one group call per step (the K trackings share one launch), and K single
calls per step.  Per step the L2 is flushed and the wall clock runs until every stream is synchronised.  Prints one JSON line:
aggregate frames/s and ms per step of each leg, and the tracking kernel's device time per launch.  Exits with 3 unless both
legs produced bit-identical poses and depth maps and the oracle replay check (oracle/replay.py, as in bench.py) passes on
every stream.  Uses the same stream, warm-up and clock sampling as bench.py (imported from it).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import KF_EVERY, METRIC, POSE_TOL, ClockSampler, nvml_index, pin_to_gpu_numa_node, render_frames  # noqa: E402


def multi_stream_run(args):
    """the two legs of --streams K on one GPU: per step, the group call and the K single calls, alternating which goes first"""
    import torch
    from lsd_slam_b200 import abi
    from lsd_slam_b200.stream import GpuStream, GpuStreamGroup

    if not torch.cuda.is_available():
        raise RuntimeError("bench.py needs a CUDA device (the product path has no CPU fallback)")
    torch.cuda.set_device(0)
    pinned_cores = pin_to_gpu_numa_node(0)
    w, h, n, K, W = args.width, args.height, args.streams, args.steps, args.warmup
    n_frames = W + K + 1
    rendered = [render_frames(w, h, 1234 + 1000 * s, n_frames) for s in range(n)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def make_leg():
        streams = []
        for seq, frames in rendered:
            ctx = abi.Context(w, h, seq.K, device=0, max_frames=8)
            ctx.stage_reserve(n_frames)
            for k in range(n_frames):
                ctx.stage_put(k, frames[k][0])
            gs = GpuStream(ctx, mode=1, kf_every=KF_EVERY)
            gs.init_gt(0, frames[0][0], frames[0][1])
            streams.append(gs)
        return streams

    legs = {"group": make_leg(), "single": make_leg()}
    group = GpuStreamGroup(legs["group"])

    def run_step(leg, k):
        if leg == "group":
            group.step([k] * n, stage_indices=[k] * n)
        else:
            for gs in legs["single"]:
                gs.step(k, stage_index=k)

    def sync_all():
        for gs in legs["group"] + legs["single"]:
            gs.ctx.synchronize()

    # warm-up: the first keyframe change of every leg runs on throwaway contexts (one-time kernel loading), then W steps
    warm = make_leg()
    wg = GpuStreamGroup(warm)
    for k in range(1, min(KF_EVERY, n_frames - 1) + 1):
        wg.step([k] * n, stage_indices=[k] * n)
        for gs in warm:
            gs.ctx.synchronize()
    for gs in warm:
        gs.ctx.close()
    for k in range(1, W + 1):
        for leg in ("group", "single"):
            run_step(leg, k)
    sync_all()
    for gs in legs["group"] + legs["single"]:
        gs.ctx.track_kernel_stats(reset=1)
    sampler = ClockSampler(nvml_index(0))
    sampler.start()
    step_ms = {"group": [], "single": []}
    for k in range(W + 1, W + 1 + K):
        order = ("group", "single") if k % 2 else ("single", "group")
        for leg in order:
            flush.fill_(k & 0xff)                                              # L2 flush between timed steps
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run_step(leg, k)
            for gs in legs[leg]:
                gs.ctx.synchronize()
            step_ms[leg].append(1e3 * (time.perf_counter() - t0))
    clocks = sampler.stop()
    out = {}
    for leg in ("group", "single"):
        kms = klaunch = 0
        for gs in legs[leg]:
            m, l, _ = gs.ctx.track_kernel_stats(reset=2)
            kms, klaunch = kms + m, klaunch + l
        sm = np.array(step_ms[leg])
        out[leg] = {"frames_per_s": n * K / (sm.sum() * 1e-3), "ms_per_step": float(sm.mean()), "p50_ms": float(np.median(sm)),
                    "p95_ms": float(np.percentile(sm, 95)), "track_kernel_launches": int(klaunch),
                    "track_kernel_us_per_launch": 1e3 * kms / max(klaunch, 1)}
    same = all(np.array_equal(np.array(a.poses), np.array(b.poses)) and a.map.current().tobytes() == b.map.current().tobytes()
               for a, b in zip(legs["group"], legs["single"]))
    for gs in legs["group"] + legs["single"]:
        gs.ctx.close()
    return rendered, out, same, clocks, pinned_cores


def multi_stream_main(args, metric):
    from oracle.replay import run_with_replay
    rendered, legs, same, clocks, pinned_cores = multi_stream_run(args)
    n_frames = args.warmup + args.steps + 1
    parity = []
    if not args.no_parity:
        for s, (seq, frames) in enumerate(rendered):
            sample = set(range(1, n_frames, 5)) | {k for k in range(1, n_frames) if k % KF_EVERY == 0}
            reps = run_with_replay(seq, frames, n_frames, kf_every=KF_EVERY, sample=sample, mode=1)
            excess = max(r["pose_rel"] - r["ref_noise_rel"] for r in reps)
            maps = all(r["map_ok"] for r in reps)
            parity.append({"stream": s, "frames": len(reps), "max_pose_rel": float(max(r["pose_rel"] for r in reps)),
                           "max_excess_over_reference_noise": float(excess), "maps_identical": bool(maps),
                           "ok": bool(excess <= POSE_TOL and maps)})
    K, n = args.steps, args.streams
    line = {"metric": metric.replace("frames/sec", f"aggregate frames/sec of {n} streams on one GPU"),
            "value": legs["group"]["frames_per_s"], "unit": "frames/s", "n_gpus": 1, "streams": n, "steps": K,
            "warmup": args.warmup, "ms_per_step": legs["group"]["ms_per_step"], "higher_is_better": True,
            "config": {"width": args.width, "height": args.height, "kf_every": KF_EVERY, "seeds": [1234 + 1000 * s for s in range(n)],
                       "input": "frames parked in HBM (prefetch ring)", "l2": "flushed between timed steps (256 MiB fill)",
                       "statistic": f"{K} timed steps per leg, legs alternating step by step; wall clock per step with every stream synchronised",
                       "semi_dense_fraction": [round(seq.density, 4) for seq, _ in rendered]},
            "group_call": legs["group"], "single_calls": legs["single"],
            "speedup_group_vs_single": legs["single"]["ms_per_step"] / legs["group"]["ms_per_step"],
            "legs_bit_identical": bool(same), "parity": parity, "clocks": clocks, "pinned_cores": pinned_cores}
    print(json.dumps(line))
    if not same or not all(p["ok"] for p in parity):
        sys.stderr.write(f"--streams {n}: legs bit-identical: {same}; parity: {[p['ok'] for p in parity]}\n")
        sys.exit(3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4, help="streams on the GPU, 2..8")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--no-parity", action="store_true", help="skip the oracle replay check (timing repeats only)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)
    if not 2 <= args.streams <= 8:
        raise SystemExit("--streams must be 2..8")
    metric = METRIC if (args.width, args.height) == (640, 480) else METRIC.replace("640x480", f"{args.width}x{args.height}")
    multi_stream_main(args, metric)


if __name__ == "__main__":
    main()
