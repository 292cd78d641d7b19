#!/usr/bin/env python
"""Depth from and to device memory: ground-truth seeding from a CUDA tensor against host memory, and the hypothesis download into a
CUDA tensor against host memory.

  python scripts/bench_device_depth.py [--sizes 640x480,1280x1024] [--calls 50] [--rounds 5] [--json FILE]

Per size:
  seeding   Frame::setDepthFromGroundTruth + DepthMap::initializeFromGTDepth (gtDepthInit after the frame is built), with the
            metric depth in
              device    a float32 CUDA tensor with a row pitch 4 floats wider than the frame (lsdgpu_frame_set_depth_gt_device)
              pinned    page-locked host memory (lsdgpu_frame_set_depth_gt)
              pageable  ordinary host memory (lsdgpu_frame_set_depth_gt)
  download  currentDepthMap in the 32-byte DepthMapPixelHypothesis layout into
              device    a uint8 CUDA tensor (lsdgpu_depth_download_device)
              host      a preallocated host array (lsdgpu_depth_download)
  `calls` back-to-back calls per arm and round, then a device synchronise: wall time per call.  The arms alternate over `rounds`
  rounds and the median round is reported.  The seeding arms must give identical idepth planes and hypotheses, the download arms
  identical bytes.
Card name, power limit and SM clock are sampled in the same run (bench.py's sampler).  Prints one JSON line per size; exits with 3
unless every parity check holds.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import ClockSampler  # noqa: E402

PITCH_EXTRA = 4


def timed(torch, ctx, fn, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    ctx.synchronize()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / calls


def alternate(torch, ctx, arms, calls, rounds):
    ms = {name: [] for name in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            ms[name].append(timed(torch, ctx, fn, calls))
    return ms


def run(w, h, calls, rounds):
    import torch
    from lsd_slam_b200 import abi, synth
    seq = synth.Sequence(w, h, seed=1234)
    img, depth = seq.render(0)
    depth = np.ascontiguousarray(depth, np.float32)
    ctx = abi.Context(w, h, seq.K, max_frames=4)
    dm = abi.DepthMap(ctx)
    ctx.upload(1, img)
    dev = torch.full((h, w + PITCH_EXTRA), float("nan"), dtype=torch.float32, device="cuda")
    dev[:, :w] = torch.from_numpy(depth).cuda()
    dev = dev[:, :w]
    pinned = torch.from_numpy(depth).pin_memory().numpy()
    seeds = {"device": dev, "pinned": pinned, "pageable": depth}

    def seed(src):
        ctx.set_depth_gt(1, src)
        dm.initializeFromGTDepth(1)

    seeded = {}
    for name, src in seeds.items():                          # warm-up, and what each arm leaves behind
        seed(src)
        seeded[name] = (ctx.download(1, abi.BUF_IDEPTH).tobytes(), ctx.download(1, abi.BUF_IDEPTH_VAR).tobytes(), dm.current().tobytes())
    seed_parity = seeded["device"] == seeded["pinned"] == seeded["pageable"]
    seed_ms = alternate(torch, ctx, {name: (lambda s=src: seed(s)) for name, src in seeds.items()}, calls, rounds)

    n = w * h
    out_dev = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    out_host = np.empty(n * 32, np.uint8)
    stream = torch.cuda.current_stream().cuda_stream
    L, p = ctx.L, ctx.ptr
    downloads = {
        "device": lambda: ctx._ck(L.lsdgpu_depth_download_device(p, out_dev.data_ptr(), out_dev.numel(), stream)),
        "host": lambda: ctx._ck(L.lsdgpu_depth_download(p, out_host.ctypes.data_as(C.POINTER(abi.Hyp)))),
    }
    for fn in downloads.values():
        fn()
    torch.cuda.synchronize()
    download_parity = out_dev.cpu().numpy().tobytes() == out_host.tobytes()
    download_ms = alternate(torch, ctx, downloads, calls, rounds)
    ctx.close()

    r = {"width": w, "height": h, "calls": calls, "rounds": rounds, "pitch_bytes": (w + PITCH_EXTRA) * 4}
    for prefix, ms in (("seed", seed_ms), ("download", download_ms)):
        for name, v in ms.items():
            r[f"{prefix}_{name}_ms_per_call"] = float(np.median(v))
            r[f"{prefix}_{name}_ms_per_call_all"] = [round(x, 4) for x in v]
    r.update({"seed_parity": bool(seed_parity), "download_parity": bool(download_parity)})
    r["parity"] = r["seed_parity"] and r["download_parity"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None, help="also append the result lines to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("bench_device_depth.py needs a CUDA device (the product path has no CPU fallback)")
    torch.cuda.set_device(0)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    results = []
    for size in args.sizes.split(","):
        w, h = (int(v) for v in size.split("x"))
        r = run(w, h, args.calls, args.rounds)
        results.append(r)
        print(json.dumps(r), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks}), flush=True)
    if args.json:
        with open(args.json, "a") as f:
            for r in results:
                f.write(json.dumps(dict(r, clocks=clocks)) + "\n")
    if not all(r["parity"] for r in results):
        print("PARITY FAILED: depth from or to device memory differs from the host path", file=sys.stderr)
        raise SystemExit(3)


if __name__ == "__main__":
    main()
