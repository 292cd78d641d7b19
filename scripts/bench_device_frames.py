#!/usr/bin/env python
"""Frames from device memory: Frame construction from a CUDA tensor against host memory, and a stream fed from CUDA tensors.

  python scripts/bench_device_frames.py [--sizes 640x480,1280x1024] [--uploads 50] [--rounds 5] [--frames 200] [--json FILE]

Per size:
  construction  Frame::Frame + the image, gradient and maxGradients pyramids of one frame, from
                  device    a uint8 CUDA tensor with a row pitch 3 bytes wider than the frame (lsdgpu_frame_upload_device_u8)
                  pinned    page-locked host memory, copied from directly (lsdgpu_frame_upload_u8)
                  pageable  ordinary host memory, through the context's pinned staging copy (lsdgpu_frame_upload_u8)
                `uploads` back-to-back calls per arm and round, then a device synchronise: wall time per frame; the arms alternate
                over `rounds` rounds and the median round is reported.  The three arms must build identical frames.
  stream        a GT-initialised GpuStream of `frames` frames (the fused track-and-map call, a keyframe every 20 frames) fed
                through the prefetch ring from CUDA tensors (lsdgpu_stage_put_device, one tensor per frame, all resident
                before the run), against the same stream fed from host images: frames per second of each, and their poses must
                be identical.
Card name, power limit and SM clock are sampled in the same run (bench.py's sampler).  Prints one JSON line per size; exits
with 3 unless every parity check holds.
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

from bench import ClockSampler  # noqa: E402

PITCH_EXTRA = 3


def frame_bytes(ctx, fid):
    from lsd_slam_b200 import abi
    parts = [ctx.download(fid, what, lvl).tobytes() for lvl in range(abi.LEVELS) for what in (abi.BUF_IMAGE, abi.BUF_GRADIENTS)]
    return b"".join(parts) + ctx.download(fid, abi.BUF_MAXGRAD).tobytes()


def construction(w, h, uploads, rounds):
    import torch
    from lsd_slam_b200 import abi, synth
    seq = synth.Sequence(w, h, seed=1234)
    img = seq.render(3)[0]
    ctx = abi.Context(w, h, seq.K, max_frames=4)
    dev = torch.zeros((h, w + PITCH_EXTRA), dtype=torch.uint8, device="cuda")
    dev[:, :w] = torch.from_numpy(img).cuda()
    dev = dev[:, :w]
    pinned = torch.from_numpy(img).pin_memory().numpy()
    pageable = np.ascontiguousarray(img)
    arms = {"device": dev, "pinned": pinned, "pageable": pageable}
    built = {}
    for i, (name, src) in enumerate(arms.items()):          # warm-up, and the frames each arm builds
        ctx.upload(i + 1, src)
        built[name] = frame_bytes(ctx, i + 1)
    parity = built["device"] == built["pinned"] == built["pageable"]
    ms = {name: [] for name in arms}
    for _ in range(rounds):
        for name, src in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(uploads):
                ctx.upload(1, src)
            ctx.synchronize()
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3 / uploads)
    ctx.close()
    return {f"{name}_ms_per_frame": float(np.median(v)) for name, v in ms.items()} | \
        {f"{name}_ms_per_frame_all": [round(x, 4) for x in v] for name, v in ms.items()} | {"construction_parity": bool(parity)}


def stream_run(seq, frames, from_device):
    import torch
    from lsd_slam_b200 import abi
    from lsd_slam_b200.stream import GpuStream
    ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=8)
    gs = GpuStream(ctx, mode=1)
    gs.init_gt(0, frames[0][0], frames[0][1])
    ctx.stage_reserve(2)
    dev = [torch.from_numpy(f[0]).cuda() for f in frames] if from_device else None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(1, len(frames)):
        if from_device:
            ctx.stage_put(k % 2, dev[k])
            gs.step(k, stage_index=k % 2)
        else:
            gs.step(k, frames[k][0])
    ctx.synchronize()
    fps = (len(frames) - 1) / (time.perf_counter() - t0)
    poses = np.stack(gs.poses)
    ctx.close()
    return fps, poses


def run(w, h, uploads, rounds, n_frames):
    from lsd_slam_b200 import synth
    r = {"width": w, "height": h, "uploads": uploads, "rounds": rounds, "pitch_bytes": w + PITCH_EXTRA}
    r.update(construction(w, h, uploads, rounds))
    seq = synth.Sequence(w, h, seed=1234)
    frames = [seq.render(k) for k in range(n_frames)]
    stream_run(seq, frames[:5], True)                        # warm-up of both paths
    stream_run(seq, frames[:5], False)
    fps_host, poses_host = stream_run(seq, frames, False)
    fps_dev, poses_dev = stream_run(seq, frames, True)
    r.update({"frames": n_frames, "stream_fps_host_images": fps_host, "stream_fps_device_tensors": fps_dev,
              "stream_pose_parity": bool(poses_host.tobytes() == poses_dev.tobytes())})
    r["parity"] = r["construction_parity"] and r["stream_pose_parity"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--uploads", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--json", default=None, help="also append the result lines to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("bench_device_frames.py needs a CUDA device (the product path has no CPU fallback)")
    torch.cuda.set_device(0)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    results = []
    for size in args.sizes.split(","):
        w, h = (int(v) for v in size.split("x"))
        r = run(w, h, args.uploads, args.rounds, args.frames)
        results.append(r)
        print(json.dumps(r), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks}), flush=True)
    if args.json:
        with open(args.json, "a") as f:
            for r in results:
                f.write(json.dumps(dict(r, clocks=clocks)) + "\n")
    if not all(r["parity"] for r in results):
        print("PARITY FAILED: frames or poses from device memory differ from those from host memory", file=sys.stderr)
        raise SystemExit(3)


if __name__ == "__main__":
    main()
