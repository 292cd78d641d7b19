#!/usr/bin/env python
"""Colour camera frames: the gray conversion (cv::cvtColor) fused into the frame construction and the prefetch ring, against
converting first and feeding gray.

  python scripts/bench_colour_input.py [--sizes 640x480,1280x1024] [--uploads 50] [--rounds 5] [--frames 200] [--json FILE]

Per size, an rgb8 camera behind the pass-through undistorter:
  host      cvt_gray   cv2.cvtColor(rgb, COLOR_RGB2GRAY) on the host + lsdgpu_frame_upload_u8 of the gray image (pageable memory);
                       "not measured" when cv2 cannot be imported
            fused      lsdgpu_frame_upload_distorted_u8 of the rgb image (3x the bytes over the bus, converted on the device)
  device    rgb        lsdgpu_frame_upload_distorted_device_u8 of a (h, w, 3) uint8 CUDA tensor
            gray       lsdgpu_frame_upload_device_u8 of a (h, w) uint8 CUDA tensor holding the converted image (for comparison)
            `uploads` back-to-back calls per arm and round, then a device synchronise: wall time per frame; the arms alternate over
            `rounds` rounds and the median round is reported.  Every arm must build the same frame.
  stream    a GT-initialised GpuStream of `frames` frames (the fused track-and-map call, a keyframe every 20 frames) fed through
            the prefetch ring from CUDA tensors: rgb tensors through lsdgpu_stage_put_raw_device against their converted gray
            images through lsdgpu_stage_put_device.  Frames per second of each; their poses must be identical.
Card name, power limit and SM clock are sampled in the same run (bench.py's sampler).  Prints one JSON line per size; exits with
3 unless every parity check holds.
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


def rgb_of(gray, seed):
    """an rgb image whose channels scatter around `gray`"""
    rng = np.random.default_rng(seed)
    g = gray.astype(np.int32)
    return np.stack([np.clip(g + rng.integers(-40, 41, g.shape), 0, 255) for _ in range(3)], -1).astype(np.uint8)


def to_gray(rgb):
    """COLOR_RGB2GRAY of OpenCV 4.13 in numpy (the same formula as the device), for the gray arms' inputs"""
    c = rgb.astype(np.int32)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def frame_bytes(ctx, fid):
    from lsd_slam_b200 import abi
    parts = [ctx.download(fid, what, lvl).tobytes() for lvl in range(abi.LEVELS) for what in (abi.BUF_IMAGE, abi.BUF_GRADIENTS)]
    return b"".join(parts) + ctx.download(fid, abi.BUF_MAXGRAD).tobytes()


def contexts(seq, max_frames=4):
    """a gray context and an rgb8 one, both behind the pass-through undistorter"""
    from lsd_slam_b200 import abi
    out = []
    for enc in ("mono8", "rgb8"):
        ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=max_frames)
        abi.UndistorterPTAM([0.5, 0.7, 0.5, 0.5, 0.0], (seq.w, seq.h), "crop", (seq.w, seq.h)).install(ctx)
        ctx.set_input_format(enc)
        out.append(ctx)
    return out


def construction(w, h, uploads, rounds):
    import torch
    from lsd_slam_b200 import synth
    try:
        import cv2
    except ImportError:
        cv2 = None
    seq = synth.Sequence(w, h, seed=1234)
    rgb = rgb_of(seq.render(3)[0], 5)
    gray_ctx, rgb_ctx = contexts(seq)
    d_rgb = torch.from_numpy(rgb).cuda()
    d_gray = torch.from_numpy(to_gray(rgb)).cuda()
    arms = {"host_fused": lambda: rgb_ctx.upload_distorted(1, rgb),
            "device_rgb": lambda: rgb_ctx.upload_distorted(1, d_rgb),
            "device_gray": lambda: gray_ctx.upload(1, d_gray)}
    if cv2 is not None:
        arms["host_cvt_gray"] = lambda: gray_ctx.upload(1, cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))
    built = set()
    for name, f in arms.items():                              # warm-up, and the frame each arm builds
        f()
        built.add(frame_bytes(gray_ctx if name in ("device_gray", "host_cvt_gray") else rgb_ctx, 1))
    ms = {name: [] for name in arms}
    for _ in range(rounds):
        for name, f in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(uploads):
                f()
            gray_ctx.synchronize()
            rgb_ctx.synchronize()
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3 / uploads)
    gray_ctx.close()
    rgb_ctx.close()
    r = {f"{name}_ms_per_frame": float(np.median(v)) for name, v in ms.items()}
    r |= {f"{name}_ms_per_frame_all": [round(x, 4) for x in v] for name, v in ms.items()}
    if cv2 is None:
        r["host_cvt_gray_ms_per_frame"] = "not measured (cv2 missing)"
    r["opencv"] = cv2.__version__ if cv2 is not None else None
    r["construction_parity"] = len(built) == 1
    return r


def stream_run(seq, frames, colour):
    import torch
    from lsd_slam_b200.stream import GpuStream
    gray_ctx, rgb_ctx = contexts(seq, max_frames=8)
    ctx = rgb_ctx if colour else gray_ctx
    (gray_ctx if colour else rgb_ctx).close()
    gs = GpuStream(ctx, mode=1)
    gs.init_gt(0, to_gray(frames[0][0]), frames[0][1])
    ctx.stage_reserve(2)
    dev = [torch.from_numpy(f[0] if colour else to_gray(f[0])).cuda() for f in frames]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(1, len(frames)):
        if colour:
            ctx.stage_put_raw(k % 2, dev[k])
        else:
            ctx.stage_put(k % 2, dev[k])
        gs.step(k, stage_index=k % 2)
    ctx.synchronize()
    fps = (len(frames) - 1) / (time.perf_counter() - t0)
    poses = np.stack(gs.poses)
    ctx.close()
    return fps, poses


def run(w, h, uploads, rounds, n_frames):
    from lsd_slam_b200 import synth
    r = {"width": w, "height": h, "uploads": uploads, "rounds": rounds}
    r.update(construction(w, h, uploads, rounds))
    seq = synth.Sequence(w, h, seed=1234)
    frames = [(rgb_of(img, k), depth) for k, (img, depth) in enumerate(seq.render(k) for k in range(n_frames))]
    stream_run(seq, frames[:5], True)                        # warm-up of both paths
    stream_run(seq, frames[:5], False)
    fps_gray, poses_gray = stream_run(seq, frames, False)
    fps_rgb, poses_rgb = stream_run(seq, frames, True)
    r.update({"frames": n_frames, "stream_fps_gray_stage_put_device": fps_gray, "stream_fps_rgb_stage_put_raw_device": fps_rgb,
              "stream_pose_parity": bool(poses_gray.tobytes() == poses_rgb.tobytes())})
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
        raise RuntimeError("bench_colour_input.py needs a CUDA device (the product path has no CPU fallback)")
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
        print("PARITY FAILED: frames or poses fed colour differ from those fed the converted gray images", file=sys.stderr)
        raise SystemExit(3)


if __name__ == "__main__":
    main()
