#!/usr/bin/env python
"""The resident map as one point cloud: lsdgpu_map_export_pointcloud against the viewer's own code.

  python scripts/bench_cloud.py [--sizes 640x480,1280x1024] [--keyframes 64,512] [--reps 5] [--level 0] [--json FILE]

Per size, a GT-initialised synthetic stream runs until it has a few real keyframes (kept resident); they are replicated into
further frame slots (lsdgpu_frame_download / lsdgpu_frame_upload_u8 / lsdgpu_frame_set_idepth) up to K keyframes with their own
camToWorld.  The context reserves K keyframes per launch, so an export is one kernel launch.  Per K:
  device time  CUDA events around the export kernel (lsdgpu_cloud_last_kernel_ms), L2 flushed before each run; algorithmic bytes
               = 12 B per interior pixel (idepth, idepthVar, image read once) + 16 B per kept point, over that time, against the
               H100 SXM data sheet's 3.35 TB/s
  end to end   wall clock of the whole call (descriptor upload, kernel, device-to-host copy of the points into a reused host array)
  device out   lsdgpu_map_export_pointcloud_device into a reused CUDA tensor (no reservation, one launch, no copy of the points):
               CUDA events around the call on the caller's stream, and the wall clock of the call (it waits for the point count);
               run alternately with the host export, in the same repetitions
  CPU          lsd_slam_viewer's KeyFrameDisplay::refreshPC + flushPC compiled unmodified (oracle/_ref/libviewer_ref.so), one
               thread as in the viewer, over the same keyframes' keyframeMsg.pointcloud; per keyframe, message packing excluded
Exits with 3 unless the GPU's points (PLY and vertex layouts, both arms) and counts are identical to the viewer's (NaN compared
as NaN).
Card name, power limit and SM clock are sampled in the same run (bench.py's sampler).  Prints one JSON line per size and K.
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

HBM_BYTES_PER_S = 3.35e12
N_REAL_KF = 4
KF_EVERY = 4


def make_map(w, h, K):
    """context + K resident keyframes: N_REAL_KF from a tracked stream, the rest copies of them with their own camToWorld"""
    from lsd_slam_b200 import abi, synth
    from lsd_slam_b200.stream import GpuStream, qts_to_sim3f
    seq = synth.Sequence(w, h, seed=1234)
    ctx = abi.Context(w, h, seq.K, max_frames=K + 2)
    gs = GpuStream(ctx, mode=1, kf_every=KF_EVERY, keep_keyframes=True)
    img, d = seq.render(0)
    gs.init_gt(0, img, d)
    k = 1
    while len(gs.keyframe_ids) < min(N_REAL_KF, K):
        gs.step(k, seq.render(k)[0])
        k += 1
    ids = list(gs.keyframe_ids)
    c2w = [qts_to_sim3f(q) for q in gs.keyframe_cam_to_world]
    for i in gs.prev_ids:
        ctx.release(i)
    rng = np.random.default_rng(7)
    planes = {}
    for j in range(len(ids), K):
        src = ids[j % len(ids)]
        if src not in planes:
            planes[src] = (np.clip(ctx.download(src, abi.BUF_IMAGE), 0, 255).astype(np.uint8),
                           ctx.download(src, abi.BUF_IDEPTH), ctx.download(src, abi.BUF_IDEPTH_VAR))
        gray, idepth, var = planes[src]
        fid = 100000 + j
        ctx.upload(fid, gray)
        ctx.set_idepth(fid, idepth, var)
        ids.append(fid)
        q = rng.standard_normal(4)
        c2w.append(np.concatenate([q / np.linalg.norm(q) * rng.uniform(0.5, 2.0), rng.uniform(-5, 5, 3)]).astype(np.float32))
    return ctx, ids, np.stack(c2w)


def same(gpu, ref) -> bool:
    g, r = np.ascontiguousarray(gpu).view(np.uint32).reshape(-1, 4), np.ascontiguousarray(ref).view(np.uint32).reshape(-1, 4)
    if g.shape != r.shape:
        return False
    gn, rn = np.isnan(g.view(np.float32)), np.isnan(r.view(np.float32))
    return bool((gn == rn).all() and (g[~gn] == r[~rn]).all())


def level_cam(ctx, level):
    """the level's fx, fy, cx, cy as Frame::initialize forms them (Frame.cpp:403-459) and keyframeMsg carries them"""
    fx, fy, cx0, cy0 = (np.float32(v) for v in (ctx.K[0, 0], ctx.K[1, 1], ctx.K[0, 2], ctx.K[1, 2]))
    cx, cy = cx0, cy0
    for lv in range(1, level + 1):
        fx, fy = np.float32(np.float64(fx) * 0.5), np.float32(np.float64(fy) * 0.5)
        cx, cy = np.float32((np.float64(cx0) + 0.5) / (1 << lv) - 0.5), np.float32((np.float64(cy0) + 0.5) / (1 << lv) - 0.5)
    return float(fx), float(fy), float(cx), float(cy)


def run(w, h, K, reps, level):
    import torch
    from lsd_slam_b200 import abi
    from oracle import cloud
    ctx, ids, c2w = make_map(w, h, K)
    ctx.cloud_reserve(K)
    wl, hl = w >> level, h >> level
    interior = (wl - 2) * (hl - 2)
    out = np.empty(K * interior, abi.CLOUD_PLY_DTYPE)
    out_dev = torch.empty((K * interior, 4), dtype=torch.float32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # larger than the H100's 50 MB L2
    ctx.export_pointcloud(ids, c2w, level=level, out=out)                  # warm-up: module load, page-in of out
    ctx.export_pointcloud(ids, c2w, level=level, out=out_dev)              # warm-up: the memory pool's first block
    dev_ms, e2e_ms, dout_ev_ms, dout_wall_ms = [], [], [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pts, counts = ctx.export_pointcloud(ids, c2w, level=level, out=out)
        e2e_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(ctx.cloud_kernel_ms())
        flush.zero_()
        torch.cuda.synchronize()
        e0.record()
        t0 = time.perf_counter()
        dpts, dcounts = ctx.export_pointcloud(ids, c2w, level=level, out=out_dev)
        dout_wall_ms.append((time.perf_counter() - t0) * 1e3)
        e1.record()
        e1.synchronize()
        dout_ev_ms.append(e0.elapsed_time(e1))
    kept = int(counts[:, 1].sum())
    dpts = dpts.cpu().numpy()
    vert, vcounts = ctx.export_pointcloud(ids, c2w, level=level, layout=abi.CLOUD_VERTEX)
    dvert, dvcounts = ctx.export_pointcloud(ids, c2w, level=level, layout=abi.CLOUD_VERTEX, out=out_dev)
    dvert = dvert.cpu().numpy()

    # the viewer's own code, one keyframe after the other (its message packing not timed)
    cam = level_cam(ctx, level)
    cpu_s, ref_ply, ref_vert, ref_counts = 0.0, [], [], []
    for i, kf in enumerate(ids):
        pc = ctx.pack_pointcloud(kf, level).reshape(hl, wl).view(cloud.INPUT_POINT_DENSE)
        t0 = time.perf_counter()
        v, p, total, shown = cloud.keyframe(pc, cam, c2w[i], None, impl="viewer")
        cpu_s += time.perf_counter() - t0
        ref_ply.append(p)
        ref_vert.append(v)
        ref_counts.append((total, shown))
    ok = (same(pts, np.concatenate(ref_ply)) and same(vert, np.concatenate(ref_vert))
          and np.array_equal(counts, np.array(ref_counts, np.int32)) and np.array_equal(vcounts, counts))
    ok_dev = (same(dpts, np.concatenate(ref_ply)) and same(dvert, np.concatenate(ref_vert))
              and np.array_equal(dcounts, counts) and np.array_equal(dvcounts, counts))
    ctx.close()
    algo_bytes = 12.0 * interior * K + 16.0 * kept
    dev = float(np.median(dev_ms))
    return {"width": w, "height": h, "level": level, "keyframes": K, "points": kept, "interior_pixels": interior * K,
            "device_ms": dev, "device_ms_all": [round(x, 4) for x in dev_ms], "algorithmic_bytes": algo_bytes,
            "device_GBps": algo_bytes / dev / 1e6, "hbm_fraction": algo_bytes / dev / 1e-3 / HBM_BYTES_PER_S,
            "e2e_ms": float(np.median(e2e_ms)), "e2e_ms_all": [round(x, 3) for x in e2e_ms],
            "device_out_event_ms": float(np.median(dout_ev_ms)), "device_out_event_ms_all": [round(x, 4) for x in dout_ev_ms],
            "device_out_wall_ms": float(np.median(dout_wall_ms)), "device_out_wall_ms_all": [round(x, 3) for x in dout_wall_ms],
            "cpu_viewer_ms": cpu_s * 1e3, "speedup_e2e_vs_viewer": cpu_s * 1e3 / float(np.median(e2e_ms)),
            "parity": bool(ok), "parity_device_out": bool(ok_dev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--keyframes", default="64,512")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--level", type=int, default=0)
    ap.add_argument("--json", default=None, help="also append the result lines to this file")
    args = ap.parse_args()
    import torch
    from oracle import cloud
    if not torch.cuda.is_available():
        raise RuntimeError("bench_cloud.py needs a CUDA device (the product path has no CPU fallback)")
    if not cloud.viewer_built():
        raise RuntimeError("oracle/_ref/libviewer_ref.so is not built (python -c 'from oracle import cloud; cloud.build()' where "
                           "the reference tree exists)")
    torch.cuda.set_device(0)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    results = []
    for size in args.sizes.split(","):
        w, h = (int(v) for v in size.split("x"))
        for K in (int(v) for v in args.keyframes.split(",")):
            r = run(w, h, K, args.reps, args.level)
            results.append(r)
            print(json.dumps(r), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks}), flush=True)
    if args.json:
        with open(args.json, "a") as f:
            for r in results:
                f.write(json.dumps(dict(r, clocks=clocks)) + "\n")
    if not all(r["parity"] and r["parity_device_out"] for r in results):
        print("PARITY FAILED: the GPU export differs from the viewer's code", file=sys.stderr)
        raise SystemExit(3)


if __name__ == "__main__":
    main()
