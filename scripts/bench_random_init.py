#!/usr/bin/env python
"""DepthMap::initializeRandomly (DepthMap.cpp:883-916): the device call against the path the C++ adapter used to take.

  python scripts/bench_random_init.py [--sizes 640x480,1280x1024] [--calls 100] [--json FILE]

Per size, on one synthetic image (rand() state type 3, a fresh seed per call):
  device       lsdgpu_depth_init_random: device time (CUDA events on the context's stream around the call: the three draw kernels,
               setDepth and the copy of the result) and wall time of the Python call, the state's round trip included
  host path    the reference's own initializeRandomly (oracle/_ref/liblsd_ref.so; the oracle's -O3 build where that is not
               built) -- its rand() loop and its Frame::setDepth -- plus the upload of the w*h hypotheses through
               lsdgpu_depth_set_hypotheses (with setDepth on the device), wall time each
Medians over --calls calls after 10 warm-up calls.  Card name, power limit and the SM clock are read in the same run.  Prints one
JSON line per size.
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

WARMUP = 10


def bench_size(w, h, calls):
    from lsd_slam_b200 import abi, synth
    from oracle import pyoracle as po
    from oracle import ref_build
    ref = "ref" if ref_build.built() else True
    seq = synth.Sequence(w, h, seed=1234)
    img = seq.render(0)[0]
    ctx = abi.Context(w, h, seq.K, max_frames=4)
    gdm = abi.DepthMap(ctx)
    ctx.upload(0, img)

    dev_ms, wall_ms = [], []
    for i in range(WARMUP + calls):
        st = abi.RandState.from_seed(1000 + i)
        ctx.synchronize()
        t0 = time.perf_counter()
        ctx.timer_begin(0)
        gdm.initializeRandomly(0, st)
        ctx.timer_end(0)
        t1 = time.perf_counter()
        if i >= WARMUP:
            dev_ms.append(ctx.timer_ms(0))
            wall_ms.append((t1 - t0) * 1e3)
    draws = gdm.last_draws

    po.set_globals(fast=ref)
    libc = C.CDLL(None)
    odm = po.DepthMap(w, h, seq.K, fast=ref)
    of = po.Frame(0, img, seq.K, fast=ref)
    loop_ms, upload_ms = [], []
    for i in range(WARMUP + calls):
        libc.srand(1000 + i)
        t0 = time.perf_counter()
        odm.initializeRandomly(of)
        t1 = time.perf_counter()
        hyp = odm.current()
        ctx.synchronize()
        t2 = time.perf_counter()
        gdm.setHypotheses(0, hyp, reactivated=False, do_set_depth=True)
        ctx.synchronize()
        t3 = time.perf_counter()
        if i >= WARMUP:
            loop_ms.append((t1 - t0) * 1e3)
            upload_ms.append((t3 - t2) * 1e3)
    libc.srand(1)
    ctx.close()
    med = lambda v: float(np.median(v))
    return {"size": f"{w}x{h}", "draws": int(draws), "calls": calls,
            "device_call_ms": med(dev_ms), "device_call_wall_ms": med(wall_ms),
            "host_loop_ms": med(loop_ms), "host_upload_ms": med(upload_ms), "host_path_ms": med(np.add(loop_ms, upload_ms)),
            "host_loop_build": "liblsd_ref.so" if ref == "ref" else "liblsd_oracle_fast.so",
            "hypothesis_bytes_uploaded": w * h * 32}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="640x480,1280x1024")
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for s in a.sizes.split(","):
        w, h = (int(x) for x in s.split("x"))
        r = bench_size(w, h, a.calls)
        r.update({"gpu": sampler.gpu_name, "power_limit_w": sampler.power_limit_w, "max_sm_mhz": sampler.max_mhz})
        rows.append(r)
    clocks = sampler.stop()
    for r in rows:
        r["sm_mhz_median"] = clocks.get("sm_mhz")
        print(json.dumps(r), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
