"""per-phase cycle counters of k_track_persistent (LSDGPU_TRACK_DEBUG=1)
   python scripts/dbg_track.py [width height [frames]]"""
import os, sys, numpy as np
sys.path.insert(0, os.getcwd())
os.environ["LSDGPU_TRACK_DEBUG"] = "1"
from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream
w, h = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (640, 480)
n = int(sys.argv[3]) if len(sys.argv) > 3 else 8
seq = synth.Sequence(w, h)
fr = [seq.render(k) for k in range(n)]
ctx = abi.Context(w, h, seq.K, max_frames=8)
gs = GpuStream(ctx, mode=1, kf_every=20)
gs.init_gt(0, fr[0][0], fr[0][1])
for k in range(1, n):
    gs.step(k, fr[k][0])
    print(list(gs.tracker.last.numCalcResidualCalls))
