"""Wall time of Frame::setPermaRef (lsdgpu_frame_set_perma_ref, the call lsd_host.cpp's Frame::setPermaRef makes) on a keyframe with
ground-truth depth, at 640x480 and 1280x1024.  The call synchronises the context's stream twice; in SLAM mode it runs once per
finished keyframe on the mapping thread, holding the context's lock.  Prints one JSON line with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lsd_slam_b200 import abi, synth  # noqa: E402

REPS, WARMUP = 200, 20


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    out = {"card": card, "reps": REPS}
    for w, h in ((640, 480), (1280, 1024)):
        seq = synth.Sequence(w, h, seed=1234)
        img, depth = seq.render(0)
        ctx = abi.Context(w, h, seq.K, max_frames=4)
        trk = abi.SE3Tracker(ctx)
        ctx.upload(0, img)
        ctx.set_depth_gt(0, depth)
        trk.importFrame(0)
        for _ in range(WARMUP):
            n = trk.setPermaRef(0)
        ms = []
        for _ in range(REPS):
            ctx.synchronize()
            t0 = time.perf_counter()
            trk.setPermaRef(0)
            ms.append((time.perf_counter() - t0) * 1e3)
        ctx.close()
        ms = np.array(ms)
        out[f"{w}x{h}"] = {"points": n, "median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)),
                           "p90_ms": float(np.percentile(ms, 90))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
