"""Records lsd_slam_viewer's own point-cloud outputs into tests/golden/cloud_viewer.json.

Runs the viewer's KeyFrameDisplay / KeyFrameGraphDisplay compiled unmodified (oracle/_ref/libviewer_ref.so, oracle/cloud.py) on the
seeded keyframes of oracle.cloud.make_case and stores, per case, the generator parameters and SHA-256 digests of refreshPC's vertex
buffer and flushPC's points with totalPoints / displayedPoints; and, for one small map, the digest of the pc.ply the viewer writes
(KeyFrameGraphDisplay.cpp:60-92) without its stray last byte.  Needs the reference tree; run from the repository root:

    python tests/golden/make_golden_cloud.py
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "cloud_viewer.json")

FILTERS = {
    "default": {},
    "support1": {"minNearSupport": 1},
    "support9": {"minNearSupport": 9},
    "tight": {"scaledDepthVarTH": 0.01, "absDepthVarTH": 0.02, "minNearSupport": 5},
    "loose": {"scaledDepthVarTH": 100.0, "absDepthVarTH": 100.0, "minNearSupport": 5},
}
# (seed, level-0 width, height, adversarial, camToWorld scale)
CASES = [(11, 64, 48, False, 1.0), (12, 64, 48, True, 1.0), (13, 80, 64, False, 2.5), (14, 80, 64, True, 0.4)]
MAP = {"seeds": [21, 22, 23], "w": 80, "h": 64, "adversarial": [False, True, False], "scale": 1.7}


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def level_case(seed, w, h, adversarial, scale, level):
    """the case at pyramid level 0 or 1: half size, and the level's camera as Frame::initialize forms it (Frame.cpp:403-459)"""
    from oracle import cloud
    pc, c2w, cam = cloud.make_case(seed, w >> level, h >> level, adversarial, scale)
    if level:
        fx, fy, cx, cy = cloud.make_case(seed, w, h, adversarial, scale)[2]
        cam = tuple(float(v) for v in np.float32([fx * 0.5, fy * 0.5, (cx + 0.5) / 2 - 0.5, (cy + 0.5) / 2 - 0.5]))
    return pc, c2w, cam


def map_inputs():
    from oracle import cloud
    pcs, c2ws = [], []
    for s, adv in zip(MAP["seeds"], MAP["adversarial"]):
        pc, c2w, cam = cloud.make_case(s, MAP["w"], MAP["h"], adv, MAP["scale"])
        pcs.append(pc)
        c2ws.append(c2w)
    return np.stack(pcs), np.stack(c2ws), cam


def main():
    from oracle import cloud
    cloud.build()
    if not cloud.viewer_built():
        raise SystemExit("the viewer library is not built (needs the reference tree)")
    rec = {"filters": FILTERS, "cases": []}
    for seed, w, h, adv, scale in CASES:
        for level in (0, 1):
            pc, c2w, cam = level_case(seed, w, h, adv, scale, level)
            for name, f in FILTERS.items():
                vert, ply, total, shown = cloud.keyframe(pc, cam, c2w, f, impl="viewer")
                rec["cases"].append({"seed": seed, "w": w, "h": h, "adversarial": adv, "scale": scale, "level": level, "filter": name,
                                     "total": total, "displayed": shown, "vertex_sha256": sha(vert.tobytes()),
                                     "ply_sha256": sha(ply.tobytes())})
    pcs, c2ws, cam = map_inputs()
    raw = cloud.viewer_map_ply(pcs, cam, c2ws)
    assert raw[-1:] == b"\xff", "the viewer's copy loop appends one 0xFF byte (KeyFrameGraphDisplay.cpp:84-85)"
    rec["map"] = dict(MAP, pc_ply_bytes=len(raw) - 1, pc_ply_sha256_without_last_byte=sha(raw[:-1]))
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1)
    print(f"wrote {OUT}: {len(rec['cases'])} keyframe cases + one map")


if __name__ == "__main__":
    main()
