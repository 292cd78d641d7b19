"""The map point-cloud export's CPU oracle (oracle/lsd_oracle_cloud.inc) against lsd_slam_viewer's own KeyFrameDisplay.cpp:
bit for bit against the digests recorded from the viewer (tests/golden/cloud_viewer.json, tests/golden/make_golden_cloud.py) for
both layouts and the counts, and directly against the viewer's compiled code where oracle/_ref/libviewer_ref.so exists.  Also
write_ply against the viewer's pc.ply, and the ctypes layout of lsdgpu_cloud_filter.  No GPU needed."""
import ctypes
import hashlib
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "cloud_viewer.json")))


def _sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def _case_id(c):
    return f"s{c['seed']}-L{c['level']}-{c['filter']}"


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=_case_id)
def test_restatement_matches_viewer_digests(case):
    from oracle import cloud
    import make_golden_cloud as mg
    pc, c2w, cam = mg.level_case(case["seed"], case["w"], case["h"], case["adversarial"], case["scale"], case["level"])
    vert, ply, total, shown = cloud.keyframe(pc, cam, c2w, GOLDEN["filters"][case["filter"]])
    assert (total, shown) == (case["total"], case["displayed"])
    assert _sha(vert.tobytes()) == case["vertex_sha256"]
    assert _sha(ply.tobytes()) == case["ply_sha256"]


def test_golden_covers_the_filter_branches():
    """every filter keeps some points and rejects others; the adversarial cases put NaN points into the output"""
    from oracle import cloud
    import make_golden_cloud as mg
    for c in GOLDEN["cases"]:
        assert 0 < c["displayed"] < c["total"], _case_id(c)
    c = next(c for c in GOLDEN["cases"] if c["adversarial"] and c["filter"] == "support1")
    pc, c2w, cam = mg.level_case(c["seed"], c["w"], c["h"], True, c["scale"], c["level"])
    _, ply, _, _ = cloud.keyframe(pc, cam, c2w, GOLDEN["filters"]["support1"])
    assert np.isnan(ply["x"]).any()
    assert (pc["idepth"][0, 1:-1] > 0).all() and (pc["idepth"][1:-1, 0] > 0).all()   # valid border rows and columns
    assert abs(float(np.sqrt((c2w[:4].astype(np.float64) ** 2).sum())) - c["scale"]) < 1e-5
    assert {c["scale"] for c in GOLDEN["cases"]} > {1.0} and {c["level"] for c in GOLDEN["cases"]} == {0, 1}


def test_write_ply_equals_viewer_file_without_stray_byte(tmp_path):
    from lsd_slam_b200 import abi
    from oracle import cloud
    import make_golden_cloud as mg
    pcs, c2ws, cam = mg.map_inputs()
    pts = np.concatenate([cloud.keyframe(p, cam, c, None)[1] for p, c in zip(pcs, c2ws)])
    path = tmp_path / "pc.ply"
    abi.write_ply(str(path), pts)
    data = path.read_bytes()
    assert len(data) == GOLDEN["map"]["pc_ply_bytes"]
    assert _sha(data) == GOLDEN["map"]["pc_ply_sha256_without_last_byte"]
    assert data.startswith(cloud.ply_header(len(pts)))


def _viewer():
    from oracle import cloud
    if not cloud.viewer_built() and not cloud.viewer_available():
        pytest.skip("the viewer's library (oracle/_ref/libviewer_ref.so) is not built here")
    return cloud


@pytest.mark.parametrize("seed,adversarial,scale", [(31, False, 1.0), (32, True, 3.0), (33, True, 0.25)])
def test_restatement_equals_viewer_code(seed, adversarial, scale):
    cloud = _viewer()
    pc, c2w, cam = cloud.make_case(seed, 96, 64, adversarial, scale)
    for f in ({}, {"minNearSupport": 1}, {"minNearSupport": 9}, {"scaledDepthVarTH": 0.05, "absDepthVarTH": 0.05}):
        a = cloud.keyframe(pc, cam, c2w, f, impl="oracle")
        b = cloud.keyframe(pc, cam, c2w, f, impl="viewer")
        assert a[2:] == b[2:]
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def test_viewer_map_ply_has_the_stray_byte():
    cloud = _viewer()
    import make_golden_cloud as mg
    pcs, c2ws, cam = mg.map_inputs()
    raw = cloud.viewer_map_ply(pcs, cam, c2ws)
    assert raw[-1:] == b"\xff" and _sha(raw[:-1]) == GOLDEN["map"]["pc_ply_sha256_without_last_byte"]


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_cloud_filter_matches_c_layout(tmp_path):
    from lsd_slam_b200 import abi
    fields = [n for n, _ in abi.CloudFilter._fields_]
    lines = ['#include <cstddef>', '#include <cstdio>', '#include "lsdgpu.h"', "int main() {",
             '    std::printf("sizeof %zu\\n", sizeof(lsdgpu_cloud_filter));',
             '    std::printf("PLY %d\\nVERTEX %d\\nERR %d\\n", (int)LSDGPU_CLOUD_PLY, (int)LSDGPU_CLOUD_VERTEX, LSDGPU_CLOUD_ERR_CAPACITY);']
    lines += [f'    std::printf("{f} %zu\\n", offsetof(lsdgpu_cloud_filter, {f}));' for f in fields]
    lines += ["    return 0;", "}"]
    src = tmp_path / "layout.cpp"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(abi.CloudFilter) == 16
    for f in fields:
        assert int(out[f]) == getattr(abi.CloudFilter, f).offset, f
    assert (int(out["PLY"]), int(out["VERTEX"]), int(out["ERR"])) == (abi.CLOUD_PLY, abi.CLOUD_VERTEX, abi.CLOUD_ERR_CAPACITY)
    assert abi.CLOUD_PLY_DTYPE.itemsize == abi.CLOUD_VERTEX_DTYPE.itemsize == 16


def test_sim3f_conversion_and_chain():
    from lsd_slam_b200.stream import IDENT_QTS, qts_to_sim3f, sim3_mul_qts
    q = np.array([0.1, -0.2, 0.3, 0.9])
    q /= np.linalg.norm(q)
    a = np.concatenate([q, [1.0, 2.0, 3.0], [1.5]])
    f7 = qts_to_sim3f(a)
    assert f7.dtype == np.float32 and np.allclose(f7[:4], q * 1.5) and np.allclose(f7[4:], [1, 2, 3])
    assert np.allclose(sim3_mul_qts(IDENT_QTS, a), a) and np.allclose(sim3_mul_qts(a, IDENT_QTS), a)
    b = sim3_mul_qts(a, a)
    assert abs(b[7] - 2.25) < 1e-12 and abs(np.linalg.norm(b[:4]) - 1) < 1e-12
