"""lsdgpu_map_export_pointcloud: the viewer's filtered point cloud of many resident keyframes in one call must equal the CPU
oracle (oracle/lsd_oracle_cloud.inc, pinned to lsd_slam_viewer's KeyFrameDisplay.cpp) byte for byte, fed with the same keyframes'
keyframeMsg.pointcloud (lsdgpu_keyframe_pack_pointcloud).  NaN values compare as NaN: their payloads may differ between the CPU
and the GPU."""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import GpuStream

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "cloud_viewer.json")))
FILTERS = [None, {"minNearSupport": 1}, {"minNearSupport": 9}, {"scaledDepthVarTH": 0.01, "absDepthVarTH": 0.02},
           {"scaledDepthVarTH": 100.0, "absDepthVarTH": 100.0}]


def _level_cam(ctx, level):
    """Frame::fx(level) etc. as ROSOutput3DWrapper.cpp:85-88 puts them into the message (Frame.cpp:403-459)"""
    fx, fy, cx, cy = np.float32(ctx.K[0, 0]), np.float32(ctx.K[1, 1]), np.float32(ctx.K[0, 2]), np.float32(ctx.K[1, 2])
    cx0, cy0 = cx, cy
    for lv in range(1, level + 1):
        fx, fy = np.float32(np.float64(fx) * 0.5), np.float32(np.float64(fy) * 0.5)
        cx = np.float32((np.float64(cx0) + 0.5) / (1 << lv) - 0.5)
        cy = np.float32((np.float64(cy0) + 0.5) / (1 << lv) - 0.5)
    return float(fx), float(fy), float(cx), float(cy)


def _oracle(ctx, kf_ids, c2w, level, filt, layout):
    from oracle import cloud
    cam = _level_cam(ctx, level)
    outs, counts = [], []
    for i, kf in enumerate(kf_ids):
        pc = ctx.pack_pointcloud(kf, level).reshape(ctx.h >> level, ctx.w >> level)
        vert, ply, total, shown = cloud.keyframe(pc.view(cloud.INPUT_POINT_DENSE), cam, c2w[i], filt)
        outs.append(vert if layout == abi.CLOUD_VERTEX else ply)
        counts.append((total, shown))
    return np.concatenate(outs).view(np.uint32).reshape(-1, 4), np.array(counts, np.int32).reshape(-1, 2)


def _same(gpu, ref):
    """byte-identical, except that NaN equals NaN"""
    g, r = np.ascontiguousarray(gpu).view(np.uint32).reshape(-1, 4), np.asarray(ref).reshape(-1, 4)
    assert g.shape == r.shape
    gn, rn = np.isnan(g.view(np.float32)), np.isnan(r.view(np.float32))
    assert (gn == rn).all()
    assert (g[~gn] == r[~rn]).all()
    return int(gn.sum())


_stream_cache = {}


def _stream(w, h, n_frames=30, kf_every=8):
    """a GT-initialised synthetic stream with its keyframes kept resident (>= 3 keyframe changes)"""
    key = (w, h)
    if key not in _stream_cache:
        seq = synth.Sequence(w, h, seed=4321)
        ctx = abi.Context(w, h, seq.K, max_frames=16)
        gs = GpuStream(ctx, mode=1, kf_every=kf_every, keep_keyframes=True)
        img, d = seq.render(0)
        gs.init_gt(0, img, d)
        for k in range(1, n_frames):
            gs.step(k, seq.render(k)[0])
        assert len(gs.keyframe_ids) >= 3
        ctx.cloud_reserve(16)
        _stream_cache[key] = gs
    return _stream_cache[key]


@pytest.mark.parametrize("w,h", [(320, 240), (640, 480)])
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("layout", [abi.CLOUD_PLY, abi.CLOUD_VERTEX])
def test_stream_keyframes_match_oracle(w, h, level, layout):
    gs = _stream(w, h)
    ctx, ids, c2w = gs.ctx, gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    assert not np.allclose(c2w[-1], c2w[0])
    for filt in FILTERS:
        pts, counts = ctx.export_pointcloud(ids, c2w, level=level, filter=filt, layout=layout)
        ref, ref_counts = _oracle(ctx, ids, c2w, level, filt, layout)
        assert (counts == ref_counts).all(), filt
        _same(pts, ref)
        if filt is None:
            assert len(pts) > 1000


def test_adversarial_planes_match_oracle():
    from oracle import cloud
    w, h = 320, 240
    K = synth.pinhole_K(w, h)
    ctx = abi.Context(w, h, K, max_frames=6)
    ctx.cloud_reserve(3)
    ids, c2ws = [], []
    for i, (adv, scale) in enumerate([(True, 1.0), (True, 2.5), (False, 0.5), (True, 0.8)]):
        pc, c2w, _ = cloud.make_case(50 + i, w, h, adv, scale)
        ctx.upload(i, np.ascontiguousarray(pc["color"][..., 0]))
        ctx.set_idepth(i, np.ascontiguousarray(pc["idepth"]), np.ascontiguousarray(pc["idepth_var"]))
        ids.append(i)
        c2ws.append(c2w)
    c2ws = np.stack(c2ws)
    n_nan = 0
    for level in (0, 1):
        for layout in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
            for filt in FILTERS:
                pts, counts = ctx.export_pointcloud(ids, c2ws, level=level, filter=filt, layout=layout)
                ref, ref_counts = _oracle(ctx, ids, c2ws, level, filt, layout)
                assert (counts == ref_counts).all()
                n_nan += _same(pts, ref)
    assert n_nan > 0
    ctx.close()


def test_golden_fixture_matches_viewer_digests():
    """level-0 cases of tests/golden/cloud_viewer.json loaded into a context: the export's bytes hash to the viewer's digests
    (NaN values replaced by the oracle's bits at the same places, where both are NaN)"""
    from oracle import cloud
    import make_golden_cloud as mg
    done = 0
    for c in GOLDEN["cases"]:
        if c["level"] != 0:
            continue
        pc, c2w, cam = mg.level_case(c["seed"], c["w"], c["h"], c["adversarial"], c["scale"], 0)
        K = np.array([[cam[0], 0, cam[2]], [0, cam[1], cam[3]], [0, 0, 1]], np.float32)
        ctx = abi.Context(c["w"], c["h"], K, max_frames=2)
        ctx.cloud_reserve(1)
        ctx.upload(0, np.ascontiguousarray(pc["color"][..., 0]))
        ctx.set_idepth(0, np.ascontiguousarray(pc["idepth"]), np.ascontiguousarray(pc["idepth_var"]))
        filt = GOLDEN["filters"][c["filter"]]
        for layout, key in ((abi.CLOUD_VERTEX, "vertex_sha256"), (abi.CLOUD_PLY, "ply_sha256")):
            pts, counts = ctx.export_pointcloud([0], c2w[None], filter=filt, layout=layout)
            assert tuple(counts[0]) == (c["total"], c["displayed"])
            ref = cloud.keyframe(pc, cam, c2w, filt)[0 if layout == abi.CLOUD_VERTEX else 1]
            g = np.ascontiguousarray(pts).view(np.uint32).copy()
            r = ref.view(np.uint32)
            nan = np.isnan(g.view(np.float32)) & np.isnan(r.view(np.float32))
            g[nan] = r[nan]
            assert hashlib.sha256(g.tobytes()).hexdigest() == c[key]
        ctx.close()
        done += 1
    assert done == len(GOLDEN["cases"]) // 2


def test_batched_export_equals_per_keyframe_exports():
    w, h = 320, 240
    seq = synth.Sequence(w, h, seed=99)
    ctx = abi.Context(w, h, seq.K, max_frames=12)
    rng = np.random.default_rng(5)
    img0, d0 = seq.render(0)
    ids, c2ws = list(range(11)), []
    for i in ids:                             # one real keyframe, replicated into further slots with its idepth perturbed
        ctx.upload(i, seq.render(i)[0])
        ctx.set_depth_gt(i, d0 * np.float32(1 + 0.01 * i))
        q = rng.standard_normal(4)
        c2ws.append(np.concatenate([q / np.linalg.norm(q) * (0.5 + 0.2 * i), rng.uniform(-1, 1, 3)]).astype(np.float32))
    c2ws = np.stack(c2ws)
    ctx.cloud_reserve(4)
    for layout in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
        for level in (0, 1):
            pts, counts = ctx.export_pointcloud(ids, c2ws, level=level, layout=layout)
            singles = [ctx.export_pointcloud([i], c2ws[i:i + 1], level=level, layout=layout) for i in ids]
            assert np.array_equal(np.concatenate([s[1] for s in singles]), counts)
            assert np.concatenate([s[0] for s in singles]).tobytes() == pts.tobytes()
            assert len(pts) == counts[:, 1].sum() > 0
            # the same through the count pass (capacity below the bound, but large enough)
            pts2, counts2 = ctx.export_pointcloud(ids, c2ws, level=level, layout=layout, capacity=len(pts))
            assert pts2.tobytes() == pts.tobytes() and np.array_equal(counts2, counts)
    ctx.close()


def _raw_export(ctx, ids, c2w, level=0, filt=None, layout=0, out=None, capacity=0):
    ids = np.ascontiguousarray(ids, np.int32)
    c2w = np.ascontiguousarray(c2w, np.float32)
    f = filt or abi.default_cloud_filter()
    npts = C.c_int64(-1)
    counts = np.full((len(ids), 2), -7, np.int32)
    rc = ctx.L.lsdgpu_map_export_pointcloud(ctx.ptr, len(ids), ids.ctypes.data_as(C.POINTER(C.c_int)),
                                            c2w.ctypes.data_as(C.POINTER(C.c_float)), level, C.byref(f), layout,
                                            None if out is None else out.ctypes.data_as(C.c_void_p), capacity, C.byref(npts),
                                            counts.ctypes.data_as(C.POINTER(C.c_int32)))
    return rc, npts.value, counts, ctx.L.lsdgpu_last_error(ctx.ptr).decode()


def test_count_only_capacity_and_rejected_inputs():
    w, h = 320, 240
    seq = synth.Sequence(w, h, seed=7)
    ctx = abi.Context(w, h, seq.K, max_frames=4)
    img, d = seq.render(0)
    ctx.upload(0, img)
    ctx.set_depth_gt(0, d)
    ctx.upload(1, seq.render(1)[0])           # a frame without depth
    c2w = np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32)
    rc, _, _, err = _raw_export(ctx, [0], c2w)
    assert rc != 0 and "lsdgpu_cloud_reserve" in err
    ctx.cloud_reserve(2)
    pts, counts = ctx.export_pointcloud([0], c2w)
    n = len(pts)
    assert n > 0
    m, cnt = ctx.count_pointcloud([0], c2w)
    assert m == n and np.array_equal(cnt, counts)
    rc, npts, cnt, _ = _raw_export(ctx, [0], c2w)                         # out = NULL: count only
    assert rc == 0 and npts == n and np.array_equal(cnt, counts)
    buf = np.full((n - 1) * 16, 0x5A, np.uint8)
    rc, npts, cnt, _ = _raw_export(ctx, [0], c2w, out=buf, capacity=n - 1)
    assert rc == abi.CLOUD_ERR_CAPACITY and npts == n and np.array_equal(cnt, counts)
    assert (buf == 0x5A).all()                                           # nothing written
    for ids, kw, word in (([0, 17], {}, "17"), ([0, 1], {}, "no depth"), ([0], {"level": 5}, "level"),
                          ([0], {"level": -1}, "level"), ([0], {"layout": 2}, "layout")):
        rc, _, _, err = _raw_export(ctx, ids, np.repeat(c2w, len(ids), 0), **kw)
        assert rc != 0 and word in err, (ids, kw, err)
    rc, _, _, err = _raw_export(ctx, [0], c2w, filt=abi.default_cloud_filter(sparsifyFactor=2))
    assert rc != 0 and "sparsifyFactor" in err
    ctx.close()


def test_interleaved_exports_leave_the_stream_unchanged():
    """a stream stepped with exports between its frames gives bit-identical poses and depth maps to one stepped without"""
    w, h = 320, 240
    seq = synth.Sequence(w, h, seed=2468)
    frames = [seq.render(k) for k in range(22)]
    logs = []
    for export in (False, True):
        ctx = abi.Context(w, h, seq.K, max_frames=12)
        ctx.cloud_reserve(2)
        gs = GpuStream(ctx, mode=1, kf_every=7, keep_keyframes=True)
        gs.init_gt(0, frames[0][0], frames[0][1])
        log = []
        for k in range(1, len(frames)):
            if export:
                for level in (0, 1):
                    ctx.export_pointcloud(gs.keyframe_ids, gs.keyframe_cam_to_world_f7(), level=level)
            pose = gs.step(k, frames[k][0])
            log.append((pose.tobytes(), gs.map.current().tobytes(), ctx.get_pose(k)[0].tobytes()))
        logs.append(log)
        ctx.close()
    assert logs[0] == logs[1]
