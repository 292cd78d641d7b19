"""GPU parity on scenes other than the smooth height field (tests/scenes.py: occluder, posts, stripes, flat, blank, blank_const).

Every other device test renders synth.Sequence's height field, whose depth is continuous: there the occlusion vote of
k_regularize<true>, the occluded-source skip of k_prop_resolve and the colour check of k_prop_project never decide anything, a
depth edge never lies on a border of the shared-memory tiles of k_regularize (32x8 + 2) or k_fill_regularize (32x16 + 4), and
no map, tracker or cloud is ever close to empty.  Here the device is checked against the oracle -- which
tests/test_ref_pin_scenes.py pins to the reference-compiled library on the same scenes, with branch counters that show those
decisions run -- on each textured scene:
  * observeDepth, updateKeyframe, random init + updates, the fill-holes and both regularisers on an observed map, propagateDepth
    from ground truth and from a mapped state, createKeyFrame without and with the tracking mask, finalizeKeyFrame +
    createKeyFrame + update_keyframe_refs: bit for bit;
  * SE3 evaluation on levels 4-1 and trackFrame in modes 0 and 1; Sim3 and permaRef on keyframes the device's mapper finished:
    the tolerances of tests/util.py;
  * the cloud export of a mapped run against the viewer oracle, and the keyframeMsg packing;
  * a replayed closed loop of 20 frames with a keyframe every 8 (oracle/replay.py), and one of `occluder` at 640x480;
and on the blank keyframes: random init (the map and the rand() state after it), mapping, the regularisers, the cloud export,
and every tracker on a keyframe with a handful of points or none, NaN where the oracle's means are over no point."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi
from lsd_slam_b200.stream import GpuStream
from oracle import replay
from tests import device_cases as cases
from tests import pin_cases as pin
from tests import scenes
from tests.util import (CLOUD_FILTERS, IDENT, SUM_TOL, Pair, assert_step_ok, check_perma_track, check_se3_eval, check_sim3_eval,
                        check_sim3_track,
                        oracle_cloud, perma_noise, same_cloud, se3_inverse, sim3_err, sim3_inverse)

pytestmark = pytest.mark.gpu

TEXTURED = list(pin.TEXTURED)
BLANK = ["blank", "blank_const"]


@pytest.fixture(params=TEXTURED)
def scene(request):
    return request.param


@pytest.fixture()
def stream(scene):
    """(320x240 sequence, lazily rendered frames) of the scene, shared with the pin"""
    return scenes.stream(scene)


@pytest.fixture()
def ctx(oracle, stream):
    seq, _ = stream
    c = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    yield c
    c.close()
    oracle.set_globals()


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def test_observe_from_gt_depth_bit_exact(ctx, oracle, stream):
    cases.observe_from_gt(ctx, oracle, *stream)


def test_update_keyframe_sequence_bit_exact(ctx, oracle, stream):
    cases.update_keyframe_sequence(ctx, oracle, *stream)


def test_random_init_observe_and_update_bit_exact(ctx, oracle, stream):
    cases.random_init_observe_and_update(ctx, oracle, *stream)


def test_fill_holes_and_regularize_on_the_observed_map_bit_exact(ctx, oracle, stream):
    """k_fill_regularize and both k_regularize instances on a map with depth edges (occluder, posts: edges on tile borders)"""
    cases.fill_holes_and_regularize_observed(ctx, oracle, *stream)


def test_propagate_from_gt_bit_exact(ctx, oracle, stream):
    """the pin's propagate_from_gt without a tracking mask: the ground-truth map propagated to frame 8, where near sources
    occlude far ones (k_prop_resolve's skip) and uncovered background fails the colour check of k_prop_project"""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "gt")
    k = pin.PROPAGATION_FRAME
    of = p.add_frame(k)
    oracle.lib().lsdo_frame_clear_refPixelWasGood(of.ptr)
    p.odm.propagateDepth(of)
    p.gdm.propagateDepth(k)
    assert p.compare(exact=True)["n_valid"] > 5000


def test_propagate_and_create_keyframe_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe(ctx, oracle, *stream, False)


def test_propagate_and_create_keyframe_with_tracking_mask_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe_device_mask(ctx, oracle, *stream)


def test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, stream):
    cases.finalize_create_and_refs(ctx, oracle, *stream)


# ---- SE3 tracker --------------------------------------------------------------------------------------------------------------
def test_se3_eval_each_level(ctx, oracle, stream):
    cases.se3_eval_each_level(ctx, oracle, *stream, sum_noise=True)


@pytest.mark.parametrize("mode", [0, 1])
def test_se3_track(ctx, oracle, stream, mode):
    cases.se3_track(ctx, oracle, *stream, mode, 3, sum_noise=True)


# ---- Sim3 and permaRef on keyframes the device's mapper finished --------------------------------------------------------------
@pytest.fixture(scope="module", params=TEXTURED)
def mapped(request, oracle):
    run = cases.MappedRun(oracle, 320, 240, request.param, seq=scenes.stream(request.param)[0])
    yield run
    run.close()


def test_mapped_keyframes_mirror_bit_exact(mapped):
    assert len(mapped.kfs) >= 3
    bad = [(k, kf, m) for k, kf, m in mapped.checks if m]
    assert not bad, bad


def test_sim3_eval_on_mapped_keyframes(mapped, oracle):
    cases.mapped_sim3_eval(mapped, oracle)


# (scene, reference keyframe, frame keyframe, startLevel, finalLevel) of the trackFrameSim3 calls on the device's mapped keyframes
# where the reference's fp32 sums take another LM decision than the same tracking with every sum exact (5 level-2 residual
# evaluations against 4); the device takes the exact-sum decision
SIM3_LM_FLIPS = {("occluder", 5, 0, 3, 2)}


def test_track_frame_sim3_on_mapped_keyframes(mapped, oracle):
    """on `occluder` the reference's fp32 sums take one more level-2 LM step than the same tracking with every sum exact; the
    device takes the exact-sum decision (DESIGN.md section 5, Scenes) and is held to that twin there"""
    cases.mapped_sim3_track(mapped, oracle, sum_noise=True, lm_flips=SIM3_LM_FLIPS)


def test_track_frame_sim3_batch_on_mapped_keyframes(mapped, oracle):
    cases.mapped_sim3_batch(mapped, oracle, sum_noise=True)


def test_perma_ref_on_mapped_keyframes(mapped, oracle):
    cases.mapped_perma(mapped, oracle, noise_aware=True)


# ---- the map's point cloud ----------------------------------------------------------------------------------------------------
def test_cloud_export_and_packing_match_oracle(ctx, oracle, stream):
    """the keyframes of a 26-frame run (keyframe every 8): the export of every filter at levels 0 and 1 equal to the viewer
    oracle; keyframeMsg's packing of the active keyframe equal to the oracle's of the same map"""
    seq, frames = stream
    gs = GpuStream(ctx, mode=1, kf_every=8, keep_keyframes=True)
    gs.init_gt(0, *frames[0])
    for k in range(1, 26):
        gs.step(k, frames[k][0])
    ids, c2w = gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    assert len(ids) >= 4
    ctx.cloud_reserve(len(ids))
    for level in (0, 1):
        for layout in (abi.CLOUD_PLY, abi.CLOUD_VERTEX):
            for filt in CLOUD_FILTERS:
                pts, counts = ctx.export_pointcloud(ids, c2w, level=level, filter=filt, layout=layout)
                ref, ref_counts = oracle_cloud(ctx, ids, c2w, level, filt, layout)
                assert (counts == ref_counts).all(), (level, layout, filt)
                same_cloud(pts, ref)
                if filt is None:
                    assert len(pts) > 1000
    kf = gs.kf_id
    okf = oracle.Frame(kf, frames[kf][0], seq.K)
    pin.set_depth(okf, gs.map.current())
    for lvl in (0, 1, 3):
        assert ctx.pack_pointcloud(kf, lvl).tobytes() == okf.pack_pointcloud(lvl).tobytes(), lvl


# ---- closed loops -----------------------------------------------------------------------------------------------------------
def test_closed_loop_replay(oracle, scene, stream):
    """20 frames, keyframe changes at 8 and 16, every step replayed on the oracle from the device's state: the pose within 1e-4
    plus the reference's own summation noise and the map bit for bit.  On `stripes` the texture repeats along x, the direction
    the camera moves, and the tracking cost of a frame can have two minima close together: at frame 15 the reference's own
    trackFrame ends in either one (9.1e-2 apart) when its start pose moves by 1e-6 (relative translation), far below the fp32
    resolution of the steps it takes.  A step whose pose misses the reference's is held there to the nearest of the reference's
    outcomes from such starts (replay.start_outcomes): the same LM call counts, and the pose within 1e-4 plus the summation
    noise plus the spread of those outcomes (the reference's own sensitivity to its start on that step)"""
    seq, frames = stream
    reps = replay.run_with_replay(seq, frames, 20, kf_every=8, keep_snapshots=scene == "stripes")
    assert len(reps) == 19 and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        if scene != "stripes" or (r["pose_rel"] <= 1e-4 + r["ref_noise_rel"] and r["rot_rad"] <= 1e-6 + r["ref_noise_rot"]):
            assert_step_ok(r)
            continue
        assert r["map_ok"], (r["frame"], r["map"])
        outs = replay.start_outcomes(seq, r["snap"], r["frame"], r["image"])
        spread = max(replay.pose_err(o[0], p[0])[0] for o in outs for p in outs)     # the reference's own start sensitivity
        best = min(outs, key=lambda o: replay.pose_err(r["pose"], o[0])[0])
        dt, ang = replay.pose_err(r["pose"], best[0])
        assert dt <= 1e-4 + r["ref_noise_rel"] + spread and ang <= 1e-6 + 10 * r["ref_noise_rot"], (r["frame"], dt, ang, spread)
        assert best[1] == r["residual_calls"], (r["frame"], best[1], r["residual_calls"])


def test_closed_loop_replay_occluder_640(oracle):
    """full size: the box's edges cross many more CTA borders of the observe, regulariser and propagation kernels; every step
    is replayed and the map compared bit for bit after each"""
    seq = scenes.sequence("occluder", 640, 480)
    reps = replay.run_with_replay(seq, scenes.Frames(seq), 20, kf_every=8)
    assert len(reps) == 19 and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        assert_step_ok(r)


# ---- blank keyframes ------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=BLANK)
def blank(request, oracle):
    seq, frames = scenes.stream(request.param)
    c = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    yield request.param, seq, frames, c
    c.close()
    oracle.set_globals()


def test_blank_random_init_mapping_and_regularisers(blank, oracle):
    """initializeRandomly draws as many values as the oracle selects pixels (a few hundred on `blank`, none on `blank_const`)
    and leaves the same rand() state; then updateKeyframe, fill-holes and both regularisers on that map, bit for bit"""
    name, seq, frames, ctx = blank
    img0 = frames[0][0]
    okf = oracle.Frame(0, img0, seq.K)
    odm = oracle.DepthMap(seq.w, seq.h, seq.K)
    libc = C.CDLL(None)
    libc.srand(1)
    odm.initializeRandomly(okf)
    nxt = np.array([libc.rand() for _ in range(pin.EMPTY_RAND_DRAWS)], np.int32)
    ctx.upload(0, img0)
    gdm = abi.DepthMap(ctx)
    st = gdm.initializeRandomly(0, abi.RandState.from_seed(1))
    assert np.array_equal(st.copy().advance(pin.EMPTY_RAND_DRAWS), nxt)
    n = int((odm.current()["isValid"][1:-1, 1:-1] > 0).sum())       # interior: valid == drawn
    assert gdm.last_draws == n and ((n == 0) if name == "blank_const" else (100 < n < 1024)), (name, n)
    assert ((gdm.current()["isValid"] > 0) == (odm.current()["isValid"] > 0)).all()

    p = Pair(ctx, oracle, seq, frames, "random")
    ofs = [p.add_frame(k) for k in (2, 3)]
    p.sync_counters()
    p.odm.updateKeyframe(ofs)
    p.gdm.updateKeyframe([2, 3])
    p.compare(exact=True)
    before = p.gdm.current().copy()
    p.odm.regularizeFillHoles()
    p.gdm.regularizeFillHoles()
    p.compare(exact=True)
    assert np.array_equal(p.gdm.integral(), p.odm.integral())
    for occl in (False, True):
        p.odm.regularize(occl, 24)
        p.gdm.regularize(occl, 24)
        p.compare(exact=True)
    if name == "blank_const":                         # nothing to fill, smooth or remove: the map stays empty
        assert not (p.gdm.current()["isValid"] > 0).any() and not (before["isValid"] > 0).any()


def test_blank_cloud_export(blank, oracle):
    """a 10-frame run from random init, keyframe every 4: a frame the tracker cannot track is reported as diverged and not
    mapped, any other device error fails; the keyframes are the initial one plus one per keyframe change of a tracked step
    (none on `blank_const`, where every step diverges); the export matches the viewer oracle, with no point on `blank_const`"""
    name, seq, frames, ctx = blank
    gs = GpuStream(ctx, mode=1, kf_every=4, keep_keyframes=True)
    gs.init_random(0, frames[0][0], abi.RandState.from_seed(1))
    tracked, changes = 0, 0                           # measured: no step of either blank stream is tracked
    for k in range(1, 10):
        change = gs.next_is_keyframe_change()
        try:
            gs.step(k, frames[k][0])
        except abi.LsdGpuError:
            raise
        except RuntimeError as e:
            assert gs.tracker.diverged and "tracking diverged" in str(e), (k, e)
            continue
        tracked += 1
        changes += change
    ids, c2w = gs.keyframe_ids, gs.keyframe_cam_to_world_f7()
    assert len(ids) == 1 + changes, (ids, changes)
    assert tracked == 0 and ids == [0], (tracked, ids)
    ctx.cloud_reserve(len(ids))
    for level in (0, 1):
        for filt in CLOUD_FILTERS:
            pts, counts = ctx.export_pointcloud(ids, c2w, level=level, filter=filt)
            ref, ref_counts = oracle_cloud(ctx, ids, c2w, level, filt, abi.CLOUD_PLY)
            assert (counts == ref_counts).all(), (level, filt)
            same_cloud(pts, ref)
            if name == "blank_const":
                assert len(pts) == 0 and not counts.any()


SIM3_MEANS = ("sumResD", "sumResP", "mean", "meanD", "meanP", "pointUsage", "affine_a_lastIt", "affine_b_lastIt")


def _check_sim3_eval_nan_aware(got, want, exact):
    """a Sim3 evaluation on a blank keyframe against the oracle's (`want`) and its all-sums-exact twin (`exact`): the counts
    exactly, every mean to SUM_TOL plus the reference's own summation noise |want - exact|, NaN in the same fields.  The one
    exception is the affine estimate sqrt((syy - sy sy / sw) / (sxx - sx sx / sw)) (Sim3Tracker.cpp:591-592) where the frame is
    constant: its numerator is exactly 0 and its computed value rounding noise of the sum order (NaN in the reference's
    sequential sums, a small number in the device's tree sums), so there only its finiteness is not compared"""
    assert (got.warpedSize, got.numTermsD, got.numTermsP, got.num_constraints) == \
        (want.warpedSize, want.numTermsD, want.numTermsP, want.num_constraints)
    for f in SIM3_MEANS:
        a, b, x = getattr(got, f), getattr(want, f), getattr(exact, f)
        if f in ("affine_a_lastIt", "affine_b_lastIt") and not (np.isfinite(want.affine_a_lastIt)
                                                                and np.isfinite(exact.affine_a_lastIt) and exact.affine_a_lastIt != 0):
            continue
        assert np.isnan(a) == np.isnan(b) and (np.isnan(b) or abs(a - b) <= SUM_TOL * abs(b) + abs(b - x) + 1e-6), (f, a, b, x)
    for x, y in ((got.A, want.A), (got.b, want.b)):
        x, y = np.array(x), np.array(y)
        assert np.abs(x - y).max() <= SUM_TOL * np.abs(y).max(), (x, y)


def test_blank_trackers_match_oracle(blank, oracle):
    """the blank keyframe on ground-truth depth: SE3 evaluation on levels 4-1 (NaN where the oracle's means are 0/0),
    trackFrame from identity (pose, diverged, trackingWasGood), setPermaRef, the overlap and trackFrameOnPermaref, and the
    Sim3 evaluation and trackFrameSim3 against a textured keyframe of the default scene in both directions"""
    name, seq, frames, ctx = blank
    okf, of = cases.se3_setup(ctx, oracle, seq, frames, 3)
    trk = abi.SE3Tracker(ctx)
    inv = se3_inverse(oracle, seq.frame_to_ref_qt(3)).astype(np.float32)
    for level in (4, 3, 2, 1):
        got = trk.eval(0, 3, level, inv)
        want = oracle.se3_eval(okf, of, level, inv)
        check_se3_eval(got, want)
        if name == "blank_const":
            assert got.warpedSize == 0 and np.isnan(got.pointUsage) and np.isnan(got.meanRes)
    trk = abi.SE3Tracker(ctx, mode=1)
    pose = trk.trackFrame(0, 3, IDENT)
    r = oracle.se3_track(okf, oracle.Frame(3, frames[3][0], seq.K), IDENT)
    assert trk.diverged == bool(r.diverged) and trk.trackingWasGood == bool(r.trackingWasGood)
    if r.diverged:
        assert np.array_equal(pose, np.array(r.frameToRef_qt))
    else:
        assert np.abs(pose - np.array(r.frameToRef_qt)).max() <= 1e-4
    if name == "blank_const":
        assert r.diverged and not r.trackingWasGood

    pr = oracle.PermaRef(okf)
    assert trk.setPermaRef(0) == pr.n
    img = frames[pin.PERMA_FRAME][0]
    ctx.upload(pin.PERMA_FRAME, img)
    fp = oracle.Frame(pin.PERMA_FRAME, img, seq.K)
    gt = se3_inverse(oracle, seq.frame_to_ref_qt(pin.PERMA_FRAME))
    ov_g, ov_o = trk.checkPermaRefOverlap([0], gt[None])[0], pr.overlap(gt)
    assert np.isnan(ov_g) == np.isnan(ov_o) and (np.isnan(ov_o) or abs(ov_g - ov_o) <= 2e-5 * abs(ov_o) + 1e-6)
    res = trk.trackFrameOnPermaref([0, 0], pin.PERMA_FRAME, np.array([gt, IDENT]))
    for g, init in zip(res, (gt, IDENT)):
        o = pr.track(fp, init)
        check_perma_track(g, o, perma_noise(oracle, pr, fp, init))
        assert bool(g.trackingWasGood) == bool(o.trackingWasGood)
        if o.diverged:
            assert np.array_equal(np.array(g.frameToRef_qt), np.array(o.frameToRef_qt))

    from lsd_slam_b200 import synth
    other = synth.Sequence(seq.w, seq.h, seed=scenes.motions.SEED)
    k = pin.EMPTY_SIM3_KF
    img6, d6 = other.render(k)
    ctx.upload(k, img6)
    ctx.set_depth_gt(k, d6)
    otex = oracle.Frame(k, img6, seq.K)
    otex.setDepthFromGroundTruth(d6)
    q = np.concatenate([seq.frame_to_ref_qt(k), [1.0]])
    q[4:7] += pin.SIM3_DT
    q[7] *= pin.SIM3_SCALE
    s3 = abi.Sim3Tracker(ctx)
    for (ref, oref), (fr, ofr), init in (((0, okf), (k, otex), q), ((k, otex), (0, okf), sim3_inverse(oracle, q))):
        r2f = sim3_inverse(oracle, init)
        for level in (4, 3, 2, 1):
            want = oracle.sim3_eval(oref, ofr, level, r2f)
            oracle.set_globals(exactSim3Sums=1)
            try:
                exact = oracle.sim3_eval(oref, ofr, level, r2f)
            finally:
                oracle.set_globals()
            _check_sim3_eval_nan_aware(s3.eval(ref, fr, level, r2f), want, exact)
        s3.trackFrameSim3(ref, fr, init, 4, 1)
        want = oracle.sim3_track(oref, ofr, init, 4, 1)
        assert s3.diverged == bool(want.diverged), (ref, fr)
        if want.diverged:                             # SE3() / Sim3() returned as the reference returns it
            assert np.array_equal(np.array(s3.last.frameToRef_qts), np.array(want.frameToRef_qts)), (ref, fr)
            continue
        # a textured keyframe tracked onto the blank frame: the reference's fp32 sums alone move its pose 8e-3 from the
        # all-sums-exact twin, and a start moved by 1e-6 (relative translation) moves it by up to 2.3e-2 with other LM counts.
        # The device is held to the nearest of those outcomes of the reference arithmetic (and the twin): the same LM call
        # counts, the pose to POSE_TOL plus the reference's distance to the twin
        if name == "blank_const":
            # onto a constant frame every image gradient is 0: the photometric Jacobian of the pose is 0 and each LM decision
            # compares residuals that differ by rounding only, so only the outcome is compared
            continue
        tw, noise = cases._sum_noise(oracle, oref, ofr, init, 4, 1, want)
        outs = [want, tw]
        rng = np.random.default_rng(0)
        for _ in range(10):
            i2 = np.array(init, np.float64)
            d = rng.normal(size=3)
            i2[4:7] += d / np.linalg.norm(d) * 1e-6 * np.linalg.norm(i2[4:7])
            outs.append(oracle.sim3_track(oref, ofr, i2, 4, 1))
        best = min(outs, key=lambda o: sim3_err(s3.last.frameToRef_qts, o.frameToRef_qts)[0])
        check_sim3_track(s3.last, best, pose_noise=noise[0])
