"""GPU parity under exposure changes (tests/photometry.py: ramp, step, saturate, dark, ramp_forward).

Every other device test renders frames at one brightness, so the trackers' c1 = P.a * color + P.b (csrc/track.cuh, csrc/sim3.cuh)
runs near the identity, the final SE3 evaluation has no bad point, and the depth map's stereo and propagation fail only where the
map is wrong.  Here the device is checked on each schedule against the oracle -- which tests/test_ref_pin_photometry.py pins to
the reference-compiled library under the same schedules -- and against the reference's recorded values:
  * the depth-map scenarios of tests/test_gpu_motions.py that do not need a motion along the optical axis (tests/device_cases.py),
    and the pin's propagation_exposure without and with the device's tracking mask: bit for bit;
  * one SE3 evaluation of frame 3 on levels 4-1 at the identity, the frame's true (g, o) and pin_cases.FAR_AFFINE: the counts
    (good and bad included) equal to the reference's recorded ones, the level-1 mask bit for bit to the reference's, the sums
    to the tolerances of tests/util.py against the oracle;
  * trackFrame in modes 0 and 1 of frames 3 and 6 (under `dark` frame 3 is not good): the tolerances of tests/util.py plus the
    reference's own summation noise on that call (its distance to the same call with exact sums: up to 1.6e-4 in translation
    and 1e-2 grey levels in affine b here, where the gain is far from 1); the point usage also by two level-1 points' worth
    (2 / refNum, 2.2e-4), as the good / bad counts are held to 2: it is that of the last evaluated pose, a rejected candidate
    solved from each side's own sums, and under `saturate` in mode 1 one border point lies inside that candidate's image on one
    side only (1.09e-4 = 1 / 9189).  trackingWasGood and the keyframe's tracked counter equal to the oracle's;
  * Sim3 evaluation, trackFrameSim3 and trackFrameOnPermaref on the keyframes oracle/cpu_stream.py mapped from the exposed
    stream: against the exact-affine-sum twin (plus the reference's own distance to that twin), and against the reference's
    recorded values wherever those agree with that twin (REFERENCE_AGREES_WITH_TWIN: 56 of the 60 calls);
  * a replayed closed loop of 20 frames with a keyframe every 8 (oracle/replay.py): the map bit for bit after every step;
  * at 640x480, ramp_forward sampled every 4th step;
  * one constant-exposure and one `ramp` stream in one group call: equal to two single calls."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from oracle import replay
from tests import device_cases as cases
from tests import photometry
from tests import pin_cases as pin
from tests.pin_cases import PROPAGATION_FRAME
from tests.util import (Pair, assert_same, assert_step_ok, check_perma_track, check_se3_eval, check_sim3_eval, check_sim3_track,
                        kf_depth_equal, oracle_sim3_track, perma_noise, se3_inverse, sim3_err)

pytestmark = pytest.mark.gpu

SCHEDULES = list(photometry.SCHEDULES)

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_PHOTOMETRY)
    return _gold


def _g(key):
    return _load()[key]


@pytest.fixture(params=SCHEDULES)
def schedule(request):
    return request.param


@pytest.fixture()
def stream(schedule):
    """(320x240 exposed sequence, lazily rendered frames) of the schedule, shared with the pin"""
    return photometry.stream(schedule)


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


def test_propagate_and_create_keyframe_bit_exact(ctx, oracle, stream):
    """without a tracking mask: propagation's colour check compares the keyframe with frame 9 in raw intensities"""
    cases.propagate_and_create_keyframe(ctx, oracle, *stream, False)


def test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, stream):
    cases.finalize_create_and_refs(ctx, oracle, *stream)


def test_fill_holes_and_regularize_on_the_observed_map_bit_exact(ctx, oracle, stream):
    cases.fill_holes_and_regularize_observed(ctx, oracle, *stream)


def test_propagate_and_create_keyframe_with_tracking_mask_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe_device_mask(ctx, oracle, *stream)


@pytest.mark.parametrize("variant", ["no mask", "mask"])
def test_propagation_exposure_bit_exact(ctx, oracle, stream, variant):
    """the pin's propagation_exposure: the ground-truth map propagated to frame 8 at its true pose.  "no mask": the colour check
    compares raw intensities across the exposure change; "mask": the device's tracking mask of frame 8 (SE3 evaluation at level 1
    at the true pose and the frame's true (a, b)), handed to the oracle"""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "gt")
    k = PROPAGATION_FRAME
    of = p.add_frame(k)
    if variant == "mask":
        inv = se3_inverse(oracle, seq.frame_to_ref_qt(k))
        abi.SE3Tracker(ctx).eval(0, k, 1, inv.astype(np.float32), *seq.affine(k), write_mask=True)
        mask = ctx.download(k, abi.BUF_GOODMASK)
        assert 0.05 < mask.mean()
        of.refPixelWasGood(create=True)[:] = mask
    before = p.odm.current().copy()
    p.odm.propagateDepth(of)
    p.gdm.propagateDepth(k)
    assert p.compare(exact=True)["n_valid"] > 5000
    assert not np.array_equal(before["idepth"], p.odm.current()["idepth"])


# ---- SE3 tracker --------------------------------------------------------------------------------------------------------------
def test_se3_eval_at_wrong_and_true_affine(ctx, oracle, stream, schedule):
    """frame 3 at its ground-truth pose, levels 4..1, at the affine estimates of pin_cases.eval_affines: counts equal to the
    reference's recorded ones, the level-1 mask bit for bit to the reference's, the rest against the oracle"""
    seq, frames = stream
    okf, of = cases.se3_setup(ctx, oracle, seq, frames, 3)
    trk = abi.SE3Tracker(ctx)
    pose = se3_inverse(oracle, seq.frame_to_ref_qt(3)).astype(np.float32)
    rec = pin.Pin(f"{schedule}/se3_eval_exposure", _load())
    n_bad = 0
    for i, (a, b) in enumerate(pin.eval_affines(seq)):
        tag = "" if i == 0 else f"a{a:g}_b{b:g}/"
        for lvl in (4, 3, 2, 1):
            got = trk.eval(0, 3, lvl, pose, a, b, write_mask=lvl == 1)
            counts = np.array([got.warpedSize, got.goodCount, got.badCount], np.float64)
            assert np.array_equal(counts, _g(f"{schedule}/se3_eval_exposure/{tag}L{lvl}/counts")[:3]), (a, b, lvl, counts)
            g = ctx.get_globals()
            oracle.set_globals(exactTrackingSums=1, **g)
            try:
                exact = oracle.se3_eval(okf, of, lvl, pose, a, b)
            finally:
                oracle.set_globals(**g)
            want = oracle.se3_eval(okf, of, lvl, pose, a, b)
            check_se3_eval(got, want, affine_b_noise=abs(want.affine_b_lastIt - exact.affine_b_lastIt))
            n_bad += got.badCount
        rec.exact(f"{tag}mask", ctx.download(3, abi.BUF_GOODMASK) != 0)
    assert n_bad > 1000


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 6])
def test_se3_track(ctx, oracle, stream, schedule, mode, k):
    """trackFrame from identity: check_se3_track holds trackingWasGood, diverged and the keyframe's tracked counter to the
    oracle's; under `dark` frame 3 is not good, every other frame is"""
    cases.se3_track(ctx, oracle, *stream, mode, k, sum_noise=True, usage_points=2)
    trk_good = ctx.get_counters(0)[0] == 1
    assert trk_good == ((schedule, k) != ("dark", photometry.DARK_FRAME))


# ---- Sim3 and permaRef on keyframes the C restatement mapped from the exposed stream ----------------------------------------------
class Loaded:
    """the C restatement's Mapped run of one schedule with its finished keyframes loaded on a device context"""

    def __init__(self, oracle, schedule):
        self.schedule = schedule
        seq, frames = photometry.stream(schedule)
        oracle.set_globals()
        self.m = m = pin.mapped(False, seq, frames)
        self.ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
        dm = abi.DepthMap(self.ctx)
        for k, f in m.of.items():
            self.ctx.upload(k, frames[k][0])
            dm.setHypotheses(k, cases.hyp_of_planes(oracle, f.idepth(0), f.idepthVar(0)), do_set_depth=True)

    def key(self, case, what):
        return f"{self.schedule}/{case}/{what}"


# schedule -> of the 12 trackFrameSim3 calls (6 ordered pairs, levels 4..1 and 3..2), those whose recorded reference pose lies
# within 5e-5 of the oracle's exact-affine-sum twin: with the gain far from 1 the other calls' affine sums move the reference by
# up to 7.2e-5 (step) and 1.2e-4 (saturate), and the device is held to the twin there
REFERENCE_AGREES_WITH_TWIN = {"ramp": 12, "step": 11, "saturate": 9, "dark": 12, "ramp_forward": 12}


@pytest.fixture(scope="module", params=SCHEDULES)
def loaded(request, oracle):
    run = Loaded(oracle, request.param)
    yield run
    run.ctx.close()


def test_sim3_on_mapped_keyframes_against_reference(loaded, oracle):
    m, trk = loaded.m, abi.Sim3Tracker(loaded.ctx)
    n_ref = 0
    for k, f in m.of.items():
        kf_depth_equal(loaded.ctx, f, k)
    for ref, fr in m.pairs():
        for perturb in (True, False):
            r2f = m.ref_to_frame(ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in pin.AB:
                    want = pin.sim3_eval_result(_g(loaded.key("sim3_eval_mapped", f"{ref}->{fr}/p{int(perturb)}/L{lvl}/a{a}")))
                    check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), want)
                far = pin.FAR_AFFINE                # far from the truth: the oracle, which the pin holds to the reference
                check_sim3_eval(trk.eval(ref, fr, lvl, r2f, *far), oracle.sim3_eval(m.of[ref], m.of[fr], lvl, r2f, *far))
        init = m.frame_to_ref(ref, fr)
        for lo, hi in ((4, 1), (3, 2)):
            trk.trackFrameSim3(ref, fr, init, lo, hi)
            want, exact = oracle_sim3_track(oracle, m.of[ref], m.of[fr], init, lo, hi)
            rec = pin.sim3_track_result(_g(loaded.key("sim3_track_mapped", f"{ref}->{fr}/{lo}{hi}")), want)
            check_sim3_track(trk.last, exact, res_tol=5e-4, pose_noise=max(sim3_err(want.frameToRef_qts, exact.frameToRef_qts)))
            # the five affine-lighting sums of calcSim3Buffers carry fp32 noise that feeds back through every accepted step; with
            # a gain far from 1 (step, saturate) it moves the reference's translation by up to 1.6e-4 from the same tracking with
            # exact sums, which the device follows: so the device against the recorded reference wherever the reference agrees
            # with its own exact-sum twin, as device_cases.sim3_batch does off the default settings
            if max(sim3_err(rec.frameToRef_qts, exact.frameToRef_qts)) <= 5e-5:
                check_sim3_track(trk.last, rec)
                n_ref += 1
    assert n_ref == REFERENCE_AGREES_WITH_TWIN[loaded.schedule]


def test_perma_ref_on_mapped_keyframes_against_reference(loaded, oracle):
    m, ctx = loaded.m, loaded.ctx
    se3 = abi.SE3Tracker(ctx)
    prs = {k: oracle.PermaRef(f) for k, f in m.of.items()}
    for k, pr in prs.items():
        assert se3.setPermaRef(k) == pr.n
    img = m.frames[pin.PERMA_FRAME][0]
    ctx.upload(pin.PERMA_FRAME, img)
    of = oracle.Frame(pin.PERMA_FRAME, img, m.seq.K)
    ids, inits, names = [], [], []
    for k in prs:
        for name, init in (("gt", pin.perma_gt(m, k, pin.PERMA_FRAME)), ("identity", pin.IDENT)):
            ids.append(k)
            inits.append(init)
            names.append(name)
    res = se3.trackFrameOnPermaref(ids, pin.PERMA_FRAME, np.array(inits))
    n_good = 0
    for k, init, name, g in zip(ids, inits, names, res):
        want = pin.perma_track_result(_g(loaded.key("perma_mapped", f"kf{k}/track_{name}")), prs[k].track(of, init))
        n_good += check_perma_track(g, want, perma_noise(oracle, prs[k], of, init))
    ctx.release(pin.PERMA_FRAME)
    assert n_good >= 2


# ---- closed loops -----------------------------------------------------------------------------------------------------------
def test_closed_loop_replay(oracle, stream):
    """20 frames, keyframe changes at 8 and 16, every step replayed on the oracle from the device's state"""
    seq, frames = stream
    reps = replay.run_with_replay(seq, frames, 20, kf_every=8)
    assert len(reps) == 19 and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        assert_step_ok(r)


def test_closed_loop_replay_640_ramp_forward(oracle):
    seq = photometry.sequence("ramp_forward", 640, 480)
    reps = replay.run_with_replay(seq, photometry.Frames(seq), 20, kf_every=8, sample=set(range(4, 20, 4)))
    assert [r["frame"] for r in reps] == [4, 8, 12, 16] and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        assert_step_ok(r)


def test_group_constant_and_ramp_equal_single_calls():
    """a constant-exposure stream and a `ramp` stream advanced by one group call per step == two single calls"""
    seqs = [lambda w, h: synth.Sequence(w, h, seed=1234), lambda w, h: photometry.sequence("ramp", w, h)]
    single = cases.run_streams(320, 240, [8, 12], 14, lambda k: False, sequences=seqs)
    group = cases.run_streams(320, 240, [8, 12], 14, lambda k: True, sequences=seqs)
    assert not any(o["diverged"] for step in single for o in step)
    assert sum(o["kf"] for step in single for o in step) == 2
    assert_same(group, single)
