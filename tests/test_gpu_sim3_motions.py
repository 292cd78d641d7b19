"""The Sim3 tracker (csrc/sim3.cuh) and the permaRef path (csrc/perma.cuh) on mapped keyframes under every camera motion, against
the reference's own code and against the oracle.

Against the reference: the keyframes of tests/test_ref_pin_sim3.py (oracle/cpu_stream.py's loop, keyframes 0, 5 and 10 of 16
frames, on the default twist and the motions of tests/motions.py) are rebuilt with the C restatement -- deterministic, and pinned
to the reference by that test -- and loaded on the device through DepthMap setHypotheses + setDepth.  Their pyramids must equal
the oracle's bit for bit.  Every Sim3 evaluation, trackFrameSim3 (one by one and batched), permaRef overlap and
trackFrameOnPermaref of the pin is then compared with the reference's recorded values (tests/golden/ref_pin_sim3_320x240.npz)
with the tolerances of tests/util.py, and each tracking also with the exact-affine-sum twin of the oracle.

Device-mapped: the scenarios of tests/test_gpu_mapped_keyframes.py (tests/device_cases.py) on keyframes the device's own mapper
finished on each motion's stream, and the 640x480 batch under forward and roll."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import device_cases as dc
from tests import motions
from tests import pin_cases as pin
from tests.util import (OVERLAP_ATOL, OVERLAP_RTOL, check_perma_track, check_sim3_eval, check_sim3_track, kf_depth_equal,
                        oracle_sim3_track, perma_noise)

pytestmark = pytest.mark.gpu

_gold = None


def _g(key):
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_SIM3)
    return _gold[key]


class Loaded:
    """the C restatement's Mapped run of one motion with its finished keyframes loaded on a device context"""

    def __init__(self, oracle, motion):
        self.motion = motion
        seq, frames = motions.stream(motion)
        oracle.set_globals()
        self.m = m = pin.mapped(False, seq, frames)
        self.ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
        self.dm = abi.DepthMap(self.ctx)
        for k, f in m.of.items():
            self.ctx.upload(k, frames[k][0])
            self.dm.setHypotheses(k, dc.hyp_of_planes(oracle, f.idepth(0), f.idepthVar(0)), do_set_depth=True)

    def key(self, case, what):
        return f"{self.motion}/{case}/{what}"


@pytest.fixture(scope="module", params=pin.SIM3_MOTIONS)
def loaded(request, oracle):
    run = Loaded(oracle, request.param)
    yield run
    run.ctx.close()


def test_loaded_keyframes_bit_exact(loaded):
    """setHypotheses + setDepth of the oracle's level-0 planes gives the oracle's pyramids at every level"""
    for k, f in loaded.m.of.items():
        kf_depth_equal(loaded.ctx, f, k)


def test_sim3_eval_against_reference(loaded):
    m, trk = loaded.m, abi.Sim3Tracker(loaded.ctx)
    n_no_depth = 0
    for ref, fr in m.pairs():
        for perturb in (True, False):
            r2f = m.ref_to_frame(ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in pin.AB:
                    want = pin.sim3_eval_result(_g(loaded.key("sim3_eval_mapped", f"{ref}->{fr}/p{int(perturb)}/L{lvl}/a{a}")))
                    check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), want)
                    n_no_depth += want.numTermsD < want.numTermsP
    assert n_no_depth > 0
    for k, v in pin.SIM3_SETTINGS.items():
        setattr(trk.settings, k, v)
    ref, fr = m.kfs[0], m.kfs[-1]
    r2f = m.ref_to_frame(ref, fr)
    for lvl in (4, 3, 2, 1):
        a, b = pin.AB[lvl % 2]
        check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), pin.sim3_eval_result(_g(loaded.key("sim3_eval_mapped", f"settings/{ref}->{fr}/L{lvl}"))))


def _track_against_reference(oracle, motion, m, got, ref, fr, init, lo, hi, key):
    """got against the reference's recorded result (the LM call counters, locals there, from the oracle pinned to it) and against
    the oracle's exact-affine-sum twin (lastDepthResidual of pin_cases.POSE_SENSITIVE_DEPTH_RESIDUAL to the reference tolerance)"""
    want, exact = oracle_sim3_track(oracle, m.of[ref], m.of[fr], init, lo, hi)
    check_sim3_track(got, pin.sim3_track_result(_g(key), want))
    sensitive = (motion, ref, fr, lo, hi) in pin.POSE_SENSITIVE_DEPTH_RESIDUAL
    check_sim3_track(got, exact, res_tol=5e-4, depth_res_tol=2e-2 if sensitive else None)


def test_track_frame_sim3_against_reference(loaded, oracle):
    m, trk = loaded.m, abi.Sim3Tracker(loaded.ctx)
    for ref, fr in m.pairs():
        init = m.frame_to_ref(ref, fr)
        for lo, hi in ((4, 1), (3, 2)):
            trk.trackFrameSim3(ref, fr, init, lo, hi)
            assert not trk.diverged
            _track_against_reference(oracle, loaded.motion, m, trk.last, ref, fr, init, lo, hi, loaded.key("sim3_track_mapped", f"{ref}->{fr}/{lo}{hi}"))


def test_track_frame_sim3_batch_against_reference(loaded, oracle):
    m, trk = loaded.m, abi.Sim3Tracker(loaded.ctx)
    pairs = m.pairs()
    inits = np.array([m.frame_to_ref(ref, fr) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    for (ref, fr), init, r in zip(pairs, inits, res):
        _track_against_reference(oracle, loaded.motion, m, r, ref, fr, init, 4, 1, loaded.key("sim3_track_mapped", f"{ref}->{fr}/41"))


def _perma_against_reference(oracle, run, m, prs, case, key=lambda k: f"kf{k}"):
    """checkPermaRefOverlap at pin.overlap_poses and the ground-truth pose, trackFrameOnPermaref of pin.PERMA_FRAME from ground
    truth and identity, on the device's permaRefs, against the recorded reference values"""
    se3 = abi.SE3Tracker(run.ctx)
    for k, pr in prs.items():
        assert se3.setPermaRef(k) == pr.n
    poses = pin.overlap_poses(prs)
    ids = [k for k in prs for _ in range(6)]
    qs = np.array([q for k in prs for q in poses[k] + [pin.perma_gt(m, k, pin.PERMA_FRAME)]])
    got = se3.checkPermaRefOverlap(ids, qs)
    want = np.concatenate([_g(run.key(case, f"{key(k)}/overlap_values")) for k in prs])
    assert np.allclose(got, want, rtol=OVERLAP_RTOL, atol=OVERLAP_ATOL), np.abs(got - want).max()

    img = m.frames[pin.PERMA_FRAME][0]
    run.ctx.upload(pin.PERMA_FRAME, img)
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
        want = pin.perma_track_result(_g(run.key(case, f"{key(k)}/track_{name}")), prs[k].track(of, init))
        n_good += check_perma_track(g, want, perma_noise(oracle, prs[k], of, init))
    run.ctx.release(pin.PERMA_FRAME)
    return n_good


def test_perma_ref_against_reference(loaded, oracle):
    m = loaded.m
    prs = {k: oracle.PermaRef(f) for k, f in m.of.items()}
    assert _perma_against_reference(oracle, loaded, m, prs, "perma_mapped") >= 2


@pytest.mark.parametrize("motion", pin.SIM3_ONLY["adversarial_map"])
def test_adversarial_map_against_reference(motion, oracle):
    """pin_cases.adversarial_keyframe loaded on the device as the active keyframe: pyramids bit for bit, then permaRef and Sim3
    against the reference's recorded values"""
    run = Loaded(oracle, motion)
    try:
        m, case = run.m, "adversarial_map"
        okf, hyp = pin.adversarial_keyframe(False, m)
        run.ctx.upload(m.active, m.frames[m.active][0])
        run.dm.setHypotheses(m.active, hyp, do_set_depth=True)
        kf_depth_equal(run.ctx, okf, m.active)
        pr = oracle.PermaRef(okf)
        _perma_against_reference(oracle, run, m, {m.active: pr}, case)
        of = dict(m.of)
        of[m.active] = okf
        trk = abi.Sim3Tracker(run.ctx)
        for ref, fr in ((m.active, m.kfs[-1]), (m.kfs[-1], m.active)):
            r2f = m.ref_to_frame(ref, fr)
            for lvl in range(abi.LEVELS):
                for a, b in pin.AB:
                    check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), pin.sim3_eval_result(_g(run.key(case, f"{ref}->{fr}/L{lvl}/a{a}"))))
            init = m.frame_to_ref(ref, fr)
            trk.trackFrameSim3(ref, fr, init, 4, 1)
            want, exact = oracle_sim3_track(oracle, of[ref], of[fr], init)
            rec = pin.sim3_track_result(_g(run.key(case, f"{ref}->{fr}/track")), want)
            assert trk.diverged == bool(rec.diverged)
            if not rec.diverged:
                check_sim3_track(trk.last, rec)
                check_sim3_track(trk.last, exact, res_tol=5e-4)
    finally:
        run.ctx.close()


# ---- keyframes the device's mapper finished, on each motion's stream (tests/device_cases.py) --------------------------------
@pytest.fixture(scope="module", params=list(motions.MOTIONS))
def mapped(request, oracle):
    run = dc.MappedRun(oracle, 320, 240, request.param)
    yield run
    run.close()


def test_mapped_keyframes_mirror_bit_exact(mapped):
    dc.mapped_mirror_bit_exact(mapped)


def test_sim3_eval_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_eval(mapped, oracle)


def test_sim3_eval_settings_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_eval_settings(mapped, oracle)


def test_track_frame_sim3_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_track(mapped, oracle)


def test_track_frame_sim3_batch_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_batch(mapped, oracle)


def test_perma_ref_on_mapped_keyframes(mapped, oracle):
    dc.mapped_perma(mapped, oracle, noise_aware=True)


def test_adversarial_map_edges(mapped, oracle):
    dc.mapped_adversarial(mapped, oracle)


@pytest.mark.parametrize("motion", ["forward", "roll"])
def test_track_frame_sim3_batch_on_mapped_keyframes_640x480(motion, oracle):
    run = dc.MappedRun(oracle, 640, 480, motion)
    try:
        assert len(run.kfs) >= 3 and not [c for c in run.checks if c[2]]
        dc.mapped_sim3_batch(run, oracle)
    finally:
        run.close()
