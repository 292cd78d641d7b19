"""GPU parity of the batched Sim3 tracker (SURVEY 8f row 1): Sim3Tracker::trackFrameSim3 and its three hot loops
(Tracking/Sim3Tracker.cpp:149-382, 414-607, 748-856, 992-1047) against the oracle, through the C ABI."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import device_cases as cases
from tests.device_cases import sim3_setup
from tests.util import POSE_TOL, check_sim3_track, oracle_sim3_track, sim3_err, sim3_init

pytestmark = pytest.mark.gpu


def test_sim3_eval_matches_oracle(oracle):
    seq, ctx, trk, of = sim3_setup(oracle)
    cases.sim3_eval(trk, oracle, seq, of)
    ctx.close()


def test_track_frame_sim3_matches_oracle(oracle):
    seq, ctx, trk, of = sim3_setup(oracle)
    for ref, fr in ((0, 6), (6, 0)):
        init = sim3_init(seq, fr, ref)
        est = trk.trackFrameSim3(ref, fr, init, 4, 1)
        want, exact = oracle_sim3_track(oracle, of[ref], of[fr], init)
        assert not want.diverged and abs(want.frameToRef_qts[7] - 1) < 5e-3
        check_sim3_track(trk.last, want)
        check_sim3_track(trk.last, exact, res_tol=5e-4)
        assert np.array_equal(est, np.array(trk.last.frameToRef_qts))
        assert np.allclose(trk.lastSim3Hessian, trk.lastSim3Hessian.T, rtol=1e-5)
    ctx.close()


def test_track_frame_sim3_scale_and_level_range(oracle):
    """keyframe 12 carries a 1.05x larger map; also the (3, 2) level range of SlamSystem::testConstraint's coarse check"""
    seq, ctx, trk, of = sim3_setup(oracle)
    init = np.concatenate([seq.frame_to_ref_qt(12, 0), [1.0]])
    trk.trackFrameSim3(0, 12, init, 4, 1)
    want, exact = oracle_sim3_track(oracle, of[0], of[12], init)
    assert abs(want.frameToRef_qts[7] - 1 / 1.05) < 5e-3
    check_sim3_track(trk.last, want)
    check_sim3_track(trk.last, exact, res_tol=5e-4)
    trk.trackFrameSim3(0, 12, init, 3, 2)
    want, exact = oracle_sim3_track(oracle, of[0], of[12], init, 3, 2)
    assert want.numCalcResidualCalls[4] == 0 and want.numCalcResidualCalls[1] == 0
    check_sim3_track(trk.last, want)
    check_sim3_track(trk.last, exact, res_tol=5e-4)
    ctx.close()


def test_track_frame_sim3_batch(oracle):
    """all ordered pairs in one launch == the same problems one by one (bit-identical) == the oracle"""
    seq, ctx, trk, of = sim3_setup(oracle)
    cases.sim3_batch(trk, oracle, seq, of)
    ctx.close()


def test_track_frame_sim3_early_returns(oracle):
    seq, ctx, trk, of = sim3_setup(oracle)
    far = np.array([0, 0, 0, 1, 50.0, 0, 0, 1.0])
    trk.trackFrameSim3(0, 6, far, 4, 1)
    want = oracle.sim3_track(of[0], of[6], far, 4, 1)
    assert want.diverged and trk.diverged
    assert np.allclose(trk.last.frameToRef_qts, [0, 0, 0, 1, 0, 0, 0, 1]) and not trk.lastSim3Hessian.any()
    with pytest.raises(abi.LsdGpuError):
        img, _ = seq.render(3)
        ctx.upload(3, img)                       # no depth on frame 3
        trk.trackFrameSim3(0, 3, far, 4, 1)
    ctx.close()


def test_cluster_sizes_agree(oracle, monkeypatch):
    """the per-problem cluster size only changes how the level is split: decisions and iteration counts are identical,
    sums differ by float re-association only"""
    seq, ctx, trk, of = sim3_setup(oracle)
    init = sim3_init(seq, 6, 0)
    out = {}
    for cs in (1, 2, 4, 8):
        monkeypatch.setenv("LSDGPU_SIM3_CLUSTER", str(cs))
        trk.trackFrameSim3(0, 6, init, 4, 1)
        out[cs] = trk.last
    for cs in (1, 2, 4):
        assert list(out[cs].numCalcResidualCalls) == list(out[8].numCalcResidualCalls)
        dt, ang, ds = sim3_err(out[cs].frameToRef_qts, out[8].frameToRef_qts)
        assert max(dt, ang, ds) < POSE_TOL
    ctx.close()
