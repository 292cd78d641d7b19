"""The Sim3 tracker (csrc/sim3.cuh) and the permaRef path (csrc/perma.cuh) on keyframes the device's own mapper has finished.

test_gpu_sim3.py and test_gpu_perma.py give their keyframes ground-truth depth: one variance everywhere
(Frame::setDepthFromGroundTruth, Frame.cpp:245-273), kept by the idepth pyramid at every level (Frame.cpp:865), and scales
between keyframes of about 1.  With that input a kernel that reads the wrong variance (the reference point's `s` vs the
frame's `sv`, Sim3Tracker.cpp:527-542, 762-835; the snapshot's colorAndVarData, Frame.cpp:149-174) computes the same
numbers.  Here the keyframes come from a GpuStream run (updateKeyframe / finalizeKeyFrame / createKeyFrame): a semi-dense map
with variances over orders of magnitude, and keyframes rescaled by createKeyFrame (DepthMap.cpp:1285-1304).  Each finished
keyframe is mirrored on the oracle through Frame::setDepth (Frame.cpp:199-243) from the device's level-0 planes, and the last
test loads a map edited to hold the value edges of a real map on both sides.  tests/test_gpu_sim3_motions.py runs the same
scenarios (tests/device_cases.py) under the other camera motions."""
import pytest

from lsd_slam_b200 import abi
from tests import device_cases as dc
from tests.util import POSE_TOL, sim3_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mapped(oracle):
    run = dc.MappedRun(oracle, 320, 240)
    yield run
    run.close()


def test_mapped_keyframes_mirror_bit_exact(mapped):
    dc.mapped_mirror_bit_exact(mapped)


def test_sim3_eval_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_eval(mapped, oracle)


def test_sim3_eval_settings_on_mapped_keyframes(mapped, oracle):
    """var_weight and huber_d other than their defaults (1, 3) reach the kernel's weights"""
    dc.mapped_sim3_eval_settings(mapped, oracle)


def test_track_frame_sim3_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_track(mapped, oracle)


def test_track_frame_sim3_batch_on_mapped_keyframes(mapped, oracle):
    dc.mapped_sim3_batch(mapped, oracle)


def test_track_frame_sim3_batch_on_mapped_keyframes_640x480(oracle):
    run = dc.MappedRun(oracle, 640, 480)
    try:
        assert len(run.kfs) >= 3 and not [c for c in run.checks if c[2]]
        dc.mapped_sim3_batch(run, oracle)
    finally:
        run.close()


def test_cluster_sizes_agree_on_mapped_keyframes(mapped, oracle, monkeypatch):
    trk = abi.Sim3Tracker(mapped.ctx)
    ref, fr = mapped.kfs[0], mapped.kfs[-1]
    init = mapped.frame_to_ref(oracle, ref, fr)
    out = {}
    for cs in (1, 2, 4, 8):
        monkeypatch.setenv("LSDGPU_SIM3_CLUSTER", str(cs))
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        out[cs] = trk.last
    for cs in (1, 2, 4):
        assert list(out[cs].numCalcResidualCalls) == list(out[8].numCalcResidualCalls)
        assert max(sim3_err(out[cs].frameToRef_qts, out[8].frameToRef_qts)) < POSE_TOL


def test_perma_ref_on_mapped_keyframes(mapped, oracle):
    dc.mapped_perma(mapped, oracle)


def test_adversarial_map_edges(mapped, oracle):
    """the edited map of the active keyframe loaded on both sides: pyramids, permaRef and Sim3 on it"""
    dc.mapped_adversarial(mapped, oracle)
