"""GPU parity of the keyframe output formats (SURVEY 8f row 4): the keyframeMsg.pointcloud packing loop
(IOWrapper/ROS/ROSOutput3DWrapper.cpp:91-110), Frame::takeReActivationData (DataStructures/Frame.cpp:107-145) and
DepthMap::setFromExistingKF (DepthEstimation/DepthMap.cpp:920-962): byte-identical to the oracle."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests.util import Pair, hyp_equal_report

pytestmark = pytest.mark.gpu


def _mapped_pair(ctx, oracle, seq, frames):
    """random init + two mapping iterations, so that the map holds valid, invalid and blacklisted pixels"""
    p = Pair(ctx, oracle, seq, frames, "random")
    for k in (4, 6):
        of = p.add_frame(k)
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
    return p


def test_pack_pointcloud_bytes(gpu_ctx_small, oracle, seq_small, frames_small):
    p = _mapped_pair(gpu_ctx_small, oracle, seq_small, frames_small)
    assert abi.POINT_DENSE.itemsize == 12
    for lvl in (0, 1, 3):
        got = gpu_ctx_small.pack_pointcloud(0, lvl)
        want = p.okf.pack_pointcloud(lvl)
        assert got.tobytes() == want.tobytes(), lvl
        assert (want["idepth_var"] > 0).sum() > 50


def test_take_reactivation_data_and_set_from_existing_kf(gpu_ctx_small, oracle, seq_small, frames_small):
    p = _mapped_pair(gpu_ctx_small, oracle, seq_small, frames_small)
    p.odm.finalizeKeyFrame()                       # ... takeReActivationData, DepthMap.cpp:1387
    p.gdm.finalizeKeyFrame()
    p.compare(exact=True)
    got, want = gpu_ctx_small.reactivation_data(0), p.okf.reactivation_data()
    for g, w, name in zip(got, want, ("idepth_reAct", "idepthVar_reAct", "validity_reAct")):
        assert g.tobytes() == w.tobytes(), name
    assert (want[1] > 0).any() and (want[1] == -1).any()

    # a second take after more mapping keeps the entries of now-invalid pixels (buffers are not cleared)
    of = p.add_frame(8)
    p.odm.updateKeyframe([of])
    p.gdm.updateKeyframe([8])
    oracle.lib().lsdo_frame_takeReActivationData(p.okf.ptr, p.odm.L.lsdo_depthmap_current(p.odm.ptr))
    gpu_ctx_small.take_reactivation_data(0)
    for g, w in zip(gpu_ctx_small.reactivation_data(0), p.okf.reactivation_data()):
        assert g.tobytes() == w.tobytes()

    # re-activate the keyframe into a fresh depth map on both sides
    odm2 = oracle.DepthMap(seq_small.w, seq_small.h, seq_small.K)
    odm2.setFromExistingKF(p.okf)
    p.gdm.reset()
    p.gdm.setFromExistingKF(0)
    rep = hyp_equal_report(p.gdm.current(), odm2.current().copy())
    assert rep["valid_mismatch"] == 0 and rep["blacklist_mismatch"] == 0 and rep["validity_mismatch"] == 0, rep
    for f in ("idepth", "idepth_var", "idepth_smoothed", "idepth_var_smoothed", "nextStereoFrameMinID"):
        assert rep[f + "_bitdiff"] == 0, rep
    assert rep["n_valid"] > 1000
    assert gpu_ctx_small.get_counters(0)[:2] == (0, 0)          # numFramesTrackedOnThis / numMappedOnThis reset, :932-933


def test_set_from_existing_kf_needs_reactivation_data(gpu_ctx_small, seq_small, frames_small):
    img, d = frames_small[0]
    gpu_ctx_small.upload(0, img)
    gpu_ctx_small.set_depth_gt(0, d)
    with pytest.raises(abi.LsdGpuError):
        abi.DepthMap(gpu_ctx_small).setFromExistingKF(0)
