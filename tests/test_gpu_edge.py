"""Edge cases of the path through the C ABI: empty maps, argument errors that must fail loudly, the maximum number of
reference frames of one updateKeyframe, and a keyframe whose depth is entirely invalid (the reference signals these
through `diverged` / asserts, SURVEY 8b)."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests.util import IDENT, Pair

pytestmark = pytest.mark.gpu


def test_tracking_on_a_keyframe_without_any_depth_diverges(gpu_ctx_small, oracle, seq_small, frames_small):
    img0, d0 = frames_small[0]
    img2, _ = frames_small[2]
    nodepth = np.full_like(d0, np.nan)                      # Frame::setDepthFromGroundTruth rejects every pixel (Frame.cpp:268-283)
    gpu_ctx_small.upload(0, img0)
    gpu_ctx_small.set_depth_gt(0, nodepth)
    gpu_ctx_small.upload(2, img2)
    okf = oracle.Frame(0, img0, seq_small.K)
    okf.setDepthFromGroundTruth(nodepth)
    of = oracle.Frame(2, img2, seq_small.K)
    want = oracle.se3_track(okf, of, IDENT)
    assert want.diverged and not want.trackingWasGood
    for mode in (0, 1):
        trk = abi.SE3Tracker(gpu_ctx_small, mode=mode)
        trk.importFrame(0)
        pose = trk.trackFrame(0, 2, IDENT)
        assert trk.diverged and not trk.trackingWasGood
        assert np.array_equal(pose, IDENT)                  # return SE3(), SE3Tracker.cpp:324-329
    s3 = abi.Sim3Tracker(gpu_ctx_small)
    gpu_ctx_small.set_depth_gt(2, frames_small[2][1])
    s3.trackFrameSim3(0, 2, np.concatenate([IDENT, [1.0]]), 4, 1)
    assert s3.diverged and not s3.lastSim3Hessian.any()


def test_update_keyframe_argument_errors(gpu_ctx_small, oracle, seq_small, frames_small):
    p = Pair(gpu_ctx_small, oracle, seq_small, frames_small, "gt")
    dm = p.gdm
    with pytest.raises(abi.LsdGpuError):
        dm.updateKeyframe([])                               # the reference dereferences referenceFrames.front() (DepthMap.cpp:1080)
    with pytest.raises(abi.LsdGpuError):
        dm.updateKeyframe([99])                             # unknown frame
    p.add_frame(1)
    with pytest.raises(abi.LsdGpuError):
        dm.updateKeyframe([1] * 17)                         # more than LSD_MAX_REFS
    dm.invalidate()
    with pytest.raises(abi.LsdGpuError):
        dm.updateKeyframe([1])                              # assert(isValid()), DepthMap.cpp:1074
    with pytest.raises(abi.LsdGpuError):
        dm.finalizeKeyFrame()
    with pytest.raises(abi.LsdGpuError):
        abi.Context(330, 240, seq_small.K)                  # width / height must be multiples of 16 (SlamSystem.cpp:53-57)


def test_many_reference_frames_in_one_update_bit_exact(seq_small, frames_small, oracle):
    """ten reference frames at once (id span 10 <= LSD_MAX_ID_SPAN): the per-pixel choice of the reference frame
    (nextStereoFrameMinID / validity based, DepthMap.cpp:318-334) must match pixel by pixel"""
    ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=14)
    p = Pair(ctx, oracle, seq_small, frames_small, "random")
    refs = list(range(1, 11))
    ofs = [p.add_frame(k) for k in refs]
    p.odm.updateKeyframe(ofs)
    p.gdm.updateKeyframe(refs)
    rep = p.compare(exact=True)
    assert rep["n_valid"] > 1000
    # and a second round on top of it (hypotheses now carry nextStereoFrameMinID > 0)
    p.odm.updateKeyframe(ofs)
    p.gdm.updateKeyframe(refs)
    p.compare(exact=True)
    ctx.close()
