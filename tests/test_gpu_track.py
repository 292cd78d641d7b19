"""GPU parity: fused warp/residual/weights/JtJ kernel and SE3Tracker::trackFrame vs the scalar-path oracle.

Tolerances (BASELINE.json north_star): pose <= 1e-4 relative on translation and rotation.  Per-evaluation sums
differ from the oracle only by summation order (sequential float on the CPU, fixed-shape tree on the GPU)."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from tests import device_cases as cases
from tests.device_cases import se3_setup
from tests.util import IDENT, check_se3_eval, pose_err, se3_inverse

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("level", [4, 3, 2, 1])
def test_single_evaluation_parity(gpu_ctx_small, oracle, seq_small, frames_small, level):
    okf, of = se3_setup(gpu_ctx_small, oracle, seq_small, frames_small, 3)
    trk = abi.SE3Tracker(gpu_ctx_small)
    # identity and a pose near the truth
    inv = se3_inverse(oracle, seq_small.frame_to_ref_qt(3))
    for pose, a, b in ((IDENT.astype(np.float32), 1.0, 0.0), (inv.astype(np.float32), 0.98, 1.5)):
        g = trk.eval(0, 3, level, pose, a, b, write_mask=True)
        o = oracle.se3_eval(okf, of, level, pose, a, b, write_mask=True)
        check_se3_eval(g, o)
        if level == 1:
            mg = gpu_ctx_small.download(3, abi.BUF_GOODMASK)
            mo = of.refPixelWasGood()
            assert (mg != mo).mean() < 1e-4


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [1, 3, 8])
def test_track_frame_pose_parity(gpu_ctx_small, oracle, seq_small, frames_small, mode, k):
    cases.se3_track(gpu_ctx_small, oracle, seq_small, frames_small, mode, k)


@pytest.mark.parametrize("mode", [0, 1])
def test_affine_lighting_off_and_zero_motion(seq_small, frames_small, oracle, mode):
    oracle.set_globals(useAffineLightningEstimation=0)      # the ROS default (cfg/LSDParams.cfg:28)
    try:
        ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, max_frames=4, useAffineLightningEstimation=0)
        okf, of = se3_setup(ctx, oracle, seq_small, frames_small, 2)
        trk = abi.SE3Tracker(ctx, mode=mode)
        pg = trk.trackFrame(0, 2, IDENT)
        r = oracle.se3_track(okf, of, IDENT)
        assert pose_err(pg, np.array(r.frameToRef_qt))[0] <= 1e-4
        assert trk.affineEstimation_a == 1.0 and trk.affineEstimation_b == 0.0
        # zero motion: keyframe image tracked against itself
        ctx.upload(50, frames_small[0][0])
        p0 = trk.trackFrame(0, 50, IDENT)
        assert np.abs(p0[:3]).max() < 1e-5 and np.abs(p0[4:]).max() < 1e-5
        ctx.close()
    finally:
        oracle.set_globals()


@pytest.mark.parametrize("mode", [0, 1])
def test_divergence_returns_identity(gpu_ctx_small, oracle, seq_small, frames_small, mode):
    """an initial estimate that looks away from the scene: < 1% of the points warp inside (SE3Tracker.cpp:324-329)"""
    okf, of = se3_setup(gpu_ctx_small, oracle, seq_small, frames_small, 1)
    far = np.array([0, 0.7071067811865476, 0, 0.7071067811865476, 0, 0, 0], np.float64)     # 90 deg about y
    trk = abi.SE3Tracker(gpu_ctx_small, mode=mode)
    p = trk.trackFrame(0, 1, far)
    r = oracle.se3_track(okf, of, far)
    assert r.diverged and trk.diverged and not trk.trackingWasGood
    assert np.array_equal(p, IDENT)


def test_tracker_modes_and_parity_hook_interleave_on_one_context(gpu_ctx_small, oracle, seq_small, frames_small):
    """mode-1 track, single evaluation (parity hook), mode-0 track, mode-1 track again on ONE context: the persistent kernel's
    monotonic barrier counter and the evaluation kernel's last-block counter must not share a word (each would break the other)"""
    okf, of = se3_setup(gpu_ctx_small, oracle, seq_small, frames_small, 3)
    r = oracle.se3_track(okf, of, IDENT)
    pose_o = np.array(r.frameToRef_qt)
    ctx = gpu_ctx_small
    t1, t0 = abi.SE3Tracker(ctx, mode=1), abi.SE3Tracker(ctx, mode=0)
    o_ev = oracle.se3_eval(okf, of, 2, IDENT.astype(np.float32), 1.0, 0.0)
    poses, counts = [], []
    for step in ("m1", "eval", "m0", "eval", "m1", "m1", "m0"):
        if step == "eval":
            check_se3_eval(t1.eval(0, 3, 2, IDENT.astype(np.float32), 1.0, 0.0), o_ev)
            continue
        trk = t1 if step == "m1" else t0
        poses.append(trk.trackFrame(0, 3, IDENT))
        counts.append((list(trk.last.numCalcResidualCalls), list(trk.last.numCalcWarpUpdateCalls)))
    for p, c in zip(poses, counts):
        assert pose_err(p, pose_o)[0] <= 1e-4
        assert c == (list(r.numCalcResidualCalls), list(r.numCalcWarpUpdateCalls))
    assert np.array_equal(poses[0], poses[2]) and np.array_equal(poses[2], poses[3])      # mode 1 is deterministic across the interleaving
    assert np.array_equal(poses[1], poses[4])


def test_new_context_never_sees_the_result_block_of_a_destroyed_one(seq_small, frames_small):
    """The device-resident tracker publishes its result in mapped pinned memory and the host polls a sequence number there.
    Pinned blocks are recycled uncleared by the driver: a fresh context must not take the (matching) sequence number left by a
    destroyed context for the completion of its own first launch.  Contexts come and go while another one stays alive (which is
    what shifted the allocator into handing the same block out again when this was found)."""
    def one(k, keep=False):
        ctx = abi.Context(seq_small.w, seq_small.h, seq_small.K, device=0, max_frames=6)
        ctx.upload(0, frames_small[0][0])
        ctx.set_depth_gt(0, frames_small[0][1])
        ctx.upload(k, frames_small[k][0])
        first = np.array(abi.SE3Tracker(ctx, mode=1).trackFrame(0, k, IDENT))        # launch number 1 of this context
        host = np.array(abi.SE3Tracker(ctx, mode=0).trackFrame(0, k, IDENT))          # host-driven LM, stream-synchronised
        if not keep:
            ctx.close()
        return first, host, ctx
    _, _, alive = one(1, keep=True)
    for k in (1, 3, 8, 2, 6, 1, 8):
        first, host, _ = one(k)
        assert pose_err(first, host)[0] <= 1e-4, k
    alive.close()
