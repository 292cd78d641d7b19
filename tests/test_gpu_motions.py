"""GPU parity under camera motions other than the default (tests/motions.py: vertical, forward, backward, roll).

Every other device test runs the synthetic stream's default twist, whose epipolar lines are all close to horizontal, so the
y-dominant depth formula of doLineStereo, the near-plane clamp, the firstX and rescale gates and the occlusion outcomes of
propagateDepth (k_prop_resolve) never run on the device there.  Here the device is checked against the oracle -- which
tests/test_ref_pin_motions.py pins to the reference-compiled library under the same motions, with branch counters that show those
branches run -- on each motion:
  * observeDepth from ground truth and from a random map, updateKeyframe over three and four frames, the fill-holes and both
    regularisers on the state the motion produced, finalizeKeyFrame + createKeyFrame + update_keyframe_refs: bit for bit;
  * propagateDepth and createKeyFrame bit for bit, without a tracking mask and with the device's mask handed to the oracle;
  * the wide-baseline update and the propagation collisions of the pin (forward, backward): bit for bit, the latter also with
    the device's own tracking mask handed to the oracle;
  * SE3 evaluation on levels 4-1 and trackFrame in modes 0 and 1: the tolerances of test_gpu_track.py;
  * a replayed closed loop of 20 frames with a keyframe every 8 (oracle/replay.py): the map bit for bit after every step;
  * at 640x480, a closed loop of forward and of roll sampled every 4th step, keyframe changes included."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from oracle import replay
from tests import motions
from tests import test_gpu_depth as gd
from tests import test_gpu_globals as gg
from tests import test_ref_pin_motions as pm
from tests.test_gpu_depth import Pair
from tests.util import IDENT

pytestmark = pytest.mark.gpu

MOTIONS = list(motions.MOTIONS)
COLLIDE = list(pm.ONLY["propagation_collisions"])
WIDE = list(pm.ONLY["wide_baseline"])


@pytest.fixture(params=MOTIONS)
def motion(request):
    return request.param


@pytest.fixture()
def stream(motion):
    """(320x240 sequence, lazily rendered frames) of the motion, shared with the pin"""
    return pm.stream(motion)


@pytest.fixture()
def ctx(oracle, stream):
    seq, _ = stream
    c = abi.Context(seq.w, seq.h, seq.K, max_frames=12)
    yield c
    c.close()
    oracle.set_globals()


# ---- depth map, bit for bit -------------------------------------------------------------------------------------------------
def test_observe_from_gt_depth_bit_exact(ctx, oracle, stream):
    gg.test_observe_from_gt_depth_bit_exact(ctx, oracle, *stream)


def test_update_keyframe_sequence_bit_exact(ctx, oracle, stream):
    gg.test_update_keyframe_sequence_bit_exact(ctx, oracle, *stream)


def test_random_init_observe_and_update_bit_exact(ctx, oracle, stream):
    gg.test_random_init_observe_and_update_bit_exact(ctx, oracle, *stream)


def test_fill_holes_and_regularize_on_the_observed_map_bit_exact(ctx, oracle, stream):
    """the passes of depthmap_individual_passes, on the map one observeDepth under the motion left"""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "gt")
    ofs = [p.add_frame(k) for k in (2, 3)]
    p.sync_counters()
    p.odm.observeDepth(ofs)
    p.gdm.observeDepth([2, 3])
    assert p.compare(exact=True)["n_valid"] > 10000
    p.odm.regularizeFillHoles()
    p.gdm.regularizeFillHoles()
    p.compare(exact=True)
    assert np.array_equal(p.gdm.integral(), p.odm.integral())
    for occl in (False, True):
        p.odm.regularize(occl, 24)
        p.gdm.regularize(occl, 24)
        p.compare(exact=True)


def test_propagate_and_create_keyframe(ctx, oracle, stream):
    gd.test_propagate_and_create_keyframe(ctx, oracle, *stream, False)


def test_propagate_and_create_keyframe_with_tracking_mask_bit_exact(ctx, oracle, stream):
    """test_gpu_depth.test_propagate_and_create_keyframe with the tracking mask, from identical inputs: each frame is tracked on
    the device and its good mask is handed to the oracle, as oracle/replay.py does.  That test's own with-mask variant lets each
    side use its own tracker's mask; the two masks differ on up to 1e-3 of the pixels (test_gpu_track.py), and under the backward
    and roll motions those pixels move the regularised depth of their neighbours after createKeyFrame by up to 1.1e-3, beyond
    the 2e-5 it allows.  With the same mask on both sides every step is bit for bit."""
    seq, frames = stream
    p = gd._tracked_pair(ctx, oracle, seq, frames, [2, 5, 9])
    trk = abi.SE3Tracker(ctx, mode=0)
    for k in (2, 5, 9):
        of = p.oframes[k]
        oracle.lib().lsdo_frame_set_depthHasBeenUpdatedFlag(p.okf.ptr, 0)
        ctx.L.lsdgpu_ref_import(ctx.ptr, 0)
        trk.trackFrame(0, k, IDENT if k == 2 else of.thisToParent()[:7])        # writes the device's mask; the pose is restored
        ctx.set_pose(k, of.thisToParent(), 0, oracle.lib().lsdo_frame_initialTrackedResidual(of.ptr))
        mask = ctx.download(k, abi.BUF_GOODMASK)
        assert mask.mean() > 0.05                      # all ones under forward: every pixel tracked well
        of.refPixelWasGood(create=True)[:] = mask
        p.sync_counters()
        p.odm.updateKeyframe([of])
        p.gdm.updateKeyframe([k])
        p.compare(exact=True)
    before = p.odm.current().copy()
    p.odm.propagateDepth(p.oframes[9])
    p.gdm.propagateDepth(9)
    assert p.compare(exact=True)["n_valid"] > 5000
    p.odm.set_current(before)
    p.gdm.setHypotheses(0, before, do_set_depth=False)
    p.odm.createKeyFrame(p.oframes[9])
    q = p.gdm.createKeyFrame(9)
    assert np.allclose(q[:7], p.oframes[9].thisToParent()[:7], atol=1e-12)
    assert np.float32(q[7]).tobytes() == np.float32(p.oframes[9].thisToParent()[7]).tobytes()
    p.compare(exact=True)
    assert np.array_equal(ctx.download(9, abi.BUF_IDEPTH, 0), p.oframes[9].idepth(0))


def test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, stream):
    gg.test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, *stream)


@pytest.mark.parametrize("motion", WIDE)
def test_wide_baseline_bit_exact(ctx, oracle, stream, motion):
    """pm.wide_baseline: one update with a frame whose depth ratio to the keyframe leaves doLineStereo's rescale gate"""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "gt")
    k = pm.WIDE_BASELINE_FRAME
    of = p.add_frame(k)
    gg._new_depth(p, k)
    p.odm.updateKeyframe([of])
    p.gdm.updateKeyframe([k])
    assert p.compare(exact=True)["n_valid"] > 10000
    gg._kf_depth_equal(ctx, p.okf, 0)


@pytest.mark.parametrize("motion", COLLIDE)
@pytest.mark.parametrize("variant", ["no mask", "mask", "validity 200"])
def test_propagation_collisions_bit_exact(ctx, oracle, stream, motion, variant):
    """pm.propagation_collisions: a random map propagated along the optical axis, so that sources at inconsistent depths land on
    one pixel and k_prop_resolve must skip the occluded ones and replace a target by a nearer source in the reference's raster
    order.  "mask": the device's tracking mask of the new keyframe (SE3 evaluation at level 1 near the true pose), handed to the
    oracle, so both sides propagate from identical inputs.  "validity 200": every merge exceeds the validity cap."""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "random")
    k = pm.PROPAGATION_FRAME
    if variant == "validity 200":
        cur = p.odm.current().copy()
        cur["validity_counter"][cur["isValid"] != 0] = 200
        p.odm.set_current(cur)
        p.gdm.setHypotheses(0, cur, do_set_depth=False)
    of = p.add_frame(k)
    if variant == "mask":
        inv = np.zeros(7)
        oracle.lib().lsdo_se3d_inverse(gg._d(seq.frame_to_ref_qt(k)), gg._d(inv))
        abi.SE3Tracker(ctx).eval(0, k, 1, inv.astype(np.float32), write_mask=True)
        mask = ctx.download(k, abi.BUF_GOODMASK)
        assert 0.05 < mask.mean() < 0.98
        of.refPixelWasGood(create=True)[:] = mask
    before = p.odm.current().copy()
    p.odm.propagateDepth(of)
    p.gdm.propagateDepth(k)
    assert p.compare(exact=True)["n_valid"] > 5000
    assert not np.array_equal(before["idepth"], p.odm.current()["idepth"])


# ---- trackers ---------------------------------------------------------------------------------------------------------------
def test_se3_eval_each_level(ctx, oracle, stream):
    gg.test_se3_eval_each_level(ctx, oracle, *stream)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 8])
def test_se3_track(ctx, oracle, stream, mode, k):
    gg.test_se3_track(ctx, oracle, *stream, mode, k)


# ---- closed loops -----------------------------------------------------------------------------------------------------------
def test_closed_loop_replay(oracle, stream):
    """20 frames, keyframe changes at 8 and 16, every step replayed on the oracle from the device's state"""
    seq, frames = stream
    reps = replay.run_with_replay(seq, frames, 20, kf_every=8)
    assert len(reps) == 19 and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        gg._assert_step_ok(r)


@pytest.mark.parametrize("motion", ["forward", "roll"])
def test_closed_loop_replay_640(oracle, motion):
    """full size: the observe kernel's CTA tiling and the propagation lists see collisions over a 640x480 frame"""
    seq = motions.sequence(motion, 640, 480)
    reps = replay.run_with_replay(seq, motions.Frames(seq), 20, kf_every=8, sample=set(range(4, 20, 4)))
    assert [r["frame"] for r in reps] == [4, 8, 12, 16] and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        gg._assert_step_ok(r)
