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
  * SE3 evaluation on levels 4-1 and trackFrame in modes 0 and 1: the tolerances of tests/util.py's checks;
  * a replayed closed loop of 20 frames with a keyframe every 8 (oracle/replay.py): the map bit for bit after every step;
  * at 640x480, a closed loop of forward and of roll sampled every 4th step, keyframe changes included."""
import numpy as np
import pytest

from lsd_slam_b200 import abi
from oracle import replay
from tests import device_cases as cases
from tests import motions
from tests.pin_cases import ONLY, PROPAGATION_FRAME, WIDE_BASELINE_FRAME
from tests.util import Pair, assert_step_ok, kf_depth_equal, new_depth, se3_inverse

pytestmark = pytest.mark.gpu

MOTIONS = list(motions.MOTIONS)
COLLIDE = list(ONLY["propagation_collisions"])
WIDE = list(ONLY["wide_baseline"])


@pytest.fixture(params=MOTIONS)
def motion(request):
    return request.param


@pytest.fixture()
def stream(motion):
    """(320x240 sequence, lazily rendered frames) of the motion, shared with the pin"""
    return motions.stream(motion)


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
    cases.fill_holes_and_regularize_observed(ctx, oracle, *stream)


def test_propagate_and_create_keyframe(ctx, oracle, stream):
    cases.propagate_and_create_keyframe(ctx, oracle, *stream, False)


def test_propagate_and_create_keyframe_with_tracking_mask_bit_exact(ctx, oracle, stream):
    cases.propagate_and_create_keyframe_device_mask(ctx, oracle, *stream)


def test_finalize_create_keyframe_and_refs_bit_exact(ctx, oracle, stream):
    cases.finalize_create_and_refs(ctx, oracle, *stream)


@pytest.mark.parametrize("motion", WIDE)
def test_wide_baseline_bit_exact(ctx, oracle, stream, motion):
    """the pin's wide_baseline: one update with a frame whose depth ratio to the keyframe leaves doLineStereo's rescale gate"""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "gt")
    k = WIDE_BASELINE_FRAME
    of = p.add_frame(k)
    new_depth(p)
    p.odm.updateKeyframe([of])
    p.gdm.updateKeyframe([k])
    assert p.compare(exact=True)["n_valid"] > 10000
    kf_depth_equal(ctx, p.okf, 0)


@pytest.mark.parametrize("motion", COLLIDE)
@pytest.mark.parametrize("variant", ["no mask", "mask", "validity 200"])
def test_propagation_collisions_bit_exact(ctx, oracle, stream, motion, variant):
    """the pin's propagation_collisions: a random map propagated along the optical axis, so that sources at inconsistent depths land on
    one pixel and k_prop_resolve must skip the occluded ones and replace a target by a nearer source in the reference's raster
    order.  "mask": the device's tracking mask of the new keyframe (SE3 evaluation at level 1 near the true pose), handed to the
    oracle, so both sides propagate from identical inputs.  "validity 200": every merge exceeds the validity cap."""
    seq, frames = stream
    p = Pair(ctx, oracle, seq, frames, "random")
    k = PROPAGATION_FRAME
    if variant == "validity 200":
        cur = p.odm.current().copy()
        cur["validity_counter"][cur["isValid"] != 0] = 200
        p.odm.set_current(cur)
        p.gdm.setHypotheses(0, cur, do_set_depth=False)
    of = p.add_frame(k)
    if variant == "mask":
        inv = se3_inverse(oracle, seq.frame_to_ref_qt(k))
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
    cases.se3_eval_each_level(ctx, oracle, *stream, sum_noise=True)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [3, 8])
def test_se3_track(ctx, oracle, stream, mode, k):
    cases.se3_track(ctx, oracle, *stream, mode, k)


# ---- closed loops -----------------------------------------------------------------------------------------------------------
def test_closed_loop_replay(oracle, stream):
    """20 frames, keyframe changes at 8 and 16, every step replayed on the oracle from the device's state"""
    seq, frames = stream
    reps = replay.run_with_replay(seq, frames, 20, kf_every=8)
    assert len(reps) == 19 and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        assert_step_ok(r)


@pytest.mark.parametrize("motion", ["forward", "roll"])
def test_closed_loop_replay_640(oracle, motion):
    """full size: the observe kernel's CTA tiling and the propagation lists see collisions over a 640x480 frame"""
    seq = motions.sequence(motion, 640, 480)
    reps = replay.run_with_replay(seq, motions.Frames(seq), 20, kf_every=8, sample=set(range(4, 20, 4)))
    assert [r["frame"] for r in reps] == [4, 8, 12, 16] and [r["frame"] for r in reps if r["kf_change"]] == [8, 16]
    for r in reps:
        assert_step_ok(r)
