"""PIN of the oracle: the hand-written C restatement (oracle/lsd_oracle.c) against the reference's OWN sources (DepthMap.cpp,
SE3Tracker.cpp, Sim3Tracker.cpp, TrackingReference.cpp, Frame.cpp, ... and the vendored Sophus) compiled unmodified by
oracle/ref_build.py into oracle/_ref/ -- on identical inputs.

* Frame builders, point cloud, stereo constants, and the WHOLE DepthMap (observe / line stereo / fill holes /
  regularise / propagate / createKeyFrame / finalizeKeyFrame) must agree BIT FOR BIT, every field of every pixel.
* Tracking (fp32 sums in another association order on neither side: both are sequential) must agree to fp32
  round-off in every reported quantity, and poses within 1e-5.

The reference side of every comparison is recorded in tests/golden/ref_pin_320x240.npz (python -m tests.golden.make_golden,
which runs the case functions of tests/pin_cases.py on the reference-compiled library): bit-exact observations as SHA-256
digests of their bytes, the others as values.  The tests run the C restatement and check each observation against the record, so they need
neither the reference sources nor oracle/_ref."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import pin_cases as pin
from tests.util import IDENT, pose_err


def test_frame_builders_bit_exact(seq_small, frames_small):
    pin.run("frame_builders", seq_small, frames_small)


def test_point_cloud_bit_exact(seq_small, frames_small):
    pin.run("point_cloud", seq_small, frames_small)


def test_prepare_for_stereo_bit_exact(seq_small, frames_small):
    pin.run("prepare_for_stereo", seq_small, frames_small)


def test_depthmap_update_sequence_bit_exact(seq_small, frames_small):
    pin.run("depthmap_update_sequence", seq_small, frames_small)


def test_depthmap_random_init_every_branch_bit_exact(seq_small, frames_small):
    pin.run("depthmap_random_init_every_branch", seq_small, frames_small)


def test_depthmap_individual_passes_bit_exact(seq_small, frames_small):
    pin.run("depthmap_individual_passes", seq_small, frames_small)


def test_create_keyframe_and_finalize_bit_exact(seq_small, frames_small):
    pin.run("create_keyframe_and_finalize", seq_small, frames_small)


def test_se3_single_evaluation_matches_reference_compiled(seq_small, frames_small):
    pin.run("se3_single_evaluation", seq_small, frames_small)


@pytest.mark.parametrize("pair", ["scalar", "sse"])
def test_se3_track_matches_reference_compiled(seq_small, frames_small, pair):
    pin.run(f"se3_track_{pair}", seq_small, frames_small)


def test_sse_vs_scalar_gap_of_the_reference_itself(seq_small, frames_small):
    """The stock build defines ENABLE_SSE (CMakeLists.txt:37-43): _mm_rcp_ps weights, N mod 4 points dropped.  The recorded
    poses of the reference's two code paths on the same input show how far they are apart (documented in DESIGN.md section 2):
    the scalar path is the parity target of the CUDA kernels, the SSE path the timing baseline.  The oracle's scalar path
    reproduces the recorded scalar pose exactly and its SSE restatement the recorded SSE pose within 1e-4."""
    g = np.load(pin.GOLD)
    ref, sse = g["sse_gap/ref"], g["sse_gap/ref_sse"]
    dt, ang = pose_err(sse, ref)
    gt = seq_small.frame_to_ref_qt(3)
    e_scalar, _ = pose_err(ref, gt)
    e_sse, _ = pose_err(sse, gt)
    print(f"reference SSE vs reference scalar: translation {dt:.2e} rel, rotation {ang:.2e} rad; "
          f"vs ground truth: scalar {e_scalar:.2e}, SSE {e_sse:.2e}")
    assert 1e-4 < dt < 5e-2             # both minimise the same cost; they are NOT within 1e-4 of each other
    assert abs(e_scalar - e_sse) < 2e-2 # and neither is closer to the ground truth than the other by more than that
    for fl, want in ((False, ref), (True, sse)):
        po.set_globals(fl, useSSE=1) if fl is True else po.set_globals(fl)
        kf = po.Frame(0, frames_small[0][0], seq_small.K, fast=fl)
        kf.setDepthFromGroundTruth(frames_small[0][1])
        f = po.Frame(3, frames_small[3][0], seq_small.K, fast=fl)
        got = np.array(po.se3_track(kf, f, IDENT, po.default_track_settings(fl)).frameToRef_qt)
        if fl is False:
            assert np.array_equal(got, want), got - want
        else:
            assert pose_err(got, want)[0] <= 1e-4
    po.set_globals(False)


def test_bench_loop_with_keyframe_changes_bit_exact(seq_small, frames_small):
    pin.run("bench_loop_with_keyframe_changes", seq_small, frames_small)
