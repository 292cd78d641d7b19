"""GPU parity of the batched permaRef path (SURVEY 8f row 2): Frame::setPermaRef, SE3Tracker::checkPermaRefOverlap and
SE3Tracker::trackFrameOnPermaref (Tracking/SE3Tracker.cpp:121-272) against the oracle, one launch for a whole candidate list."""
import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from tests import device_cases as cases
from tests.util import IDENT, check_perma_overlap

pytestmark = pytest.mark.gpu


def _setup(oracle, w=640, h=480, kf_ids=(0, 6, 12)):
    seq = synth.Sequence(w, h, seed=1234)
    ctx = abi.Context(w, h, seq.K, max_frames=8)
    trk, prs = cases.perma_setup(ctx, oracle, seq, kf_ids, 200)
    return seq, ctx, trk, prs


def test_check_perma_ref_overlap_batch(oracle):
    seq, ctx, trk, prs = _setup(oracle)
    want = check_perma_overlap(trk, oracle, prs, np.random.default_rng(3))
    assert want.min() < 0.9 < want.max()             # the candidates really differ
    ctx.close()


def test_track_frame_on_permaref_batch(oracle):
    seq, ctx, trk, prs = _setup(oracle)
    assert cases.perma_batch(ctx, oracle, seq, trk, prs, 9) >= 3
    ctx.close()


def test_perma_batch_of_many_candidates_is_consistent(oracle):
    """256 copies of the same candidate in one launch give 256 identical results (no cross-CTA state)"""
    seq, ctx, trk, prs = _setup(oracle, kf_ids=(0,))
    img, _ = seq.render(4)
    ctx.upload(4, img)
    res = trk.trackFrameOnPermaref([0] * 256, 4, np.tile(IDENT, (256, 1)))
    first = np.array(res[0].frameToRef_qt)
    assert all(np.array_equal(np.array(r.frameToRef_qt), first) for r in res)
    ctx.close()
