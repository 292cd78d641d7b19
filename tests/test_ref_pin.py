"""PIN of the oracle: the hand-written C restatement (oracle/lsd_oracle.c) against the reference's OWN sources (DepthMap.cpp,
SE3Tracker.cpp, Sim3Tracker.cpp, TrackingReference.cpp, Frame.cpp, ... and the vendored Sophus) compiled unmodified by
oracle/ref_build.py into oracle/_ref/ -- on identical inputs.

* Frame builders, point cloud, stereo constants, and the WHOLE DepthMap (observe / line stereo / fill holes /
  regularise / propagate / createKeyFrame / finalizeKeyFrame) must agree BIT FOR BIT, every field of every pixel.
* Tracking (fp32 sums in another association order on neither side: both are sequential) must agree to fp32
  round-off in every reported quantity, and poses within 1e-5.

The reference side of every comparison is recorded in tests/golden/ref_pin_320x240.npz (python -m tests.golden.make_golden,
which runs the same functions below on the reference-compiled library): bit-exact observations as SHA-256 digests of their
bytes, the others as values.  The tests run the C restatement and check each observation against the record, so they need
neither the reference sources nor oracle/_ref."""
import contextlib
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.util import IDENT, pose_err

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin_320x240.npz")

FIELDS = ("isValid", "blacklisted", "nextStereoFrameMinID", "validity_counter", "idepth", "idepth_var",
          "idepth_smoothed", "idepth_var_smoothed")


def _bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


class Pin:
    """The observations of one comparison.  Recording (gold=None): stores them.  Checking: `exact` asserts the digest of the
    observation equals the recorded one; `value` returns the recorded value for the caller's own tolerance."""

    def __init__(self, case, gold=None):
        self.case, self.gold, self.rec = case, gold, {}

    def _key(self, what):
        return f"{self.case}/{what}"

    def exact(self, what, a):
        d = bytes.fromhex(_digest(a))
        if self.gold is None:
            self.rec[self._key(what)] = np.frombuffer(d, np.uint8)
        else:
            assert self.gold[self._key(what)].tobytes() == d, f"{self.case}: {what} differs from the reference"

    def value(self, what, a):
        a = np.asarray(a)
        if self.gold is None:
            self.rec[self._key(what)] = a.copy()
            return a
        return self.gold[self._key(what)]

    def hyp(self, what, h):
        """isValid and blacklisted on every pixel; every other field, as bit patterns, on every valid pixel.  (The reference's
        DepthMapPixelHypothesis() constructor sets only isValid and blacklisted -- DepthMapPixelHypothesis.h:63-64 -- so the
        other fields of a never-valid pixel are uninitialised heap memory in the reference and carry no information.)"""
        va = h["isValid"] != 0
        self.exact(f"{what}/isValid", va)
        self.exact(f"{what}/blacklisted", np.ascontiguousarray(h["blacklisted"]))
        for f in FIELDS[2:]:
            self.exact(f"{what}/{f}", _bits(np.ascontiguousarray(h[f]))[va])
        return int(va.sum())


_gold = None

# the run-time settings of util/settings.cpp:80-88 the cases run under, on both flavours; empty = the reference's defaults.
# tests/test_ref_pin_globals.py runs cases under others (the ranges of cfg/LSDParams.cfg:13-34).
_SETTINGS: dict = {}


def set_globals(fl, **kw):
    return po.set_globals(fl, **_SETTINGS, **kw)


@contextlib.contextmanager
def settings(**g):
    """run cases under the run-time settings `g` (each unset one at its default)"""
    global _SETTINGS
    old, _SETTINGS = _SETTINGS, dict(g)
    try:
        yield
    finally:
        _SETTINGS = old


def _check(case):
    global _gold
    if _gold is None:
        _gold = np.load(GOLD)
    return Pin(case, _gold)


class Side:
    """one flavour's keyframe, depth map and frames, driven through the call sequence of a test"""

    def __init__(self, seq, frames, fl, init="gt"):
        self.seq, self.frames, self.fl = seq, frames, fl
        set_globals(fl)
        img0, d0 = frames[0]
        self.kf = po.Frame(0, img0, seq.K, fast=fl)
        self.dm = po.DepthMap(seq.w, seq.h, seq.K, fast=fl)
        if init == "gt":
            self.kf.setDepthFromGroundTruth(d0)
            self.dm.initializeFromGTDepth(self.kf)
        else:
            C.CDLL(None).srand(1)                   # DepthMap.cpp:898 draws from glibc rand(): same stream on both sides
            self.dm.initializeRandomly(self.kf)
        self.fr = {0: self.kf}

    def add_frame(self, k, qts, itr=0.0, mask=None, parent=0):
        f = po.Frame(k, self.frames[k][0], self.seq.K, fast=self.fl)
        f.set_thisToParent(qts, self.fr[parent])
        f.L.lsdo_frame_set_initialTrackedResidual(f.ptr, float(itr))
        if mask is not None:
            f.refPixelWasGood(create=True)[:] = mask
        self.fr[k] = f


def _gt_qts(seq, k):
    return np.concatenate([seq.frame_to_ref_qt(k), [1.0]])


# ---- the comparisons: each runs one flavour and hands its observations to `pin` -----------------------------------------
def frame_builders(pin, fl, seq, frames):
    """Frame.cpp:35-54, 491-630, 643-680, 690-767, 245-293, 775-877"""
    set_globals(fl)
    img, d0 = frames[0]
    a = po.Frame(0, img, seq.K, fast=fl)
    a.setDepthFromGroundTruth(d0)
    for lvl in range(5):
        pin.exact(f"image{lvl}", a.image(lvl))
        pin.exact(f"gradients{lvl}", _bits(a.gradients(lvl)))
        pin.exact(f"idepth{lvl}", _bits(a.idepth(lvl)))
        pin.exact(f"idepthVar{lvl}", _bits(a.idepthVar(lvl)))
        K, Ki = a.K(lvl)
        pin.exact(f"K{lvl}", np.asarray(K))
        pin.exact(f"Kinv{lvl}", _bits(np.asarray(Ki)))
    # buildMaxGradients: rows 1 and h-2 read never-written pool memory in the reference (SURVEY App. A-12); interior is defined
    pin.exact("maxGradients", _bits(a.maxGradients(0)[2:-2]))
    pin.exact("numPoints", np.int64(a.L.lsdo_frame_numPoints(a.ptr)))
    pin.exact("meanIdepth", np.float32(a.L.lsdo_frame_meanIdepth(a.ptr)))


def point_cloud(pin, fl, seq, frames):
    """TrackingReference::makePointCloud (TrackingReference.cpp:96-147)"""
    img, d0 = frames[0]
    a = po.Frame(0, img, seq.K, fast=fl)
    a.setDepthFromGroundTruth(d0)
    for lvl in (1, 2, 3, 4):
        pc = a.point_cloud(lvl)
        assert len(pc[0]) > 100
        for i, x in enumerate(pc):
            pin.exact(f"L{lvl}/{i}", _bits(np.ascontiguousarray(x)))


def prepare_for_stereo(pin, fl, seq, frames):
    """Frame::prepareForStereoWith (Frame.cpp:295-317): Sim3 inverse, K*R*s, columns of thisToOther_R"""
    rng = np.random.default_rng(5)
    K = np.ascontiguousarray(seq.K, np.float32).reshape(9)
    fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
    for trial in range(8):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        qts = np.concatenate([q, rng.normal(size=3) * 0.3, [np.exp(rng.normal() * 0.2) if trial else 1.0]])
        kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
        f = po.Frame(3, frames[3][0], seq.K, fast=fl)
        o = np.zeros(30, np.float32)
        f.L.lsdo_ref_prepareForStereoWith(f.ptr, kf.ptr, qts.ctypes.data_as(dp), K.ctypes.data_as(fp), o.ctypes.data_as(fp))
        ref = pin.value(f"trial{trial}", o)
        assert np.array_equal(o.view(np.uint32), ref.view(np.uint32)), (trial, o - ref)


def depthmap_update_sequence(pin, fl, seq, frames):
    """updateKeyframe x6 (1, 2 and 3 reference frames, with and without the tracking mask) -- DepthMap.cpp:111-473,
    1072-1213, 1442-1972, 656-880 and Frame::setDepth, every field of every pixel"""
    s = Side(seq, frames, fl, "gt")
    rng = np.random.default_rng(11)
    w1, h1 = seq.w // 2, seq.h // 2
    groups = [[1], [2, 3], [4], [5, 6, 7], [8], [9]]
    for gi, ks in enumerate(groups):
        for k in ks:
            mask = (rng.random((h1, w1)) > 0.15).astype(np.uint8) if gi % 2 == 0 else None
            s.add_frame(k, _gt_qts(seq, k), itr=0.05 * gi, mask=mask)
        s.dm.updateKeyframe([s.fr[k] for k in ks])
        n = pin.hyp(f"updateKeyframe{ks}", s.dm.current())
        # the keyframe's exported depth (Frame::setDepth + pyramids) as the tracker will read it
        for lvl in range(5):
            pin.exact(f"updateKeyframe{ks}/kf_idepth{lvl}", _bits(s.kf.idepth(lvl)))
            pin.exact(f"updateKeyframe{ks}/kf_idepthVar{lvl}", _bits(s.kf.idepthVar(lvl)))
    assert n > 15000


def depthmap_random_init_every_branch(pin, fl, seq, frames):
    """random hypotheses drive doLineStereo / observeDepthUpdate through their failure, inconsistency and skip branches.
    Only those that depend on the map: under the default motion every search runs along a near-horizontal epipolar line, so
    the y-dominant depth formula, the left and top clips of the search segment, the near-plane clamp and the firstX and
    rescale gates never run here (tests/test_ref_pin_motions.py reaches them with other camera motions)"""
    s = Side(seq, frames, fl, "random")
    pin.hyp("initializeRandomly", s.dm.current())
    for k in (4, 6, 8, 10, 12):
        s.add_frame(k, _gt_qts(seq, k))
        s.dm.updateKeyframe([s.fr[k]])
        n = pin.hyp(f"updateKeyframe[{k}]", s.dm.current())
    assert n > 5000


def depthmap_individual_passes(pin, fl, seq, frames):
    """observeDepth, regularizeDepthMapFillHoles, regularizeDepthMap<true/false> one by one (private members of the
    reference class called as they are)"""
    s = Side(seq, frames, fl, "gt")
    s.add_frame(2, _gt_qts(seq, 2))
    s.add_frame(3, _gt_qts(seq, 3))
    s.dm.observeDepth([s.fr[2], s.fr[3]])
    pin.hyp("observeDepth", s.dm.current())
    s.dm.regularizeFillHoles()
    pin.hyp("fillHoles", s.dm.current())
    s.dm.regularize(False, 24)
    pin.hyp("regularize<false>", s.dm.current())
    s.dm.regularize(True, 24)
    pin.hyp("regularize<true>", s.dm.current())
    pin.exact("integral", np.ascontiguousarray(s.dm.integral()))


def create_keyframe_and_finalize(pin, fl, seq, frames_in):
    """finalizeKeyFrame + createKeyFrame (propagateDepth with the tracking mask, 2x regularise, fill holes, rescale,
    pose scale) -- DepthMap.cpp:475-653, 1222-1327, 1363-1395; then mapping continues on the new keyframe, including with
    frames that were tracked on the PREVIOUS keyframe (:1085-1099).
    The scene is rescaled so that keyframe 0 already has mean inverse depth 1, as every keyframe after the first has in a real
    run: doLineStereo only accepts a reference frame whose depth ratio to the keyframe is within 0.7..1.4 (:119 `rescaleFactor`),
    so with a 2x scale jump between keyframes the off-parent frames would be rejected pixel by pixel and test nothing."""
    d0 = frames_in[0][1]
    sc = float(np.mean(1.0 / d0[d0 > 0]))
    frames = {k: (frames_in[k][0], (frames_in[k][1] * sc).astype(np.float32)) for k in range(13)}

    def qts(k, ref=0):
        q = seq.frame_to_ref_qt(k, ref=ref).copy()
        q[4:7] *= sc
        return np.concatenate([q, [1.0]])
    s = Side(seq, frames, fl, "gt")
    rng = np.random.default_rng(3)
    w1, h1 = seq.w // 2, seq.h // 2
    for k in (1, 2, 3):
        s.add_frame(k, qts(k), itr=0.1)
        s.dm.updateKeyframe([s.fr[k]])
    pin.hyp("before finalize", s.dm.current())
    s.dm.finalizeKeyFrame()
    pin.hyp("finalizeKeyFrame", s.dm.current())
    mask = (rng.random((h1, w1)) > 0.1).astype(np.uint8)
    s.add_frame(9, qts(9), itr=0.1, mask=mask)
    s.dm.createKeyFrame(s.fr[9])
    pin.hyp("createKeyFrame", s.dm.current())
    pa = s.fr[9].thisToParent()                                   # rescaled Sim3 (DepthMap.cpp:1305)
    pb = pin.value("thisToParent9", pa)
    assert np.allclose(pa, pb, rtol=0, atol=1e-12), pa - pb
    assert 0.8 < pa[7] < 1.25
    # frames tracked on the PREVIOUS keyframe, mapped on the new one: refToKf comes from the chained absolute poses (:1099), and the
    # tracking-mask gate of :245 / :322 is off for them
    for k in (4, 5):
        s.add_frame(k, qts(k), itr=0.07, mask=mask, parent=0)
    before = s.dm.current().copy()
    s.dm.updateKeyframe([s.fr[4], s.fr[5]])
    after = s.dm.current()
    n = pin.hyp("updateKeyframe with frames tracked on the previous keyframe", after)
    both = (before["isValid"] != 0) & (after["isValid"] != 0)
    assert n > 10000 and int((before["idepth"][both] != after["idepth"][both]).sum()) > 2000     # they did observe
    # frames tracked on the NEW keyframe
    for k in (10, 11):
        q = qts(k, ref=9)
        q[4:7] /= pa[7]                                           # the new keyframe's units
        s.add_frame(k, q, itr=0.1, parent=9)
        s.dm.updateKeyframe([s.fr[k]])
        pin.hyp(f"updateKeyframe on new keyframe [{k}]", s.dm.current())
    q = qts(12, ref=9)
    q[4:7] /= pa[7]
    s.add_frame(12, q, itr=0.1, parent=9)
    s.add_frame(6, qts(6), itr=0.05, mask=mask, parent=0)
    s.dm.updateKeyframe([s.fr[6], s.fr[12]])                       # mixed parents in one call
    pin.hyp("updateKeyframe with mixed tracking parents", s.dm.current())


def se3_single_evaluation(pin, fl, seq, frames):
    """calcResidualAndBuffers + calcWeightsAndResidual + calculateWarpUpdate (SE3Tracker.cpp:885-1029, 749-790,
    1258-1299, LGSX.h:184-402), the reference's private members called directly"""
    set_globals(fl)
    kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
    kf.setDepthFromGroundTruth(frames[0][1])
    f = po.Frame(3, frames[3][0], seq.K, fast=fl)
    inv = np.zeros(7)
    g = np.ascontiguousarray(seq.frame_to_ref_qt(3), np.float64)
    po.lib(False).lsdo_se3d_inverse(g.ctypes.data_as(C.POINTER(C.c_double)), inv.ctypes.data_as(C.POINTER(C.c_double)))
    pose = inv.astype(np.float32)
    names = ("meanUnweightedRes", "meanWeightedRes", "lsError", "meanRes", "affine_a_lastIt", "affine_b_lastIt")
    for lvl in (4, 3, 2, 1):
        ra = po.se3_eval(kf, f, lvl, pose, 1.0, 0.0, po.default_track_settings(fl), write_mask=(lvl == 1))
        counts = np.array([ra.warpedSize, ra.goodCount, ra.badCount, ra.pointUsage], np.float64)
        cb = pin.value(f"L{lvl}/counts", counts)
        assert counts[0] == cb[0] > 50
        assert np.array_equal(counts[1:], cb[1:]), (lvl, counts, cb)
        x = np.array([getattr(ra, n) for n in names], np.float64)
        y = pin.value(f"L{lvl}/scalars", x)
        for n, xi, yi in zip(names, x, y):
            assert abs(xi - yi) <= 2e-6 * max(abs(yi), 1.0), (lvl, n, xi, yi)
        A, B = np.array(ra.A), pin.value(f"L{lvl}/A", np.array(ra.A))
        assert np.abs(A - B).max() <= 2e-6 * np.abs(B).max(), lvl
        b, bb = np.array(ra.b), pin.value(f"L{lvl}/b", np.array(ra.b))
        assert np.abs(b - bb).max() <= 2e-6 * np.abs(bb).max() + 1e-9, lvl
    pin.exact("mask", f.refPixelWasGood(create=False) != 0)


def _se3_track_sequence(pin, fl, seq, frames, exact):
    """SE3Tracker::trackFrame over a tracked + mapped sequence: pose, every reported statistic, the good-mask"""
    set_globals(fl, useSSE=1) if fl is True else set_globals(fl)
    kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
    kf.setDepthFromGroundTruth(frames[0][1])
    dm = po.DepthMap(seq.w, seq.h, seq.K, fast=fl)
    dm.initializeFromGTDepth(kf)
    st = po.default_track_settings(fl)
    last, keep = IDENT, []
    for k in range(1, 7):
        f = po.Frame(k, frames[k][0], seq.K, fast=fl)
        keep.append(f)
        kf.L.lsdo_frame_set_depthHasBeenUpdatedFlag(kf.ptr, 0)
        r = po.se3_track(kf, f, last, st)
        last = np.array(r.frameToRef_qt)
        x = np.array([r.lastResidual, r.pointUsage, r.lastGoodCount, r.lastBadCount, r.lastMeanRes,
                      r.affineEstimation_a, r.affineEstimation_b, r.diverged, r.trackingWasGood, r.initialTrackedResidual], np.float64)
        mask = f.refPixelWasGood(create=False).copy() != 0
        pose_b, y = pin.value(f"f{k}/pose", last), pin.value(f"f{k}/stats", x)
        if exact:
            # scalar path, strict IEEE on both sides: the restatement reproduces the reference-compiled tracker BIT FOR BIT
            # (pose as doubles, every statistic, the mask) -- same sequential sums, same LDLT, same Sophus arithmetic
            assert np.array_equal(last, pose_b), (k, last - pose_b)
            assert np.array_equal(x.astype(np.float32), y.astype(np.float32)), (k, x, y)
            pin.exact(f"f{k}/mask", mask)
        else:
            # timing flavours: both are -O3 builds with FMA contraction left to the compiler, so only fp32 round-off agreement
            dt, ang = pose_err(last, pose_b)
            assert dt <= 1e-4 and ang <= 1e-6, (k, dt, ang)
            for i in (0, 1, 5, 9):
                assert abs(x[i] - y[i]) <= 2e-4 * max(abs(y[i]), 1.0), (k, i, x[i], y[i])
            assert abs(x[4] - y[4]) <= 1e-2 and abs(x[6] - y[6]) <= 1e-2    # mean signed residual, affine b (grey levels): fp32 cancellation
            assert abs(x[2] - y[2]) <= 3 and abs(x[3] - y[3]) <= 3, (k, x[2:4], y[2:4])       # good / bad counts
            assert x[7] == y[7] and x[8] == y[8]
            mb = np.unpackbits(pin.value(f"f{k}/mask_bits", np.packbits(mask)))[: mask.size].reshape(mask.shape) != 0
            assert (mask != mb).mean() <= 1e-3
        dm.updateKeyframe([f])


def se3_track_scalar(pin, fl, seq, frames):
    _se3_track_sequence(pin, fl, seq, frames, exact=True)


def se3_track_sse(pin, fl, seq, frames):
    """the oracle's restatement of the SSE loops (SE3Tracker.cpp:492-575, 1033-1130, LGSX.h:205-386) against the stock
    ENABLE_SSE build of the reference"""
    _se3_track_sequence(pin, fl, seq, frames, exact=False)


def bench_loop_with_keyframe_changes(pin, fl, seq, frames, n_frames=26):
    """the loop bench.py and the full-size GPU tests run (oracle/cpu_stream.py: track, map, forced finalizeKeyFrame +
    createKeyFrame every 10 frames) over frames 1..n_frames-1: every pose equal as doubles, final map identical"""
    from oracle.cpu_stream import CpuStream
    set_globals(fl)
    cs = CpuStream(seq, fl, kf_every=10)
    cs.init_gt(0, *frames[0])
    for k in range(1, n_frames):
        cs.step(k, frames[k][0])
    assert cs.kf_changes == list(range(10, n_frames, 10))
    poses = np.array(cs.poses)
    assert np.array_equal(poses, pin.value("poses", poses))
    pin.hyp(f"after {n_frames - 1} frames and {len(cs.kf_changes)} keyframe changes", cs.dm.current())


# case -> (function, C-restatement flavour, reference-compiled flavour it is pinned to)
CASES = {
    "frame_builders": (frame_builders, False, "ref"),
    "point_cloud": (point_cloud, False, "ref"),
    "prepare_for_stereo": (prepare_for_stereo, False, "ref"),
    "depthmap_update_sequence": (depthmap_update_sequence, False, "ref"),
    "depthmap_random_init_every_branch": (depthmap_random_init_every_branch, False, "ref"),
    "depthmap_individual_passes": (depthmap_individual_passes, False, "ref"),
    "create_keyframe_and_finalize": (create_keyframe_and_finalize, False, "ref"),
    "se3_single_evaluation": (se3_single_evaluation, False, "ref"),
    "se3_track_scalar": (se3_track_scalar, False, "ref"),
    "se3_track_sse": (se3_track_sse, True, "ref_sse"),
    "bench_loop_with_keyframe_changes": (bench_loop_with_keyframe_changes, False, "ref"),
}


def record(seq, frames):
    """runs every case on the reference-compiled library (needs oracle/_ref); returns the arrays of the golden file"""
    out = {}
    for name, (fn, _, ref_fl) in CASES.items():
        pin = Pin(name)
        fn(pin, ref_fl, seq, frames)
        out.update(pin.rec)
    # the reference's own gap between its two code paths (test_sse_vs_scalar_gap_of_the_reference_itself)
    for fl in ("ref", "ref_sse"):
        po.set_globals(fl)
        kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
        kf.setDepthFromGroundTruth(frames[0][1])
        f = po.Frame(3, frames[3][0], seq.K, fast=fl)
        out[f"sse_gap/{fl}"] = np.array(po.se3_track(kf, f, IDENT, po.default_track_settings(fl)).frameToRef_qt)
    return out


def _run(case, seq, frames):
    fn, fl, _ = CASES[case]
    fn(_check(case), fl, seq, frames)


def test_frame_builders_bit_exact(seq_small, frames_small):
    _run("frame_builders", seq_small, frames_small)


def test_point_cloud_bit_exact(seq_small, frames_small):
    _run("point_cloud", seq_small, frames_small)


def test_prepare_for_stereo_bit_exact(seq_small, frames_small):
    _run("prepare_for_stereo", seq_small, frames_small)


def test_depthmap_update_sequence_bit_exact(seq_small, frames_small):
    _run("depthmap_update_sequence", seq_small, frames_small)


def test_depthmap_random_init_every_branch_bit_exact(seq_small, frames_small):
    _run("depthmap_random_init_every_branch", seq_small, frames_small)


def test_depthmap_individual_passes_bit_exact(seq_small, frames_small):
    _run("depthmap_individual_passes", seq_small, frames_small)


def test_create_keyframe_and_finalize_bit_exact(seq_small, frames_small):
    _run("create_keyframe_and_finalize", seq_small, frames_small)


def test_se3_single_evaluation_matches_reference_compiled(seq_small, frames_small):
    _run("se3_single_evaluation", seq_small, frames_small)


@pytest.mark.parametrize("pair", ["scalar", "sse"])
def test_se3_track_matches_reference_compiled(seq_small, frames_small, pair):
    _run(f"se3_track_{pair}", seq_small, frames_small)


def test_sse_vs_scalar_gap_of_the_reference_itself(seq_small, frames_small):
    """The stock build defines ENABLE_SSE (CMakeLists.txt:37-43): _mm_rcp_ps weights, N mod 4 points dropped.  The recorded
    poses of the reference's two code paths on the same input show how far they are apart (documented in DESIGN.md section 2):
    the scalar path is the parity target of the CUDA kernels, the SSE path the timing baseline.  The oracle's scalar path
    reproduces the recorded scalar pose exactly and its SSE restatement the recorded SSE pose within 1e-4."""
    g = np.load(GOLD)
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
    _run("bench_loop_with_keyframe_changes", seq_small, frames_small)
