"""The case library of the oracle's pin: each case function runs one call sequence on one flavour of the oracle -- the hand-written
C restatement (oracle/lsd_oracle.c) or the reference's own sources compiled unmodified by oracle/ref_build.py into oracle/_ref/ --
and hands its observations to a Pin, which records them (to write a golden file) or checks them against the record.

tests/test_ref_pin.py runs the cases at the reference's default run-time settings on the default stream,
tests/test_ref_pin_globals.py under the settings of SETS, tests/test_ref_pin_motions.py under the camera motions of
tests/motions.py (with two more cases only those reach), tests/test_ref_pin_sim3.py runs the Sim3 tracker and the permaRef
path on keyframes the mapper finished, under every motion, tests/test_ref_pin_photometry.py runs cases under the exposure
schedules of tests/photometry.py, tests/test_ref_pin_cameras.py the cases that read K through the cameras of tests/cameras.py,
tests/test_ref_pin_scenes.py the depth-map, tracker and cloud cases on the scenes of tests/scenes.py;
tests/golden/make_golden*.py record each of them."""
import contextlib
import ctypes as C
import hashlib
import os

import numpy as np

from oracle import pyoracle as po
from tests import cameras, motions, photometry, scenes
from tests.util import IDENT, pose_err

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = os.path.join(GOLDEN, "ref_pin_320x240.npz")

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
# SETS below holds others (the ranges of cfg/LSDParams.cfg:13-34).
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
    rescale gates never run here (the motion pin reaches them with other camera motions)"""
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


def se3_single_evaluation(pin, fl, seq, frames, affines=((1.0, 0.0),)):
    """calcResidualAndBuffers + calcWeightsAndResidual + calculateWarpUpdate (SE3Tracker.cpp:885-1029, 749-790,
    1258-1299, LGSX.h:184-402), the reference's private members called directly, at the ground-truth pose of frame 3 and each
    affine estimate (a, b) of `affines` (the first one's observations carry no prefix)"""
    set_globals(fl)
    kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
    kf.setDepthFromGroundTruth(frames[0][1])
    f = po.Frame(3, frames[3][0], seq.K, fast=fl)
    inv = np.zeros(7)
    g = np.ascontiguousarray(seq.frame_to_ref_qt(3), np.float64)
    po.lib(False).lsdo_se3d_inverse(g.ctypes.data_as(C.POINTER(C.c_double)), inv.ctypes.data_as(C.POINTER(C.c_double)))
    pose = inv.astype(np.float32)
    for i, (a, b) in enumerate(affines):
        _se3_eval_levels(pin, fl, kf, f, pose, a, b, "" if i == 0 else f"a{a:g}_b{b:g}/")


def _se3_eval_levels(pin, fl, kf, f, pose, a, b, tag):
    names = ("meanUnweightedRes", "meanWeightedRes", "lsError", "meanRes", "affine_a_lastIt", "affine_b_lastIt")
    for lvl in (4, 3, 2, 1):
        ra = po.se3_eval(kf, f, lvl, pose, a, b, po.default_track_settings(fl), write_mask=(lvl == 1))
        counts = np.array([ra.warpedSize, ra.goodCount, ra.badCount, ra.pointUsage], np.float64)
        cb = pin.value(f"{tag}L{lvl}/counts", counts)
        assert counts[0] == cb[0] > 50
        assert np.array_equal(counts[1:], cb[1:]), (lvl, counts, cb)
        x = np.array([getattr(ra, n) for n in names], np.float64)
        y = pin.value(f"{tag}L{lvl}/scalars", x)
        for n, xi, yi in zip(names, x, y):       # no good point: the mean over the good points is 0/0 on both sides
            assert abs(xi - yi) <= 2e-6 * max(abs(yi), 1.0) or (np.isnan(xi) and np.isnan(yi)), (lvl, n, xi, yi)
        A, B = np.array(ra.A), pin.value(f"{tag}L{lvl}/A", np.array(ra.A))
        assert np.abs(A - B).max() <= 2e-6 * np.abs(B).max(), lvl
        bv, bb = np.array(ra.b), pin.value(f"{tag}L{lvl}/b", np.array(ra.b))
        assert np.abs(bv - bb).max() <= 2e-6 * np.abs(bb).max() + 1e-9, lvl
    pin.exact(f"{tag}mask", f.refPixelWasGood(create=False) != 0)


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
    """runs every case on the reference-compiled library (needs oracle/_ref); returns the arrays of ref_pin_320x240.npz"""
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


def run(case, seq, frames):
    """one case on the C restatement, checked against ref_pin_320x240.npz"""
    fn, fl, _ = CASES[case]
    fn(_check(case), fl, seq, frames)


# ---- non-default run-time settings (util/settings.cpp:80-88, cfg/LSDParams.cfg:13-34) --------------------------------------
GOLD_GLOBALS = os.path.join(GOLDEN, "ref_pin_globals_320x240.npz")

DEPTH = ("depthmap_update_sequence", "depthmap_random_init_every_branch", "depthmap_individual_passes",
         "create_keyframe_and_finalize")
TRACK = ("se3_single_evaluation", "se3_track_scalar")
LOOP = ("bench_loop_with_keyframe_changes",)

# set name -> (settings, cases that read them)
SETS = {
    "allowNegativeIdepths=0": (dict(allowNegativeIdepths=0), DEPTH + LOOP),
    "useSubpixelStereo=0": (dict(useSubpixelStereo=0), DEPTH + LOOP),
    "minUseGrad=2.5": (dict(minUseGrad=2.5), ("frame_builders",) + DEPTH + TRACK + LOOP),
    "minUseGrad=10": (dict(minUseGrad=10.0), ("frame_builders",) + DEPTH + TRACK + LOOP),
    "cameraPixelNoise2=1": (dict(cameraPixelNoise2=1.0), DEPTH + TRACK + LOOP),
    "cameraPixelNoise2=36": (dict(cameraPixelNoise2=36.0), DEPTH + TRACK + LOOP),
    "depthSmoothingFactor=0": (dict(depthSmoothingFactor=0.0), DEPTH + LOOP),
    "depthSmoothingFactor=3": (dict(depthSmoothingFactor=3.0), DEPTH + LOOP),
    "useAffineLightningEstimation=0": (dict(useAffineLightningEstimation=0), TRACK + LOOP),
    "combined": (dict(minUseGrad=7.5, cameraPixelNoise2=9.0, depthSmoothingFactor=2.0, allowNegativeIdepths=0,
                      useSubpixelStereo=0, useAffineLightningEstimation=0), ("frame_builders",) + DEPTH + TRACK + LOOP),
}
SETTINGS_PAIRS = [(s, c) for s, (_, cases) in SETS.items() for c in cases]


def run_under_settings(set_name, case, gold, seq, frames):
    """runs one case under one set on the C restatement (gold = the record) or on the reference-compiled library (gold = None);
    returns the case's Pin.  The libraries are back at the defaults afterwards."""
    g, _ = SETS[set_name]
    fn, fl, ref_fl = CASES[case]
    fl = ref_fl if gold is None else fl
    p = Pin(f"{set_name}/{case}", gold)
    try:
        with settings(**g):
            fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_globals(seq, frames):
    """every (set, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_globals_320x240.npz"""
    out = {}
    for s, c in SETTINGS_PAIRS:
        out.update(run_under_settings(s, c, None, seq, frames).rec)
    return out


# ---- camera motions (tests/motions.py) ---------------------------------------------------------------------------------------
GOLD_MOTIONS = os.path.join(GOLDEN, "ref_pin_motions_320x240.npz")

WIDE_BASELINE_FRAME = 40
PROPAGATION_FRAME = 8


def wide_baseline(p, fl, seq, frames):
    """updateKeyframe with one frame far from the keyframe, on ground-truth depth and poses"""
    s = Side(seq, frames, fl, "gt")
    k = WIDE_BASELINE_FRAME
    s.add_frame(k, _gt_qts(seq, k))
    s.dm.updateKeyframe([s.fr[k]])
    assert p.hyp(f"updateKeyframe[{k}]", s.dm.current()) > 10000


def propagation_collisions(p, fl, seq, frames):
    """propagateDepth of a random map: its sources disagree about depth, so under a motion along the optical axis many land on one
    pixel at inconsistent depths (DepthMap.cpp:588-601); validity 200 makes every merge exceed the cap of :626"""
    k = PROPAGATION_FRAME
    mask = (np.random.default_rng(8).random((seq.h // 2, seq.w // 2)) > 0.15).astype(np.uint8)
    for what, m, validity in (("no mask", None, None), ("mask", mask, None), ("validity 200", None, 200)):
        s = Side(seq, frames, fl, "random")
        if validity is not None:
            cur = s.dm.current().copy()
            cur["validity_counter"][cur["isValid"] != 0] = validity
            s.dm.set_current(cur)
        s.add_frame(k, _gt_qts(seq, k), mask=m)
        s.dm.propagateDepth(s.fr[k])
        assert p.hyp(f"propagateDepth[{k}] {what}", s.dm.current()) > 5000




# the case functions above that read the camera motion
GEOMETRY = ("prepare_for_stereo", "depthmap_update_sequence", "depthmap_random_init_every_branch", "depthmap_individual_passes",
            "create_keyframe_and_finalize", "se3_single_evaluation", "se3_track_scalar", "bench_loop_with_keyframe_changes")
# case -> (function, C-restatement flavour, reference-compiled flavour), as CASES
MOTION_CASES = {c: CASES[c] for c in GEOMETRY}
MOTION_CASES["wide_baseline"] = (wide_baseline, False, "ref")
MOTION_CASES["propagation_collisions"] = (propagation_collisions, False, "ref")
ONLY = {"wide_baseline": ("forward", "backward"), "propagation_collisions": ("forward", "backward")}
MOTION_PAIRS = [(m, c) for m in motions.MOTIONS for c in MOTION_CASES if m in ONLY.get(c, (m,))]


def run_under_motion(motion, case, gold):
    """runs one case under one motion on the C restatement (gold = the record) or on the reference-compiled library
    (gold = None); returns the case's Pin"""
    fn, fl, ref_fl = MOTION_CASES[case]
    fl = ref_fl if gold is None else fl
    seq, frames = motions.stream(motion)
    p = Pin(f"{motion}/{case}", gold)
    try:
        fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_motions():
    """every (motion, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_motions_320x240.npz"""
    out = {}
    for m, c in MOTION_PAIRS:
        out.update(run_under_motion(m, c, None).rec)
    return out


# ---- Sim3 and permaRef on keyframes the mapper finished (tests/test_ref_pin_sim3.py) ----------------------------------------
GOLD_SIM3 = os.path.join(GOLDEN, "ref_pin_sim3_320x240.npz")

MAPPED_KF_EVERY = 5
MAPPED_FRAMES = 16              # keyframe changes at frames 5, 10 and 15: keyframes 0, 5 and 10 finished, 15 active
PERMA_FRAME = 12                # a frame that is not a keyframe, for trackFrameOnPermaref
SIM3_DT, SIM3_SCALE = (0.01, -0.005, 0.004), 1.02       # the perturbation of util.sim3_init
AB = ((1.0, 0.0), (0.97, 1.5))
SIM3_SETTINGS = dict(var_weight=2.5, huber_d=1.5)        # the one non-default tracker setting set (class defaults: 1, 3)
OVERLAP_SIGMA = (0.2, 0.2, 0.3, 0.05, 0.05, 0.05)         # util.check_perma_overlap's random poses

# (motion, reference keyframe, frame keyframe, startLevel, finalLevel) of the trackFrameSim3 calls whose lastDepthResidual is
# ill-conditioned in the final pose.  Under `vertical`, 0 -> 10 over levels 3..2 rejects every level-2 step, so the reported
# depth residual is that of the last accepted level-3 step (722 depth terms).  A change of the final translation by 7e-6
# (relative, a tenth of what tree-ordered sums move the device's pose by elsewhere) moves that residual by up to 4.2e-3 relative
# with no point changing its pixel or its depth status (other calls: 1e-5 to 4e-5, e.g. the reverse pair or the default
# motion's 0 -> 10); the device's pose lies 7.2e-6 from the exact-affine-sum twin and its
# depth residual 4.5e-3.  Pivoting the device's 7x7 solve does not change either.  For these calls lastDepthResidual is held to
# the reference tolerance (2e-2) against the twin as well; every other field keeps its tolerance.
POSE_SENSITIVE_DEPTH_RESIDUAL = {("vertical", 0, 10, 3, 2)}
SENSITIVE_TRANSLATION = 7e-6


def depth_residual_sensitivity(m, ref, fr, lo, hi, n=50):
    """-> (largest relative change of the oracle's level-`lo` meanD, largest change of its depth / warped term counts) when the
    final translation of the exact-affine-sum trackFrameSim3 moves by SENSITIVE_TRANSLATION (relative) in n seeded directions"""
    init = m.frame_to_ref(ref, fr)
    set_globals(False, exactAffineSums=1)
    try:
        ex = po.sim3_track(m.of[ref], m.of[fr], init, lo, hi)
    finally:
        set_globals(False)
    a, b = ex.affineEstimation_a, ex.affineEstimation_b

    def ev(q):
        return po.sim3_eval(m.of[ref], m.of[fr], lo, _qts_op("lsdo_sim3d_inverse", 8, q), a, b)
    base = ev(np.array(ex.frameToRef_qts))
    rng = np.random.default_rng(0)
    dmax, cmax = 0.0, 0
    for _ in range(n):
        q = np.array(ex.frameToRef_qts)
        d = rng.normal(size=3)
        q[4:7] += d * SENSITIVE_TRANSLATION * np.linalg.norm(q[4:7]) / np.linalg.norm(d)
        e = ev(q)
        dmax = max(dmax, abs(e.meanD - base.meanD) / base.meanD)
        cmax = max(cmax, abs(e.numTermsD - base.numTermsD), abs(e.warpedSize - base.warpedSize))
    return dmax, cmax


def _qts_op(fn, n, *args):
    out = np.zeros(n, np.float64)
    arrs = [np.ascontiguousarray(a, np.float64) for a in args]
    getattr(po.lib(False), fn)(*[po._dp(a) for a in arrs], po._dp(out))
    return out


class Mapped:
    """oracle/cpu_stream.py's loop on one flavour over frames 0..MAPPED_FRAMES-1 with a keyframe every MAPPED_KF_EVERY frames:
    the finished keyframes' Frames (`of`: id -> Frame), the active keyframe's id and hypotheses, and each keyframe's
    camToWorld chained in double by the C restatement's Sophus from the C restatement's thisToParent -- on both flavours, so
    that both start the Sim3 tracker from the same doubles (each flavour's own thisToParent is pinned by _kf_depth)"""

    def __init__(self, fl, seq, frames):
        from oracle.cpu_stream import CpuStream
        set_globals(fl)
        cs = CpuStream(seq, fl, kf_every=MAPPED_KF_EVERY, keep_keyframes=True)
        cs.init_gt(0, *frames[0])
        for k in range(1, MAPPED_FRAMES):
            cs.step(k, frames[k][0])
        self.seq, self.frames = seq, frames
        self.of = {f.id: f for f in cs.finished}
        self.kfs = list(self.of)
        self.active, self.active_hyp = cs.kf.id, cs.dm.current().copy()
        self.thisToParent = {f.id: f.thisToParent() for f in cs.finished + [cs.kf]}
        if fl is not False:                 # the Sim3 starts are computed once, from the C restatement's chain, for both flavours
            self.c2w = mapped(False, seq, frames).c2w
            return
        self.c2w = {}
        last = np.array([0, 0, 0, 1, 0, 0, 0, 1], np.float64)
        for f in cs.finished + [cs.kf]:
            if f.id:
                last = _qts_op("lsdo_sim3d_mul", 8, last, self.thisToParent[f.id])
            self.c2w[f.id] = last

    def frame_to_ref(self, ref, fr, perturb=True):
        q = _qts_op("lsdo_sim3d_mul", 8, _qts_op("lsdo_sim3d_inverse", 8, self.c2w[ref]), self.c2w[fr])
        if perturb:
            q[4:7] += SIM3_DT
            q[7] *= SIM3_SCALE
        return q

    def ref_to_frame(self, ref, fr, perturb=True):
        return _qts_op("lsdo_sim3d_inverse", 8, self.frame_to_ref(ref, fr, perturb))

    def pairs(self):
        return [(a, b) for a in self.kfs for b in self.kfs if a != b]


_mapped: dict = {}


def mapped(fl, seq, frames):
    """the Mapped run of (flavour, sequence), made once per process"""
    key = (fl, id(seq))
    if key not in _mapped:
        _mapped[key] = (seq, Mapped(fl, seq, frames))
    return _mapped[key][1]


def sim3_eval_fields(r):
    """what a Sim3 evaluation returns, as one float64 row: A (49), b (7), num_constraints, numTermsD, numTermsP, warpedSize,
    sumResD, sumResP, mean, meanD, meanP, pointUsage, affine_a_lastIt, affine_b_lastIt"""
    return np.concatenate([np.array(r.A, np.float64), np.array(r.b, np.float64),
                           [r.num_constraints, r.numTermsD, r.numTermsP, r.warpedSize, r.sumResD, r.sumResP, r.mean, r.meanD,
                            r.meanP, r.pointUsage, r.affine_a_lastIt, r.affine_b_lastIt]])


def sim3_track_fields(r):
    """what trackFrameSim3 returns that the reference exports: the pose (8 doubles), the Hessian (49), lastResidual,
    lastDepthResidual, lastPhotometricResidual, pointUsage, affineEstimation_a, affineEstimation_b, diverged"""
    return np.concatenate([np.array(r.frameToRef_qts), np.array(r.lastSim3Hessian, np.float64),
                           [r.lastResidual, r.lastDepthResidual, r.lastPhotometricResidual, r.pointUsage,
                            r.affineEstimation_a, r.affineEstimation_b, r.diverged]])


def perma_track_fields(r):
    """what trackFrameOnPermaref returns that the reference exports: referenceToFrame (7 doubles), pointUsage, lastGoodCount,
    lastBadCount, lastMeanRes, lastResidual, affineEstimation_a, affineEstimation_b, diverged, trackingWasGood"""
    return np.concatenate([np.array(r.frameToRef_qt), [r.pointUsage, r.lastGoodCount, r.lastBadCount, r.lastMeanRes,
                                                         r.lastResidual, r.affineEstimation_a, r.affineEstimation_b,
                                                         r.diverged, r.trackingWasGood]])


def _same_pose(pin, what, x, n):
    """a pose read back from Sophus' non-unit quaternion (its normalisation differs from the restatement's division in the
    last bits: 1e-12, as tests/test_oracle_kats.py allows), every other field bit for bit as float32 / float64"""
    y = pin.value(what, x)
    assert np.allclose(x[:n], y[:n], rtol=0, atol=1e-12), (what, x[:n] - y[:n])
    assert np.array_equal(x[n:], y[n:]), (what, np.flatnonzero(x[n:] != y[n:]), x[n:], y[n:])


def _kf_depth(pin, m):
    """each finished keyframe's pyramids and its rescaled thisToParent: the input every Sim3 / permaRef call reads"""
    for k, f in m.of.items():
        for lvl in range(po.LEVELS):
            pin.exact(f"kf{k}/idepth{lvl}", _bits(f.idepth(lvl)))
            pin.exact(f"kf{k}/idepthVar{lvl}", _bits(f.idepthVar(lvl)))
        _same_pose(pin, f"kf{k}/thisToParent", m.thisToParent[k], 8)


def _eval(pin, what, ref, fr, lvl, r2f, a, b, st):
    r = po.sim3_eval(ref, fr, lvl, r2f, a, b, settings=st)
    x = sim3_eval_fields(r)
    y = pin.value(what, x)
    assert np.array_equal(x, y), (what, np.flatnonzero(x != y), x[x != y], y[x != y])
    return r


def sim3_eval_mapped(pin, fl, seq, frames):
    """calcSim3Buffers + calcSim3WeightsAndResidual + calcSim3LGS (Sim3Tracker.cpp:414-607, 748-856, 992-1047) for every ordered
    pair of finished keyframes, levels 4-1, from the chained pose with and without util.sim3_init's perturbation, at two affine
    estimates; once more on one pair under SIM3_SETTINGS.  Bit for bit."""
    m = mapped(fl, seq, frames)
    set_globals(fl)
    _kf_depth(pin, m)
    st = po.default_track_settings(fl, main_tracker=False)
    for ref, fr in m.pairs():
        for perturb in (True, False):
            r2f = m.ref_to_frame(ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in AB:
                    r = _eval(pin, f"{ref}->{fr}/p{int(perturb)}/L{lvl}/a{a}", m.of[ref], m.of[fr], lvl, r2f, a, b, st)
                    assert r.warpedSize > 10
    for k, v in SIM3_SETTINGS.items():
        setattr(st, k, v)
    ref, fr = m.kfs[0], m.kfs[-1]
    r2f = m.ref_to_frame(ref, fr)
    for lvl in (4, 3, 2, 1):
        a, b = AB[lvl % 2]
        _eval(pin, f"settings/{ref}->{fr}/L{lvl}", m.of[ref], m.of[fr], lvl, r2f, a, b, st)


def sim3_track_mapped(pin, fl, seq, frames):
    """Sim3Tracker::trackFrameSim3 (Sim3Tracker.cpp:149-382) for every ordered pair of finished keyframes, levels 4..1 and 3..2,
    from the perturbed chained pose"""
    m = mapped(fl, seq, frames)
    set_globals(fl)
    for ref, fr in m.pairs():
        init = m.frame_to_ref(ref, fr)
        for lo, hi in ((4, 1), (3, 2)):
            r = po.sim3_track(m.of[ref], m.of[fr], init, lo, hi)
            _same_pose(pin, f"{ref}->{fr}/{lo}{hi}", sim3_track_fields(r), 8)


def overlap_poses(kfs):
    """util.check_perma_overlap's five random refToFrame poses per keyframe (seed 3)"""
    rng = np.random.default_rng(3)
    return {k: [_qts_op("lsdo_se3d_exp", 7, rng.normal(0, OVERLAP_SIGMA)) for _ in range(5)] for k in kfs}


def perma_gt(m, k, frame):
    """refToFrame of `frame` on keyframe k from ground truth, the translation in the keyframe's map units"""
    gt = m.seq.frame_to_ref_qt(frame, ref=k)
    gt[4:7] /= m.c2w[k][7]
    return _qts_op("lsdo_se3d_inverse", 7, gt)


def _perma(pin, fl, m, prs, tag=""):
    """checkPermaRefOverlap (SE3Tracker.cpp:121-157) at overlap_poses and at the ground-truth pose of PERMA_FRAME, and
    trackFrameOnPermaref (:162-272) of PERMA_FRAME from ground truth and from identity, on each snapshot of prs"""
    f = po.Frame(PERMA_FRAME, m.frames[PERMA_FRAME][0], m.seq.K, fast=fl)
    poses = overlap_poses(prs)
    for k, pr in prs.items():
        gt = perma_gt(m, k, PERMA_FRAME)
        ov = np.array([pr.overlap(q) for q in poses[k] + [gt]], np.float32)
        pin.exact(f"{tag}kf{k}/overlap", _bits(ov))
        pin.value(f"{tag}kf{k}/overlap_values", ov)
        for name, init in (("gt", gt), ("identity", IDENT)):
            _same_pose(pin, f"{tag}kf{k}/track_{name}", perma_track_fields(pr.track(f, init)), 7)


def perma_mapped(pin, fl, seq, frames):
    """Frame::setPermaRef of each finished keyframe (the snapshot bit for bit), then the overlap check and the tracking on it"""
    m = mapped(fl, seq, frames)
    set_globals(fl)
    prs = {}
    for k, f in m.of.items():
        prs[k] = pr = po.PermaRef(f)
        assert pr.n > 30
        pin.exact(f"kf{k}/snapshot_pos", _bits(pr.pos[:pr.n]))
        pin.exact(f"kf{k}/snapshot_colvar", _bits(pr.colvar[:pr.n]))
    _perma(pin, fl, m, prs)


def adversarial_edit(hyp, rng):
    """A real map with a few hundred pixels edited to the value edges of Frame::setDepth, the idepth pyramid and
    makePointCloud:
      * for every pyramid level L = 1..4, aligned 2^L x 2^L blocks whose left half holds +a and right half -a with one
        variance: the level-(L-1) pixels of the block are exact negatives of each other, so the inverse-variance weighted
        sum is exactly 0 at level L and the pyramid gives 1 / (ivarSum / 0) = 0 there (Frame.cpp:862-864); in a third
        block per level the negative side is one ulp larger, which leaves a tiny idepth (a point very far away);
      * idepths in [-0.05, 0) (kept by the gate of Frame.cpp:219; the floats at and below -0.05 are dropped by it);
      * idepth exactly 0.0 and -0.0 with a valid variance (skipped as points, TrackingReference.cpp:133);
      * runs of five neighbouring pixels with variances 1e-7, 1e-5, 1e-3, 1e-1, 1e1.
    Only valid pixels are read or written, so the uninitialised fields of the reference's invalid pixels do not matter."""
    hyp = hyp.copy()
    h, w = hyp.shape
    free = np.zeros((h, w), bool)                    # interior pixels no edit has touched yet
    free[2:-2, 2:-2] = True
    typical = np.float32(np.median(hyp["idepth_smoothed"][hyp["isValid"] > 0]))

    def put(ys, xs, idepth, var=None):
        hyp["isValid"][ys, xs] = 1
        hyp["blacklisted"][ys, xs] = 0
        for f in ("idepth", "idepth_smoothed"):
            hyp[f][ys, xs] = idepth
        if var is not None:
            for f in ("idepth_var", "idepth_var_smoothed"):
                hyp[f][ys, xs] = var
        free[ys, xs] = False

    for lvl in range(po.LEVELS - 1, 0, -1):
        s = 1 << lvl
        by, bx = h // s, w // s
        ok = free[:by * s, :bx * s].reshape(by, s, bx, s).all(axis=(1, 3)).ravel()
        for j, i in enumerate(rng.choice(np.flatnonzero(ok), 3, replace=False)):
            y0, x0 = (int(i) // bx) * s, (int(i) % bx) * s
            a = np.float32(rng.uniform(0.005, 0.05))
            b = -a if j < 2 else -np.nextafter(a, np.float32(1))
            var = np.float32(10.0 ** rng.uniform(-4, -1))
            put(slice(y0, y0 + s), slice(x0, x0 + s // 2), a, var)
            put(slice(y0, y0 + s), slice(x0 + s // 2, x0 + s), b, var)

    def pick(n):
        ys, xs = np.nonzero(free & (hyp["isValid"] > 0))
        i = rng.choice(ys.size, n, replace=False)
        return ys[i], xs[i]

    ys, xs = pick(64)
    neg = rng.uniform(-0.0499, -1e-4, 64).astype(np.float32)
    neg[:4] = [np.nextafter(np.float32(-0.05), np.float32(0)), np.float32(-1e-6), np.float32(-0.05), np.float32(-0.06)]
    put(ys, xs, neg)
    ys, xs = pick(32)
    put(ys, xs, np.where(np.arange(32) % 2 == 0, np.float32(0.0), np.float32(-0.0)).astype(np.float32))
    runs = 0
    for y, x in zip(*pick(80)):
        x = min(max(x - x % 2, 2), w - 8)
        if runs < 40 and free[y, x:x + 5].all():
            put(y, slice(x, x + 5), typical, np.float32([1e-7, 1e-5, 1e-3, 1e-1, 1e1]))
            runs += 1
    assert runs == 40
    return hyp


def set_depth(frame, hyp):
    """Frame::setDepth (Frame.cpp:199-243) of a hypothesis map"""
    h = np.ascontiguousarray(hyp, po.HYP_DTYPE)
    frame.L.lsdo_frame_setDepth(frame.ptr, h.ctypes.data_as(C.POINTER(po.Hyp)))


def adversarial_keyframe(fl, m):
    """the active keyframe's image with adversarial_edit (seed 7) of its hypotheses loaded through Frame::setDepth"""
    hyp = adversarial_edit(m.active_hyp, np.random.default_rng(7))
    f = po.Frame(m.active, m.frames[m.active][0], m.seq.K, fast=fl)
    set_depth(f, hyp)
    return f, hyp


def adversarial_map(pin, fl, seq, frames):
    """adversarial_keyframe: its pyramids, then permaRef and Sim3 on it (both directions against the last finished keyframe, the
    active keyframe's chained pose).  Points with negative idepth lie behind the camera and can warp into the image mirrored;
    the reference has no Wz > 0 test in calcSim3Buffers or checkPermaRefOverlap."""
    m = mapped(fl, seq, frames)
    set_globals(fl)
    okf, _ = adversarial_keyframe(fl, m)
    for lvl in range(po.LEVELS):
        pin.exact(f"idepth{lvl}", _bits(okf.idepth(lvl)))
        pin.exact(f"idepthVar{lvl}", _bits(okf.idepthVar(lvl)))
    idepth0, valid0 = okf.idepth(0), okf.idepthVar(0) > 0
    assert ((idepth0 < 0) & valid0).sum() >= 50 and ((idepth0 == 0) & valid0).sum() >= 32
    for lvl in range(1, po.LEVELS):                  # the cancelled blocks reach every level
        assert ((okf.idepth(lvl) == 0) & (okf.idepthVar(lvl) > 0)).any(), lvl
    pr = po.PermaRef(okf)
    pin.exact("snapshot_pos", _bits(pr.pos[:pr.n]))
    pin.exact("snapshot_colvar", _bits(pr.colvar[:pr.n]))
    _perma(pin, fl, m, {m.active: pr})
    of = dict(m.of)
    of[m.active] = okf
    other = m.kfs[-1]
    st = po.default_track_settings(fl, main_tracker=False)
    for ref, fr in ((m.active, other), (other, m.active)):
        r2f = m.ref_to_frame(ref, fr)
        for lvl in range(po.LEVELS):
            for a, b in AB:
                _eval(pin, f"{ref}->{fr}/L{lvl}/a{a}", of[ref], of[fr], lvl, r2f, a, b, st)
        r = po.sim3_track(of[ref], of[fr], m.frame_to_ref(ref, fr), 4, 1)
        _same_pose(pin, f"{ref}->{fr}/track", sim3_track_fields(r), 8)


# case -> (function, C-restatement flavour, reference-compiled flavour), as CASES
SIM3_CASES = {
    "sim3_eval_mapped": (sim3_eval_mapped, False, "ref"),
    "sim3_track_mapped": (sim3_track_mapped, False, "ref"),
    "perma_mapped": (perma_mapped, False, "ref"),
    "adversarial_map": (adversarial_map, False, "ref"),
}
SIM3_ONLY = {"adversarial_map": (motions.DEFAULT, "forward")}
SIM3_MOTIONS = (motions.DEFAULT,) + tuple(motions.MOTIONS)
SIM3_PAIRS = [(m, c) for m in SIM3_MOTIONS for c in SIM3_CASES if m in SIM3_ONLY.get(c, (m,))]


def run_sim3(motion, case, gold):
    """runs one case under one motion on the C restatement (gold = the record) or on the reference-compiled library
    (gold = None); returns the case's Pin"""
    fn, fl, ref_fl = SIM3_CASES[case]
    fl = ref_fl if gold is None else fl
    seq, frames = motions.stream(motion)
    p = Pin(f"{motion}/{case}", gold)
    try:
        fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_sim3():
    """every (motion, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_sim3_320x240.npz"""
    out = {}
    for m, c in SIM3_PAIRS:
        out.update(run_sim3(m, c, None).rec)
    return out


def sim3_eval_result(row) -> po.Sim3EvalResult:
    """the recorded sim3_eval_fields row as the struct the checks of tests/util.py read"""
    r = po.Sim3EvalResult()
    r.A[:], r.b[:] = [float(x) for x in row[:49]], [float(x) for x in row[49:56]]
    (r.num_constraints, r.numTermsD, r.numTermsP, r.warpedSize) = (int(x) for x in row[56:60])
    (r.sumResD, r.sumResP, r.mean, r.meanD, r.meanP, r.pointUsage, r.affine_a_lastIt, r.affine_b_lastIt) = row[60:68]
    return r


def sim3_track_result(row, calls) -> po.Sim3Result:
    """the recorded sim3_track_fields row as a Sim3Result, with the LM call counters (locals in the reference) of `calls`"""
    r = po.Sim3Result()
    r.frameToRef_qts[:], r.lastSim3Hessian[:] = [float(x) for x in row[:8]], [float(x) for x in row[8:57]]
    (r.lastResidual, r.lastDepthResidual, r.lastPhotometricResidual, r.pointUsage, r.affineEstimation_a,
     r.affineEstimation_b) = row[57:63]
    r.diverged = int(row[63])
    r.numCalcResidualCalls[:], r.numCalcWarpUpdateCalls[:] = list(calls.numCalcResidualCalls), list(calls.numCalcWarpUpdateCalls)
    return r


def perma_track_result(row, calls) -> po.TrackResult:
    """the recorded perma_track_fields row as a TrackResult, with the LM call counters (not counted in the reference) of `calls`"""
    r = po.TrackResult()
    r.frameToRef_qt[:] = [float(x) for x in row[:7]]
    (r.pointUsage, r.lastGoodCount, r.lastBadCount, r.lastMeanRes, r.lastResidual, r.affineEstimation_a,
     r.affineEstimation_b) = row[7:14]
    r.diverged, r.trackingWasGood = int(row[14]), int(row[15])
    r.numCalcResidualCalls[:], r.numCalcWarpUpdateCalls[:] = list(calls.numCalcResidualCalls), list(calls.numCalcWarpUpdateCalls)
    return r


# ---- exposure changes (tests/photometry.py) -----------------------------------------------------------------------------------
GOLD_PHOTOMETRY = os.path.join(GOLDEN, "ref_pin_photometry_320x240.npz")

FAR_AFFINE = (1.4, -20.0)       # an affine estimate far from every schedule's truth at frame 3


def eval_affines(seq):
    """se3_single_evaluation's affine estimates under an exposure schedule: the identity, frame 3's true (a, b), FAR_AFFINE"""
    return ((1.0, 0.0), tuple(round(float(x), 6) for x in seq.affine(3)), FAR_AFFINE)


def se3_eval_exposure(pin, fl, seq, frames):
    """se3_single_evaluation at the affine estimates of eval_affines: counts, statistics, normal equations and the level-1 mask"""
    se3_single_evaluation(pin, fl, seq, frames, affines=eval_affines(seq))


def propagation_exposure(pin, fl, seq, frames):
    """propagateDepth of the ground-truth map to frame PROPAGATION_FRAME at its true pose, without a tracking mask (the colour
    check of DepthMap.cpp:559-569 compares raw intensities, so a change of exposure drops sources) and with one (:550-555)"""
    k = PROPAGATION_FRAME
    mask = (np.random.default_rng(8).random((seq.h // 2, seq.w // 2)) > 0.15).astype(np.uint8)
    for what, m in (("no mask", None), ("mask", mask)):
        s = Side(seq, frames, fl, "gt")
        s.add_frame(k, _gt_qts(seq, k), mask=m)
        s.dm.propagateDepth(s.fr[k])
        assert pin.hyp(f"propagateDepth[{k}] {what}", s.dm.current()) > 5000


# case -> (function, C-restatement flavour, reference-compiled flavour), as CASES
PHOTOMETRY_CASES = {c: CASES[c] for c in DEPTH}
PHOTOMETRY_CASES["propagation_exposure"] = (propagation_exposure, False, "ref")
PHOTOMETRY_CASES["se3_eval_exposure"] = (se3_eval_exposure, False, "ref")
PHOTOMETRY_CASES["se3_track_scalar"] = CASES["se3_track_scalar"]
PHOTOMETRY_CASES["bench_loop_with_keyframe_changes"] = CASES["bench_loop_with_keyframe_changes"]
for _c in ("sim3_eval_mapped", "sim3_track_mapped", "perma_mapped"):
    PHOTOMETRY_CASES[_c] = SIM3_CASES[_c]
PHOTOMETRY_PAIRS = [(s, c) for s in photometry.SCHEDULES for c in PHOTOMETRY_CASES]
# the depth-map counters (pyoracle.BRANCHES) that no depth-map case of tests/test_ref_pin.py reaches on the default stream at the
# default settings: the colour check of propagateDepth needs two frames that disagree in brightness, the negative-idepth -2 of
# doLineStereo needs allowNegativeIdepths = 0
UNREACHED_BY_DEFAULT_PHOTOMETRIC = ("stereo_negative", "prop_color")


def run_under_exposure(schedule, case, gold):
    """runs one case under one exposure schedule on the C restatement (gold = the record) or on the reference-compiled library
    (gold = None); returns the case's Pin"""
    fn, fl, ref_fl = PHOTOMETRY_CASES[case]
    fl = ref_fl if gold is None else fl
    seq, frames = photometry.stream(schedule)
    p = Pin(f"{schedule}/{case}", gold)
    try:
        fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_photometry():
    """every (schedule, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_photometry_320x240.npz"""
    out = {}
    for s, c in PHOTOMETRY_PAIRS:
        out.update(run_under_exposure(s, c, None).rec)
    return out


# ---- cameras other than synth.pinhole_K (tests/cameras.py) -------------------------------------------------------------------
GOLD_CAMERAS = os.path.join(GOLDEN, "ref_pin_cameras_320x240.npz")

# case -> (function, C-restatement flavour, reference-compiled flavour), as CASES: every case that reads K
CAMERA_CASES = {c: CASES[c] for c in ("frame_builders", "point_cloud") + GEOMETRY}
CAMERA_CASES.update(SIM3_CASES)
CAMERA_STREAMS = cameras.SMALL + (cameras.VERTICAL,)
CAMERA_ONLY = {c: cameras.SMALL for c in CAMERA_CASES if c not in DEPTH}          # the vertical stream: the depth-map cases
CAMERA_ONLY.update({c: ("offset", "general") for c in SIM3_CASES})
# (camera, reference keyframe, frame keyframe, startLevel, finalLevel) of a trackFrameSim3 call whose pose the reference's
# sequential fp32 sums of the normal equations move by a large part of POSE_TOL (tests/test_ref_pin_cameras.py)
SIM3_SUM_SENSITIVE = ("offset", 10, 5, 4, 1)
CAMERA_PAIRS = [(cam, c) for cam in CAMERA_STREAMS for c in CAMERA_CASES if cam in CAMERA_ONLY.get(c, (cam,))]


def run_under_camera(camera, case, gold, seq=None):
    """runs one case through one camera on the C restatement (gold = the record) or on the reference-compiled library
    (gold = None); returns the case's Pin.  seq: another sequence that the case reads K from instead, with the camera's images"""
    fn, fl, ref_fl = CAMERA_CASES[case]
    fl = ref_fl if gold is None else fl
    cam_seq, frames = cameras.stream(camera)
    p = Pin(f"{camera}/{case}", gold)
    try:
        fn(p, fl, cam_seq if seq is None else seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_cameras():
    """every (camera, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_cameras_320x240.npz"""
    out = {}
    for cam, c in CAMERA_PAIRS:
        out.update(run_under_camera(cam, c, None).rec)
    return out


# ---- scenes other than the smooth height field (tests/scenes.py) -------------------------------------------------------------
GOLD_SCENES = os.path.join(GOLDEN, "ref_pin_scenes_320x240.npz")

EMPTY_SIM3_KF = 6               # the textured keyframe empty_keyframe pairs the blank one with in the Sim3 tracker
EMPTY_RAND_DRAWS = 16           # rand() values drawn after initializeRandomly: the state the call leaves


def propagate_from_gt(pin, fl, seq, frames):
    """propagateDepth of the ground-truth map to frame PROPAGATION_FRAME, without and with a tracking mask: on a scene with a
    near object its sources land behind and in front of each other (DepthMap.cpp:588-601) and uncover background whose colour
    disagrees (:559-569)"""
    propagation_exposure(pin, fl, seq, frames)


def _bits_equal(pin, what, x, n_pose=0):
    """x against the record bit for bit, NaN payloads included; a leading pose of n_pose doubles to 1e-12 (_same_pose)"""
    x = np.ascontiguousarray(x, np.float64)
    y = np.asarray(pin.value(what, x), np.float64)
    assert x.shape == y.shape and np.allclose(x[:n_pose], y[:n_pose], rtol=0, atol=1e-12), (what, x[:n_pose], y[:n_pose])
    assert np.array_equal(x[n_pose:].view(np.uint64), y[n_pose:].view(np.uint64)), (what, x, y)


def empty_keyframe(pin, fl, seq, frames):
    """a keyframe with (almost) no texture: initializeRandomly (the map it leaves and the rand() values after it), updateKeyframe,
    fill-holes and both regularisers on that map; SE3 evaluation and trackFrame, makePointCloud, setPermaRef and
    trackFrameOnPermaref, Sim3 evaluation and trackFrameSim3 against a textured ground-truth keyframe of the default scene, on
    ground-truth depth.  Every value bit for bit, NaN included: an empty sum is 0 and a mean over no point 0/0 in the reference"""
    s = Side(seq, frames, fl, "random")
    rnd = np.array([C.CDLL(None).rand() for _ in range(EMPTY_RAND_DRAWS)], np.int64)
    pin.exact("rand_after", rnd)
    pin.value("selected", np.int64(pin.hyp("initializeRandomly", s.dm.current())))
    for k in (2, 3):
        s.add_frame(k, _gt_qts(seq, k))
    s.dm.updateKeyframe([s.fr[2], s.fr[3]])
    pin.hyp("updateKeyframe", s.dm.current())
    s.dm.regularizeFillHoles()
    pin.hyp("fillHoles", s.dm.current())
    for occl in (False, True):
        s.dm.regularize(occl, 24)
        pin.hyp(f"regularize<{str(occl).lower()}>", s.dm.current())

    set_globals(fl)
    kf = po.Frame(0, frames[0][0], seq.K, fast=fl)
    kf.setDepthFromGroundTruth(frames[0][1])
    f = po.Frame(3, frames[3][0], seq.K, fast=fl)
    inv = np.zeros(7)
    g = np.ascontiguousarray(seq.frame_to_ref_qt(3), np.float64)
    po.lib(False).lsdo_se3d_inverse(g.ctypes.data_as(C.POINTER(C.c_double)), inv.ctypes.data_as(C.POINTER(C.c_double)))
    names = ("warpedSize", "goodCount", "badCount", "pointUsage", "meanUnweightedRes", "meanWeightedRes", "lsError", "meanRes",
             "affine_a_lastIt", "affine_b_lastIt")
    for lvl in (4, 3, 2, 1):
        r = po.se3_eval(kf, f, lvl, inv.astype(np.float32), 1.0, 0.0, po.default_track_settings(fl), write_mask=(lvl == 1))
        _bits_equal(pin, f"se3_eval/L{lvl}", [getattr(r, n) for n in names] + list(r.A) + list(r.b))
    pin.exact("se3_eval/mask", f.refPixelWasGood(create=False) != 0)
    r = po.se3_track(kf, po.Frame(3, frames[3][0], seq.K, fast=fl), IDENT, po.default_track_settings(fl))
    x = list(r.frameToRef_qt) + [r.lastResidual, r.pointUsage, r.lastGoodCount, r.lastBadCount, r.lastMeanRes,
                                 r.affineEstimation_a, r.affineEstimation_b, r.diverged, r.trackingWasGood]
    if not r.diverged:                  # a diverged trackFrame returns before it writes the frame's value (SE3Tracker.cpp:326, :482)
        x.append(r.initialTrackedResidual)
    _bits_equal(pin, "se3_track", x, 7)
    for lvl in (1, 2, 3, 4):
        pin.value(f"point_cloud/L{lvl}", np.int64(len(kf.point_cloud(lvl)[0])))

    pr = po.PermaRef(kf)
    pin.value("perma/n", np.int64(pr.n))
    fp = po.Frame(PERMA_FRAME, frames[PERMA_FRAME][0], seq.K, fast=fl)
    gt = _qts_op("lsdo_se3d_inverse", 7, seq.frame_to_ref_qt(PERMA_FRAME))
    _bits_equal(pin, "perma/overlap", [pr.overlap(gt)])
    for name, init in (("gt", gt), ("identity", IDENT)):
        _bits_equal(pin, f"perma/track_{name}", perma_track_fields(pr.track(fp, init)), 7)

    from lsd_slam_b200 import synth
    other = synth.Sequence(seq.w, seq.h, seed=motions.SEED)
    img6, d6 = other.render(EMPTY_SIM3_KF)
    tex = po.Frame(EMPTY_SIM3_KF, img6, seq.K, fast=fl)
    tex.setDepthFromGroundTruth(d6)
    fr_to_ref = np.concatenate([seq.frame_to_ref_qt(EMPTY_SIM3_KF), [1.0]])
    fr_to_ref[4:7] += SIM3_DT
    fr_to_ref[7] *= SIM3_SCALE
    st = po.default_track_settings(fl, main_tracker=False)
    for ref, fr, q, tag in ((kf, tex, fr_to_ref, "blank->tex"), (tex, kf, _qts_op("lsdo_sim3d_inverse", 8, fr_to_ref), "tex->blank")):
        r2f = _qts_op("lsdo_sim3d_inverse", 8, q)
        for lvl in (4, 3, 2, 1):
            _bits_equal(pin, f"sim3_eval/{tag}/L{lvl}", sim3_eval_fields(po.sim3_eval(ref, fr, lvl, r2f, 1.0, 0.0, settings=st)))
        r = po.sim3_track(ref, fr, q, 4, 1)
        x = sim3_track_fields(r)
        if r.diverged:                  # left at level 4 (Sim3Tracker.cpp:186-190): the reference never wrote lastSim3Hessian
            x = np.concatenate([x[:8], x[57:]])
        _bits_equal(pin, f"sim3_track/{tag}", x, 8)


# case -> (function, C-restatement flavour, reference-compiled flavour), as CASES
SCENE_CASES = {c: CASES[c] for c in DEPTH + TRACK + ("point_cloud",)}
SCENE_CASES["propagate_from_gt"] = (propagate_from_gt, False, "ref")
SCENE_CASES.update({c: SIM3_CASES[c] for c in ("sim3_eval_mapped", "sim3_track_mapped", "perma_mapped")})
SCENE_CASES["empty_keyframe"] = (empty_keyframe, False, "ref")
TEXTURED = ("occluder", "posts", "stripes", "flat")
SCENE_ONLY = {c: TEXTURED for c in SCENE_CASES}
SCENE_ONLY["empty_keyframe"] = ("blank", "blank_const")
SCENE_PAIRS = [(sc, c) for sc in scenes.NAMES for c in SCENE_CASES if sc in SCENE_ONLY[c]]


def run_under_scene(scene, case, gold):
    """runs one case on one scene on the C restatement (gold = the record) or on the reference-compiled library (gold = None);
    returns the case's Pin"""
    fn, fl, ref_fl = SCENE_CASES[case]
    fl = ref_fl if gold is None else fl
    seq, frames = scenes.stream(scene)
    p = Pin(f"{scene}/{case}", gold)
    try:
        fn(p, fl, seq, frames)
    finally:
        po.set_globals(fl)
    return p


def record_scenes():
    """every (scene, case) on the reference-compiled library (needs oracle/_ref): the arrays of ref_pin_scenes_320x240.npz"""
    out = {}
    for sc, c in SCENE_PAIRS:
        out.update(run_under_scene(sc, c, None).rec)
    return out
