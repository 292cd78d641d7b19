"""The Sim3 tracker (csrc/sim3.cuh) and the permaRef path (csrc/perma.cuh) on keyframes the device's own mapper has finished.

test_gpu_sim3.py and test_gpu_perma.py give their keyframes ground-truth depth: one variance everywhere
(Frame::setDepthFromGroundTruth, Frame.cpp:245-273), kept by the idepth pyramid at every level (Frame.cpp:865), and scales
between keyframes of about 1.  With that input a kernel that reads the wrong variance (the reference point's `s` vs the
frame's `sv`, Sim3Tracker.cpp:527-542, 762-835; the snapshot's colorAndVarData, Frame.cpp:149-174) computes the same
numbers.  Here the keyframes come from a GpuStream run (updateKeyframe / finalizeKeyFrame / createKeyFrame): a semi-dense map
with variances over orders of magnitude, and keyframes rescaled by createKeyFrame (DepthMap.cpp:1285-1304).  Each finished
keyframe is mirrored on the oracle through Frame::setDepth (Frame.cpp:199-243) from the device's level-0 planes, and the last
test loads a map edited to hold the value edges of a real map on both sides."""
import ctypes as C

import numpy as np
import pytest

from lsd_slam_b200 import abi, synth
from lsd_slam_b200.stream import IDENT, GpuStream, sim3_mul_qts
from tests.util import (POSE_TOL, check_perma_overlap, check_perma_track, check_sim3_eval, check_sim3_track, oracle_sim3_track,
                        se3_inverse, sim3_err, sim3_inverse)

pytestmark = pytest.mark.gpu

KF_EVERY = 5
N_FRAMES = 16                   # keyframe changes at frames 5, 10 and 15: keyframes 0, 5 and 10 finished, 15 active
PERMA_FRAME = 12                # a frame that is not a keyframe, for trackFrameOnPermaref
DT = (0.01, -0.005, 0.004)      # the perturbation of util.sim3_init
AB = ((1.0, 0.0), (0.97, 1.5))


def _set_depth(oracle, frame, hyp):
    h = np.ascontiguousarray(hyp, oracle.HYP_DTYPE)
    frame.L.lsdo_frame_setDepth(frame.ptr, h.ctypes.data_as(C.POINTER(oracle.Hyp)))


def _mirror(oracle, ctx, seq, kf, img):
    """an oracle Frame of the same image given the device keyframe's level-0 plane through Frame::setDepth: valid pixels
    (var > 0) are >= -0.05 there, so setDepth keeps them as they are and turns every other pixel into -1 / -1 again"""
    idepth, var = ctx.download(kf, abi.BUF_IDEPTH, 0), ctx.download(kf, abi.BUF_IDEPTH_VAR, 0)
    hyp = np.zeros(idepth.shape, oracle.HYP_DTYPE)
    hyp["isValid"] = var > 0
    hyp["idepth"] = hyp["idepth_smoothed"] = idepth
    hyp["idepth_var"] = hyp["idepth_var_smoothed"] = var
    f = oracle.Frame(kf, img, seq.K)
    _set_depth(oracle, f, hyp)
    return f


def _pyramid_mismatches(ctx, kf, of):
    """(level, plane) pairs whose bits differ between the device keyframe and its oracle Frame"""
    bad = []
    for lvl in range(abi.LEVELS):
        for name, buf, plane in (("idepth", abi.BUF_IDEPTH, of.idepth), ("idepthVar", abi.BUF_IDEPTH_VAR, of.idepthVar)):
            if not np.array_equal(ctx.download(kf, buf, lvl).view(np.uint32), plane(lvl).view(np.uint32)):
                bad.append((lvl, name))
    return bad


class MappedRun:
    """A GpuStream of the seed-1234 sequence with its finished keyframes resident and an oracle mirror of each.
    After every keyframe change it compares the pyramids of every resident keyframe with the oracle (`checks`)."""

    def __init__(self, oracle, w, h):
        self.seq = seq = synth.Sequence(w, h, seed=1234)
        self.ctx = ctx = abi.Context(w, h, seq.K, max_frames=12)
        self.gs = gs = GpuStream(ctx, kf_every=KF_EVERY, keep_keyframes=True)
        self.images = {}
        img, d = seq.render(0)
        self.images[0] = img
        gs.init_gt(0, img, d)
        self.of, self.checks = {}, []
        for k in range(1, N_FRAMES):
            self.images[k] = seq.render(k)[0]
            change = gs.next_is_keyframe_change()
            gs.step(k, self.images[k])
            if not change:
                continue
            for kf in gs.keyframe_ids[:-1]:           # finished: mirrored once, then re-checked after every later change
                if kf not in self.of:
                    self.of[kf] = _mirror(oracle, ctx, seq, kf, self.images[kf])
                self.checks.append((k, kf, _pyramid_mismatches(ctx, kf, self.of[kf])))
            active = gs.keyframe_ids[-1]              # the new keyframe as createKeyFrame left it
            self.checks.append((k, active, _pyramid_mismatches(ctx, active, _mirror(oracle, ctx, seq, active, self.images[active]))))
        self.kfs = gs.keyframe_ids[:-1]
        self.active = gs.keyframe_ids[-1]
        self.active_hyp = gs.map.current()            # the active keyframe's hypotheses (DepthMap::currentDepthMap)

    def frame_to_ref(self, oracle, ref, fr, perturb=True):
        """the relative Sim3 SlamSystem starts from: reference->getScaledCamToWorld().inverse() * frame->getScaledCamToWorld()
        (scale ratio of the two keyframes included), with util.sim3_init's perturbation of translation and scale"""
        c2w = dict(zip(self.gs.keyframe_ids, self.gs.keyframe_cam_to_world))
        q = sim3_mul_qts(sim3_inverse(oracle, c2w[ref]), c2w[fr])
        if perturb:
            q[4:7] += DT
            q[7] *= 1.02
        return q

    def ref_to_frame(self, oracle, ref, fr, perturb=True):
        return sim3_inverse(oracle, self.frame_to_ref(oracle, ref, fr, perturb))

    def pairs(self):
        return [(a, b) for a in self.kfs for b in self.kfs if a != b]

    def close(self):
        self.ctx.close()


@pytest.fixture(scope="module")
def mapped(oracle):
    run = MappedRun(oracle, 320, 240)
    yield run
    run.close()


def test_mapped_keyframes_mirror_bit_exact(mapped):
    """every resident keyframe's idepth / idepthVar pyramid (levels 0-4) equals the oracle's Frame::setDepth of the same
    level-0 plane, and a finished keyframe stays so through the later map swaps and createKeyFrame calls of the run"""
    assert len(mapped.kfs) >= 3
    assert [kf for _, kf, _ in mapped.checks].count(mapped.kfs[0]) >= 3
    bad = [(k, kf, m) for k, kf, m in mapped.checks if m]
    assert not bad, bad
    ctx = mapped.ctx
    spread = []
    for kf in mapped.kfs:                             # what this file is about: a semi-dense map, no variance shared by all
        var = ctx.download(kf, abi.BUF_IDEPTH_VAR, 0)
        v = var[var > 0]
        assert 0.2 < v.size / var.size < 0.7 and np.unique(v).size > 100, (kf, v.size / var.size, np.unique(v).size)
        spread.append(v.max() / v.min())
    assert max(spread) > 30, spread
    scales = [q[7] for q in mapped.gs.keyframe_cam_to_world]
    assert max(scales) / min(scales) > 1.2, scales       # createKeyFrame rescales every new keyframe


def test_sim3_eval_on_mapped_keyframes(mapped, oracle):
    trk = abi.Sim3Tracker(mapped.ctx)
    of = mapped.of
    n_no_depth = 0
    for ref, fr in mapped.pairs():
        for perturb in (True, False):
            r2f = mapped.ref_to_frame(oracle, ref, fr, perturb)
            for lvl in (4, 3, 2, 1):
                for a, b in AB:
                    got = trk.eval(ref, fr, lvl, r2f, a, b)
                    want = oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b)
                    assert want.warpedSize > 10, (ref, fr, lvl)
                    check_sim3_eval(got, want)
                    n_no_depth += want.numTermsD < want.numTermsP      # warped onto frame pixels without depth (sim3.cuh:116-117)
    assert n_no_depth > 0


def test_sim3_eval_settings_on_mapped_keyframes(mapped, oracle):
    """var_weight and huber_d other than their defaults (1, 3) reach the kernel's weights"""
    trk = abi.Sim3Tracker(mapped.ctx)
    st = oracle.default_track_settings(main_tracker=False)
    for s in (trk.settings, st):
        s.var_weight, s.huber_d = 2.5, 1.5
    for ref, fr in mapped.pairs():
        r2f = mapped.ref_to_frame(oracle, ref, fr)
        for lvl in (4, 3, 2, 1):
            a, b = AB[lvl % 2]
            check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), oracle.sim3_eval(mapped.of[ref], mapped.of[fr], lvl, r2f, a, b, settings=st))


def test_track_frame_sim3_on_mapped_keyframes(mapped, oracle):
    trk = abi.Sim3Tracker(mapped.ctx)
    n_converged = 0
    for ref, fr in mapped.pairs():
        init = mapped.frame_to_ref(oracle, ref, fr)
        for lo, hi in ((4, 1), (3, 2)):
            est = trk.trackFrameSim3(ref, fr, init, lo, hi)
            want, exact = oracle_sim3_track(oracle, mapped.of[ref], mapped.of[fr], init, lo, hi)
            check_sim3_track(trk.last, want)
            check_sim3_track(trk.last, exact, res_tol=5e-4)
            assert np.array_equal(est, np.array(trk.last.frameToRef_qts))
            n_converged += not want.diverged
    assert n_converged >= len(mapped.pairs())


def _check_batch(run, oracle):
    trk = abi.Sim3Tracker(run.ctx)
    pairs = run.pairs()
    inits = np.array([run.frame_to_ref(oracle, ref, fr) for ref, fr in pairs])
    res = trk.trackFrameSim3Batch([p[0] for p in pairs], [p[1] for p in pairs], inits, 4, 1)
    for (ref, fr), init, r in zip(pairs, inits, res):
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        assert bytes(trk.last) == bytes(r)
        check_sim3_track(r, oracle.sim3_track(run.of[ref], run.of[fr], init, 4, 1))


def test_track_frame_sim3_batch_on_mapped_keyframes(mapped, oracle):
    _check_batch(mapped, oracle)


def test_track_frame_sim3_batch_on_mapped_keyframes_640x480(oracle):
    run = MappedRun(oracle, 640, 480)
    try:
        assert len(run.kfs) >= 3 and not [c for c in run.checks if c[2]]
        _check_batch(run, oracle)
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
    ctx, seq = mapped.ctx, mapped.seq
    se3 = abi.SE3Tracker(ctx)
    prs = {}
    for k in mapped.kfs:
        prs[k] = oracle.PermaRef(mapped.of[k])
        assert se3.setPermaRef(k) == prs[k].n > 30
    want = check_perma_overlap(se3, oracle, prs, np.random.default_rng(3))
    assert want.min() < 0.9 < want.max()

    # trackFrameOnPermaref for a frame that is not a keyframe, from its ground-truth pose (translation in the keyframe's map
    # units: the chain's scale of the keyframe) and from identity
    img = seq.render(PERMA_FRAME)[0]
    ctx.upload(PERMA_FRAME, img)
    of = oracle.Frame(PERMA_FRAME, img, seq.K)
    scale = dict(zip(mapped.gs.keyframe_ids, [q[7] for q in mapped.gs.keyframe_cam_to_world]))
    ids, inits = [], []
    for k in prs:
        gt = seq.frame_to_ref_qt(PERMA_FRAME, ref=k)
        gt[4:7] /= scale[k]
        gt_inv = se3_inverse(oracle, gt)
        for init in (gt_inv, IDENT):
            ids.append(k)
            inits.append(init)
    res = se3.trackFrameOnPermaref(ids, PERMA_FRAME, np.array(inits))
    n_good = sum(check_perma_track(g, prs[k].track(of, init)) for k, init, g in zip(ids, inits, res))
    assert n_good >= 2
    ctx.release(PERMA_FRAME)


def _adversarial(hyp, rng):
    """A real map with a few hundred pixels edited to the value edges of Frame::setDepth, the idepth pyramid and
    makePointCloud:
      * for every pyramid level L = 1..4, aligned 2^L x 2^L blocks whose left half holds +a and right half -a with one
        variance: the level-(L-1) pixels of the block are exact negatives of each other, so the inverse-variance weighted
        sum is exactly 0 at level L and the pyramid gives 1 / (ivarSum / 0) = 0 there (Frame.cpp:862-864); in a third
        block per level the negative side is one ulp larger, which leaves a tiny idepth (a point very far away);
      * idepths in [-0.05, 0) (kept by the gate of Frame.cpp:219; the floats at and below -0.05 are dropped by it);
      * idepth exactly 0.0 and -0.0 with a valid variance (skipped as points, TrackingReference.cpp:133);
      * runs of five neighbouring pixels with variances 1e-7, 1e-5, 1e-3, 1e-1, 1e1."""
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

    for lvl in range(abi.LEVELS - 1, 0, -1):
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


def test_adversarial_map_edges(mapped, oracle):
    """the edited map of the active keyframe loaded on both sides (DepthMap setHypotheses + Frame::setDepth): pyramids,
    permaRef and Sim3 on it.  Points with negative idepth lie behind the camera and can warp into the image mirrored; the
    reference has no Wz > 0 test in calcSim3Buffers or checkPermaRefOverlap, and neither have the kernels."""
    ctx, seq = mapped.ctx, mapped.seq
    kf, other = mapped.active, mapped.kfs[-1]
    hyp = _adversarial(mapped.active_hyp, np.random.default_rng(7))
    mapped.gs.map.setHypotheses(kf, hyp, do_set_depth=True)
    okf = oracle.Frame(kf, mapped.images[kf], seq.K)
    _set_depth(oracle, okf, hyp)
    assert not _pyramid_mismatches(ctx, kf, okf)
    idepth0, valid0 = okf.idepth(0), okf.idepthVar(0) > 0
    assert ((idepth0 < 0) & valid0).sum() >= 50 and ((idepth0 == 0) & valid0).sum() >= 32
    for lvl in range(1, abi.LEVELS):                  # the cancelled blocks reach every level
        assert ((okf.idepth(lvl) == 0) & (okf.idepthVar(lvl) > 0)).any(), lvl

    se3 = abi.SE3Tracker(ctx)
    pr = oracle.PermaRef(okf)
    assert se3.setPermaRef(kf) == pr.n
    check_perma_overlap(se3, oracle, {kf: pr}, np.random.default_rng(5))

    of = dict(mapped.of)
    of[kf] = okf
    trk = abi.Sim3Tracker(ctx)
    for ref, fr in ((kf, other), (other, kf)):
        r2f = mapped.ref_to_frame(oracle, ref, fr)
        for lvl in range(abi.LEVELS):
            for a, b in AB:
                check_sim3_eval(trk.eval(ref, fr, lvl, r2f, a, b), oracle.sim3_eval(of[ref], of[fr], lvl, r2f, a, b))
        init = mapped.frame_to_ref(oracle, ref, fr)
        trk.trackFrameSim3(ref, fr, init, 4, 1)
        want, exact = oracle_sim3_track(oracle, of[ref], of[fr], init)
        assert trk.diverged == bool(want.diverged)
        if not want.diverged:
            check_sim3_track(trk.last, want)
            check_sim3_track(trk.last, exact, res_tol=5e-4)
