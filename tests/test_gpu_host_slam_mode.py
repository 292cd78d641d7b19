"""SlamSystem's SLAM mode through the C++ adapter (lsd_slam_b200/host/lsd_host.h): Frame::setPermaRef, SE3Tracker::checkPermaRefOverlap /
trackFrameOnPermaref, DepthMap::setFromExistingKF(Frame*), FrameMemory::setMaxDeviceRecords and the reference's run-time globals,
driven by tests/native/host_slam_mode.cpp in SlamSystem's order and compared bit for bit with the same calls made through abi.py.  Those ABI
calls are held to the reference's recorded values by test_gpu_sim3_motions.py / test_gpu_perma.py / test_gpu_globals.py."""
import os
import struct
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES, KF_EVERY = 16, 5                 # keyframes 0, 5, 10, 15
REACTIVATE = (12, 5)                       # before frame 12, keyframe 10 is finished and keyframe 5 re-activated; the reference's
                                           # tracker (the oracle) tracks frame 12 as good on it
GLOBALS_AT = 8
GLOBALS = dict(minUseGrad=7.5, cameraPixelNoise2=9.0, depthSmoothingFactor=2.0, allowNegativeIdepths=0, useSubpixelStereo=0,
               useAffineLightningEstimation=0)      # the combined set of test_gpu_globals.py
GLOBALS_ARGS = ["--globals", str(GLOBALS_AT), "7.5", "9", "2", "0", "0", "0"]

# record tags and fixed sizes of host_slam_mode's output (the depth-map records add w*h hypotheses of 32 bytes)
TRACK, KEYFRAME, REACT, FINAL, OVERLAP, PERMA, SIM3 = range(1, 8)
_SIZE = {TRACK: 160, KEYFRAME: 80, REACT: 16, FINAL: 4, OVERLAP: 76, PERMA: 160, SIM3: 364}
_HAS_DEPTH = (KEYFRAME, REACT, FINAL)
IDENT_SE3 = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    exe = tmp_path_factory.mktemp("slam_mode") / "host_slam_mode"
    here = os.path.dirname(build.HOST_OUT)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(ROOT, "tests", "native", "host_slam_mode.cpp"),
                        "-L" + here, "-Wl,-rpath," + here, "-l:liblsdgpu_host.so", "-l:liblsdgpu.so", "-pthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


def test_adapter_exports_the_slam_mode_calls_and_the_globals():
    from lsd_slam_b200 import build
    build.build()
    build.build_host()
    syms = subprocess.run(["nm", "-DC", build.HOST_OUT], capture_output=True, text=True).stdout
    for s in ("lsd_slam::SE3Tracker::trackFrameOnPermaref(lsd_slam::Frame*, lsd_slam::Frame*, lsd_slam::SE3)",
              "lsd_slam::SE3Tracker::checkPermaRefOverlap(lsd_slam::Frame*, lsd_slam::SE3)",
              "lsd_slam::Frame::setPermaRef(lsd_slam::TrackingReference*)",
              "lsd_slam::DepthMap::setFromExistingKF(lsd_slam::Frame*)"):
        assert any(ln.endswith(" T " + s) for ln in syms.splitlines()), s
    for g in ("minUseGrad", "cameraPixelNoise2", "depthSmoothingFactor", "allowNegativeIdepths", "useSubpixelStereo",
              "useAffineLightningEstimation"):
        assert any(ln.endswith(" D lsd_slam::" + g) for ln in syms.splitlines()), g


def test_globals_start_at_the_library_defaults(driver):
    """host only: the adapter's globals before any change equal lsdgpu_default_globals (util/settings.cpp:80-88)"""
    r = subprocess.run([driver, "--print-globals"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    name, *vals = r.stdout.split()
    g = abi.Globals()
    abi.load().lsdgpu_default_globals(abi.C.byref(g))
    assert name == "globals"
    assert [float(v) for v in vals] == [float(getattr(g, f)) for f, _ in abi.Globals._fields_]


# ---- the GPU runs ---------------------------------------------------------------------------------------------------------------
def _frames_file(path, seq, frames):
    with open(path, "wb") as f:
        np.array([seq.w, seq.h, N_FRAMES], np.int32).tofile(f)
        seq.K.astype(np.float32).tofile(f)
        frames[0][1].astype(np.float32).tofile(f)
        for k in range(N_FRAMES):
            frames[k][0].tofile(f)


def _records(buf, wh):
    out, o = [], 0
    while o < len(buf):
        tag = struct.unpack_from("<i", buf, o)[0]
        n = _SIZE[tag] + (32 * wh if tag in _HAS_DEPTH else 0)
        out.append((tag, buf[o:o + n]))
        o += n
    assert o == len(buf)
    return out


class Run:
    def __init__(self, driver, tmp_path, seq, frames, *args):
        _frames_file(tmp_path / "frames.bin", seq, frames)
        main, cons = tmp_path / "main.bin", tmp_path / "constraints.bin"
        r = subprocess.run([driver, str(tmp_path / "frames.bin"), str(main), str(cons), "--kf-every", str(KF_EVERY)] + list(args),
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        self.main, self.cons = main.read_bytes(), cons.read_bytes()
        self.lines = [ln.split() for ln in r.stdout.splitlines()]
        wh = seq.w * seq.h
        self.main_records, self.cons_records = _records(self.main, wh), _records(self.cons, wh)

    def globals(self, what):
        return next([float(v) for v in ln[1:]] for ln in self.lines if ln[0] == what)


def _first_difference(a, b):
    n = min(len(a), len(b))
    d = np.flatnonzero(np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8))
    return int(d[0]) if d.size else n


def assert_same(a: bytes, b: bytes, what):
    assert a == b, f"{what}: {len(a)} vs {len(b)} bytes, first difference at byte {_first_difference(a, b)}"


def _pack(fmt, *v):
    return struct.pack("<" + fmt, *v)


class AbiMirror:
    """The driver's script through abi.py, with the adapter's host-side bookkeeping restated: the keyframe counters that
    DepthMap::updateKeyframe hands to the device, and which tracker members each call leaves set.  The initial estimates are the
    ones the driver computed from its FramePoseStruct chain, read from its records."""

    def __init__(self, seq, frames, adapter: Run, globals_at=None, react=None, on_reactivated=None):
        self.ctx = ctx = abi.Context(seq.w, seq.h, seq.K, max_frames=16)
        self.trk, self.dm = abi.SE3Tracker(ctx), abi.DepthMap(ctx)
        self.ctr, self.s3 = abi.SE3Tracker(ctx), abi.Sim3Tracker(ctx)            # the constraint thread's trackers
        self.perma_residual = 0.0
        self.s3m = dict(pointUsage=0.0, lastResidual=0.0, lastDepthResidual=0.0, lastPhotometricResidual=0.0, a=1.0, b=0.0, diverged=0,
                        H=[0.0] * 49)
        self.main, self.cons = bytearray(), bytearray()
        self.inits = iter([(struct.unpack_from("<ii", r, 4), r[12:68]) for t, r in adapter.main_records if t == TRACK])
        self.cinits = iter([(t, struct.unpack_from("<ii", r, 4), r[12:76 if t == SIM3 else 68]) for t, r in adapter.cons_records])
        self.finished, self.order, self.points, self.counters = [], [], {}, {0: [0, 0]}
        ctx.upload(0, frames[0][0])
        ctx.set_depth_gt(0, frames[0][1])
        self.dm.initializeFromGTDepth(0)
        cur, ref_kf, last_frame = 0, None, None
        for k in range(1, N_FRAMES):
            if k == globals_at:
                ctx.set_globals(**GLOBALS)
            if react and k == react[0]:
                old, first = cur, self.finish(cur)
                self.dm.setFromExistingKF(react[1])
                cur = react[1]
                self.counters[cur] = [0, 0]
                self.main += _pack("iiii", REACT, old, cur, self.points[old]) + self.dm.current().tobytes()
                if on_reactivated:
                    on_reactivated(ctx, cur)
                if first:
                    self.constraints(old)
            ctx.upload(k, frames[k][0])
            if ref_kf != cur or ctx.depth_updated_flag(cur):
                self.trk.importFrame(cur)
                ref_kf = cur
            ids, init = next(self.inits)
            assert ids == (k, cur)
            pose = self.trk.trackFrame(cur, k, np.frombuffer(init, np.float64))
            t = self.trk
            self.main += _pack("iii", TRACK, k, cur) + init + pose.tobytes() + _pack(
                "7f2i", t.pointUsage, t.lastGoodCount, t.lastMeanRes, t.lastBadCount, t.lastResidual, t.affineEstimation_a,
                t.affineEstimation_b, t.diverged, t.trackingWasGood)
            self.counters[cur][0] += t.trackingWasGood
            if last_frame is not None:
                ctx.release(last_frame)
                last_frame = None
            if k % KF_EVERY == 0:
                old, first = cur, self.finish(cur)
                q = self.dm.createKeyFrame(k)
                cur = k
                self.counters[k] = [0, 0]
                self.main += _pack("iiii", KEYFRAME, old, k, self.points[old]) + q.tobytes() + self.dm.current().tobytes()
                if first:
                    self.constraints(old)
            else:
                ctx.set_counters(cur, *self.counters[cur])
                d = (abi.RefDesc * 1)()
                d[0].frame_id, d[0].tracked_on_kf = k, 1
                ctx._ck(ctx.L.lsdgpu_depth_update_keyframe_refs(ctx.ptr, d, 1))
                self.counters[cur][1] += 1
                ctx.clear_good_mask(k)
                last_frame = k
        self.main += _pack("i", FINAL) + self.dm.current().tobytes()
        self.main, self.cons = bytes(self.main), bytes(self.cons)
        ctx.close()

    def finish(self, kf):                      # SlamSystem::finishCurrentKeyframe
        self.dm.finalizeKeyFrame()
        self.trk.importFrame(kf)
        self.points[kf] = self.trk.setPermaRef(kf)
        first = kf not in self.order
        if first:
            self.order.append(kf)
        return first

    def _next(self, tag, ref, fr):
        t, ids, init = next(self.cinits)
        assert (t, ids) == (tag, (ref, fr))
        return init

    def perma(self, ref, fr):
        init = self._next(PERMA, ref, fr)
        r = self.ctr.trackFrameOnPermaref([ref], fr, np.frombuffer(init, np.float64))[0]
        pose = IDENT_SE3
        if not r.diverged:
            self.perma_residual = r.lastResidual
            pose = tuple(r.frameToRef_qt)
        self.cons += _pack("iii", PERMA, ref, fr) + init + _pack("7d7f2i", *pose, r.pointUsage, r.lastGoodCount, r.lastMeanRes,
                                                                 r.lastBadCount, self.perma_residual, r.affineEstimation_a,
                                                                 r.affineEstimation_b, r.diverged, r.trackingWasGood)

    def sim3(self, ref, fr):
        init = self._next(SIM3, ref, fr)
        self.trk.importFrame(ref)                                     # TrackingReference::importFrame of the reference keyframe
        self.s3.trackFrameSim3(ref, fr, np.frombuffer(init, np.float64), 4, 1)
        r, m = self.s3.last, self.s3m                                 # Sim3Tracker's members as lsd_host.cpp's take() leaves them
        m.update(pointUsage=r.pointUsage, a=r.affineEstimation_a, b=r.affineEstimation_b, diverged=r.diverged)
        zero = all(v == 0 for v in r.lastSim3Hessian)
        pose = IDENT_SE3 + (1.0,)
        if not (r.diverged and zero):
            m["H"] = list(r.lastSim3Hessian)
            if not (r.diverged or zero):
                m.update(lastResidual=r.lastResidual, lastDepthResidual=r.lastDepthResidual, lastPhotometricResidual=r.lastPhotometricResidual)
                pose = tuple(r.frameToRef_qts)
        self.cons += _pack("iii", SIM3, ref, fr) + init + _pack("8d6fi49f", *pose, m["pointUsage"], m["lastResidual"], m["lastDepthResidual"],
                                                                m["lastPhotometricResidual"], m["a"], m["b"], m["diverged"], *m["H"])

    def constraints(self, kf):
        for c in self.finished:
            c2f = self._next(OVERLAP, c, kf)
            u = self.ctr.checkPermaRefOverlap([c], np.frombuffer(c2f, np.float64))[0]
            self.cons += _pack("iii", OVERLAP, c, kf) + c2f + _pack("ff", u, u)
            self.perma(c, kf)
            self.perma(kf, c)
            self.sim3(c, kf)
            self.sim3(kf, c)
        self.finished.append(kf)


@pytest.fixture(scope="module")
def runs(driver, tmp_path_factory, seq_small, frames_small):
    """the adapter's runs, each once: the base script with a re-activation, the same with globals changed, with pruning, and the
    script without re-activation sequentially and with the constraint calls on a second thread"""
    react = ["--reactivate", str(REACTIVATE[0]), str(REACTIVATE[1])]
    args = {"base": react, "globals": react + GLOBALS_ARGS, "pruned": react + ["--prune", "2"], "sequential": [],
            "threads": ["--threads"]}
    return {name: Run(driver, tmp_path_factory.mktemp(name), seq_small, frames_small, *a) for name, a in args.items()}


@pytest.mark.gpu
def test_slam_mode_adapter_equals_the_abi(runs, seq_small, frames_small, oracle):
    """every pose, tracker member, permaRef point count and depth map after every keyframe change, bit for bit"""
    from tests.device_cases import mirror
    base = runs["base"]
    tags = [t for t, _ in base.main_records]
    assert tags.count(KEYFRAME) == 3 and tags.count(REACT) == 1 and tags.count(TRACK) == N_FRAMES - 1
    ctags = [t for t, _ in base.cons_records]
    assert ctags.count(OVERLAP) == 3 and ctags.count(PERMA) == 6 and ctags.count(SIM3) == 6     # pairs (5,0), (10,0), (10,5)
    good = {}

    def reactivated(ctx, kf):                  # the reference's tracker on the re-activated keyframe's depth
        okf = mirror(oracle, ctx, seq_small, kf, frames_small[kf][0])
        of = oracle.Frame(REACTIVATE[0], frames_small[REACTIVATE[0]][0], seq_small.K)
        init = next(np.frombuffer(r[12:68], np.float64) for t, r in base.main_records if t == TRACK and struct.unpack_from("<i", r, 4)[0] == REACTIVATE[0])
        good["oracle"] = oracle.se3_track(okf, of, init).trackingWasGood

    m = AbiMirror(seq_small, frames_small, base, react=REACTIVATE, on_reactivated=reactivated)
    assert good["oracle"], f"frame {REACTIVATE[0]} is not tracked as good on keyframe {REACTIVATE[1]}"
    assert_same(base.main, m.main, "tracking and mapping")
    assert_same(base.cons, m.cons, "constraint calls")
    points = [struct.unpack_from("<i", r, 12)[0] for t, r in base.main_records if t in (KEYFRAME, REACT)]
    assert min(points) > 50, points
    perma_good = [struct.unpack_from("<i", r, 156)[0] for t, r in base.cons_records if t == PERMA]
    assert any(perma_good), "no permaRef tracking was good"


@pytest.mark.gpu
def test_slam_mode_follows_the_reference_globals(runs, seq_small, frames_small):
    """lsd_slam::minUseGrad ... changed before frame 8 act like Context.set_globals at that frame, reach the context, and a
    DeviceContext created afterwards starts with them"""
    run = runs["globals"]
    m = AbiMirror(seq_small, frames_small, run, globals_at=GLOBALS_AT, react=REACTIVATE)
    assert_same(run.main, m.main, "tracking and mapping")
    assert_same(run.cons, m.cons, "constraint calls")
    base = runs["base"]
    n_before = sum(1 for t, r in base.main_records if t == TRACK and struct.unpack_from("<i", r, 4)[0] < GLOBALS_AT)
    assert run.main_records[:n_before + 1] == base.main_records[:n_before + 1]      # the same up to the change
    assert run.main != base.main
    want = [GLOBALS[f] for f, _ in abi.Globals._fields_]
    assert run.globals("context") == want and run.globals("fresh") == want
    d = abi.Globals()
    abi.load().lsdgpu_default_globals(abi.C.byref(d))
    assert base.globals("context") == [float(getattr(d, f)) for f, _ in abi.Globals._fields_]


@pytest.mark.gpu
def test_slam_mode_reactivates_a_minimized_keyframe(runs):
    """keyframe 5, minimized by pruneActiveFrames, re-activated by setFromExistingKF(Frame*) and tracked and mapped on: the same
    outputs as the run that never minimized it; the permaRef calls against a minimized keyframe leave it minimized"""
    pruned, base = runs["pruned"], runs["base"]
    assert ["REACTIVATE", str(REACTIVATE[1]), "0"] in pruned.lines
    assert ["REACTIVATE", str(REACTIVATE[1]), "1"] in base.lines
    assert_same(pruned.main, base.main, "tracking and mapping")
    assert_same(pruned.cons, base.cons, "constraint calls")
    calls = [ln for ln in pruned.lines if ln[0] == "ACTIVE"]
    minimized = [ln for ln in calls if ln[3] == "0"]
    assert minimized, calls
    assert all(ln[4] == "0" for ln in minimized), minimized


@pytest.mark.gpu
def test_slam_mode_constraint_thread_on_one_context(runs):
    """the constraint calls on a second thread of the same DeviceContext give the sequential run's outputs.  The context has
    enough frame slots that FrameMemory never minimizes for room: the on-demand minimize clears a frame's refPixelWasGood, and
    which frame it picked would then depend on the threads' timing."""
    seq, thr = runs["sequential"], runs["threads"]
    assert [t for t, _ in seq.cons_records].count(OVERLAP) == 3
    assert_same(thr.main, seq.main, "tracking and mapping")
    assert_same(thr.cons, seq.cons, "constraint calls")


def _memory(run):
    """the MEMORY lines of a --device-records run: (n_device, device_bytes, n_host, host_bytes) before the re-activation, if any,
    then at the end"""
    return [tuple(int(v) for v in ln[1:]) for ln in run.lines if ln[0] == "MEMORY"]


@pytest.mark.gpu
def test_setFromExistingKF_on_an_offloaded_keyframe(driver, tmp_path, seq_small, frames_small):
    """FrameMemory::setMaxDeviceRecords(0) with two active frames: keyframe 5 is re-activated from host memory by
    setFromExistingKF(Frame*) and tracked and mapped on; the permaRef and Sim3 calls read offloaded keyframes"""
    react = ["--reactivate", str(REACTIVATE[0]), str(REACTIVATE[1])]
    run = Run(driver, tmp_path, seq_small, frames_small, *react, "--prune", "2", "--device-records", "0")
    assert ["REACTIVATE", str(REACTIVATE[1]), "0"] in run.lines
    before, end = _memory(run)
    assert before[0] == 0 and before[2] >= 1, before      # keyframe 5 is minimized, so its record is in host memory
    assert end[0] == 0 and end[2] >= 2, end
    m = AbiMirror(seq_small, frames_small, run, react=REACTIVATE)
    assert_same(run.main, m.main, "tracking and mapping")
    assert_same(run.cons, m.cons, "constraint calls")


@pytest.mark.gpu
def test_constraint_thread_with_offloaded_keyframes(driver, tmp_path, seq_small, frames_small):
    """the constraint calls on a second thread while the main thread prunes and offloads.  Three active frames: the two frames a
    constraint call holds and the active keyframe, so that pruning always finds a frame to minimize; which one it picks depends on
    the threads' timing, and none of the outputs does."""
    run = Run(driver, tmp_path, seq_small, frames_small, "--threads", "--prune", "3", "--device-records", "0")
    (end,) = _memory(run)
    assert end[0] == 0 and end[2] >= 1, end
    m = AbiMirror(seq_small, frames_small, run)
    assert_same(run.main, m.main, "tracking and mapping")
    assert_same(run.cons, m.cons, "constraint calls")


@pytest.mark.gpu
def test_slam_mode_misuse(driver, tmp_path, seq_small, frames_small):
    """setPermaRef with a TrackingReference of another frame throws and changes nothing; trackFrameOnPermaref on a keyframe
    without a permaRef throws naming it"""
    _frames_file(tmp_path / "frames.bin", seq_small, frames_small)
    r = subprocess.run([driver, "--errors", str(tmp_path / "frames.bin")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lines = {ln.split()[0]: ln for ln in r.stdout.splitlines()}
    assert lines["setPermaRef"].startswith("setPermaRef error Frame::setPermaRef: the TrackingReference holds frame 1, not frame 0")
    assert lines["trackFrameOnPermaref"].startswith("trackFrameOnPermaref error SE3Tracker::trackFrameOnPermaref (keyframe 1)")
    assert "no permaRef" in lines["trackFrameOnPermaref"]
    _, n0, n0_after, u0, u0_after, n1, u1 = lines["permaRef"].split()
    assert n0 == n0_after and u0 == u0_after and int(n0) > 50
    assert u1 != u0                            # the rejected call would have changed the overlap
