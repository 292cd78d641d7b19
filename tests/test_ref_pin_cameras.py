"""PIN of the oracle through cameras other than synth.pinhole_K (tests/cameras.py: aspect, offset, general).

Every other pin runs one camera, fx == fy with the principal point at the image centre, where reading fx for fy (fxi for fyi, cx
for cy) gives the same bits and the per-level principal point is exact in float as in double.  This module runs every case
function of tests/pin_cases.py that reads K -- frame_builders (with K and KInv of every level), point_cloud, the GEOMETRY cases
and the keyframe loop -- through each camera, the Sim3 / permaRef cases on mapped keyframes through `offset` and `general`, and
the depth-map cases through `general` under the vertical motion (cameras.VERTICAL), which alone reaches the y-dominant depth
formula.  Every observation is checked against tests/golden/ref_pin_cameras_320x240.npz, recorded from oracle/_ref/liblsd_ref.so by
python -m tests.golden.make_golden_ref_pin_cameras.

Non-vacuity: each camera's record differs from the default camera's record in every case both have; the same images with fx and
fy swapped, or with the principal point one pixel lower, do not match the record in any case that does not record K itself."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import cameras, motions
from tests import pin_cases as pin

PAIRS = pin.CAMERA_PAIRS

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_CAMERAS)
    return _gold


@pytest.mark.parametrize("camera,case", PAIRS, ids=[f"{m}-{c}" for m, c in PAIRS])
def test_matches_reference_compiled_through_camera(camera, case):
    po.branch_counts_reset()
    pin.run_under_camera(camera, case, _load())
    if camera == cameras.VERTICAL:                  # the y-dominant depth formula, the one that reads fyi, ran
        assert po.branch_counts()["depth_y"] >= 5000, po.branch_counts()


def test_cameras_are_what_they_claim():
    """float32 entries, a semi-dense density inside 30-50 %, fx != fy where stated, the principal point off centre where stated,
    and one camera whose level cy depends on the precision of the level formula"""
    for name in cameras.SMALL + ("euroc640",):
        K = cameras.camera_K(name)
        assert K.dtype == np.float32 and K[0, 1] == 0 and np.array_equal(K[2], [0, 0, 1])
    w, h = 320, 240
    for name, (fx_ne_fy, off_centre) in {"aspect": (True, False), "offset": (False, True), "general": (True, True)}.items():
        seq = cameras.sequence(name)
        seq.check_density()
        K = seq.K
        assert (K[0, 0] != K[1, 1]) == fx_ne_fy and (K[0, 2] != (w - 1) / 2 and K[1, 2] != (h - 1) / 2) == off_centre, name
    assert cameras.level_cy_rounds("general") == [1, 2, 3, 4]
    assert not cameras.level_cy_rounds("offset") and not cameras.level_cy_rounds("aspect")


def test_euroc640_is_the_undistorters_K():
    """cameras.EUROC640 is still what UndistorterOpenCV hands to the system for the EuRoC calibration at 640x480"""
    from lsd_slam_b200 import abi
    from tests.golden import make_golden_opencv_undistort as mg
    u = abi.UndistorterOpenCV(mg.EUROC, (752, 480), "full", (640, 480))
    assert u.status == 0
    assert u.getK().tobytes() == cameras.camera_K("euroc640").tobytes()
    cameras.CameraSequence(u.getK(), 640, 480).check_density()


def test_pinned_level_intrinsics():
    """Frame::K(level) of the reference equals the level formula in double (Frame.cpp:446-450) for every camera: the record of
    K{l} is the hash of that matrix"""
    g = _load()
    for name in cameras.SMALL:
        _, _, fx, fy, cx, cy = cameras.CAMERAS[name]
        for lvl in range(5):
            fxl, fyl = fx, fy
            for _ in range(lvl):
                fxl, fyl = np.float32(np.float64(fxl) * 0.5), np.float32(np.float64(fyl) * 0.5)
            cxl = cx if lvl == 0 else cameras.level_c(cx, lvl)
            cyl = cy if lvl == 0 else cameras.level_c(cy, lvl)
            K = np.array([[fxl, 0, cxl], [0, fyl, cyl], [0, 0, 1]], np.float32)
            assert g[f"{name}/frame_builders/K{lvl}"].tobytes() == bytes.fromhex(pin._digest(K)), (name, lvl)


def _default_key(key):
    """the same observation in the default camera's records (ref_pin, ref_pin_sim3's default motion)"""
    case, rest = key.split("/", 2)[1], key.split("/", 1)[1]
    if case in pin.SIM3_CASES:
        return pin.GOLD_SIM3, f"{motions.DEFAULT}/{rest}"
    return pin.GOLD, rest


@pytest.mark.parametrize("camera", cameras.SMALL)
def test_each_camera_changes_the_recorded_outputs(camera):
    """every case's record through the camera differs from the default camera's record somewhere: the camera reached the
    reference's code in each of them"""
    g = _load()
    golds, differ = {}, {}
    for key in (k for k in g.files if k.startswith(camera + "/")):
        path, dk = _default_key(key)
        d = golds.setdefault(path, np.load(path))
        if dk in d.files:
            differ.setdefault(key.split("/")[1], []).append(not np.array_equal(g[key], d[dk]))
    cases = {c for m, c in PAIRS if m == camera}
    assert set(differ) == cases, cases - set(differ)
    assert all(any(v) for v in differ.values()), [c for c, v in differ.items() if not any(v)]


def _swapped(K):
    K = K.copy()
    K[0, 0], K[1, 1] = K[1, 1], K[0, 0]
    return K


def _cy_plus_one(K):
    K = K.copy()
    K[1, 2] += np.float32(1.0)
    return K


# camera -> (what changes, the K the oracle is given instead, with the camera's own images)
WRONG = {"aspect": ("fx and fy swapped", _swapped), "offset": ("cy one pixel lower", _cy_plus_one)}
SENSITIVE_CASES = ("point_cloud", "depthmap_update_sequence", "se3_single_evaluation", "se3_track_scalar")


@pytest.mark.parametrize("case", SENSITIVE_CASES)
@pytest.mark.parametrize("camera", list(WRONG))
def test_record_tells_a_wrong_camera_apart(camera, case):
    """the same images given to the oracle with the wrong camera do not match the record: the fixture can tell fx from fy and cy
    from cy + 1 in cases that never record K itself"""
    _, wrong = WRONG[camera]
    seq = cameras.sequence(camera, K=wrong(cameras.camera_K(camera)))
    record = _load()
    checked = []

    class Watched(pin.Pin):
        """a Pin that reports which recorded observation the run first disagreed with"""

        def exact(self, what, a):
            checked.append(what)
            return super().exact(what, a)

        def value(self, what, a):
            checked.append(what)
            return super().value(what, a)

    fn, fl, _ = pin.CAMERA_CASES[case]
    p = Watched(f"{camera}/{case}", record)
    try:
        with pytest.raises(AssertionError) as err:
            fn(p, fl, seq, cameras.stream(camera)[1])
    finally:
        po.set_globals(False)
    # the assertion that failed compares the last observation taken from the record: a mismatch with the record, not one of
    # the case's own sanity checks before it
    assert checked and f"{camera}/{case}/{checked[-1]}" in record.files, checked
    tb = err.traceback
    assert any(e.frame.code.name in ("exact", "_se3_eval_levels", "_se3_track_sequence") for e in tb[-2:]), str(err.value)


def test_sim3_pose_moved_by_the_references_own_sums():
    """pin_cases.SIM3_SUM_SENSITIVE: the recorded reference pose of that trackFrameSim3 call lies more than 4e-5 (relative
    translation) from the same tracking with every sum of the Sim3 tracker exact (lsdo_globals.exactSim3Sums), with the same LM
    call counts, and over three times as far as from the twin that makes only the affine sums exact.  So the fp32 order of the
    normal-equation sums alone moves this pose by a large part of POSE_TOL, and a device that sums in another order is held to
    the all-sums-exact twin plus the reference's distance to it (device_cases.mapped_sim3_track, DESIGN.md section 5, Cameras)"""
    from tests.util import oracle_sim3_exact, oracle_sim3_track, sim3_err
    cam, ref, fr, lo, hi = pin.SIM3_SUM_SENSITIVE
    po.set_globals(False)
    m = pin.mapped(False, *cameras.stream(cam))
    init = m.frame_to_ref(ref, fr)
    want, affine = oracle_sim3_track(po, m.of[ref], m.of[fr], init, lo, hi)
    rec = _load()[f"{cam}/sim3_track_mapped/{ref}->{fr}/{lo}{hi}"][:8]
    assert np.allclose(np.array(want.frameToRef_qts), rec, rtol=0, atol=1e-12)
    exact = oracle_sim3_exact(po, m.of[ref], m.of[fr], init, lo, hi)
    assert list(exact.numCalcResidualCalls) == list(want.numCalcResidualCalls)
    d_all = sim3_err(rec, exact.frameToRef_qts)[0]
    d_affine = sim3_err(rec, affine.frameToRef_qts)[0]
    assert d_all > 4e-5 and d_all > 3 * d_affine, (d_all, d_affine)
