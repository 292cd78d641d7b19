"""PIN of the oracle under exposure changes (tests/photometry.py: ramp, step, saturate, dark, ramp_forward).

Every other pin renders frames at one brightness, so the trackers' affine model c1 = a * I_ref + b (SE3Tracker.cpp:952,
Sim3Tracker.cpp:510) stays near the identity, the final SE3 evaluation has no bad point, and the depth map, which compares raw
intensities, fails a stereo search or a propagation only where the map itself is wrong.  This module runs under each schedule:
  * the depth-map cases of tests/pin_cases.py (DEPTH), and propagation_exposure: the ground-truth map propagated to frame 8
    without and with a tracking mask;
  * se3_eval_exposure: one SE3 evaluation of frame 3, levels 4-1, at the affine estimates (1, 0), the frame's true (g, o) and
    pin_cases.FAR_AFFINE -- counts, statistics, normal equations and the level-1 mask;
  * se3_track_scalar (frames 1-6 tracked and mapped; under `dark` frame 3 is not good), bench_loop_with_keyframe_changes;
  * sim3_eval_mapped, sim3_track_mapped and perma_mapped on the keyframes oracle/cpu_stream.py mapped from the exposed stream.
Every observation is checked against tests/golden/ref_pin_photometry_320x240.npz, recorded from oracle/_ref/liblsd_ref.so by
python -m tests.golden.make_golden_ref_pin_photometry.

Non-vacuity: the C restatement's counters (pyoracle.BRANCHES) reach the minima of REACHES in each (schedule, case); the recorded
tracker outputs show bad points, a clipped-away good mask, affine estimates far from the identity and a not-good frame; each
schedule's record differs from the constant-exposure record."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import motions, photometry
from tests import pin_cases as pin

PAIRS = pin.PHOTOMETRY_PAIRS

# (schedule, case) -> {counter: at least this many runs} on the C restatement, about half the measured count.  se3_eval_exposure,
# sim3_track_mapped and perma_mapped run no depth-map pass.  For comparison, on the constant-exposure stream
# depthmap_update_sequence reaches stereo_unclear 132 times and update_inconsistent 13 times, and no stereo -3 at all.
REACHES = {
    ("ramp", "depthmap_update_sequence"): dict(stereo_unclear=80, update_inconsistent=100),
    ("ramp", "depthmap_random_init_every_branch"):
        dict(stereo_err_search=10000, stereo_err_interp=4000, stereo_unclear=1000, update_inconsistent=10000,
             create_blacklist=4),
    ("ramp", "depthmap_individual_passes"): dict(stereo_unclear=40, update_inconsistent=30),
    ("ramp", "create_keyframe_and_finalize"): dict(stereo_unclear=100, update_inconsistent=1000, prop_mask=1000),
    ("ramp", "propagation_exposure"): dict(prop_mask=2000),
    ("ramp", "se3_eval_exposure"): dict(),
    ("ramp", "se3_track_scalar"): dict(stereo_unclear=80, update_inconsistent=50),
    ("ramp", "bench_loop_with_keyframe_changes"):
        dict(stereo_err_interp=4, stereo_unclear=300, update_fail_invalidate=30, update_inconsistent=400, create_blacklist=10,
             prop_mask=100),
    ("ramp", "sim3_eval_mapped"):
        dict(stereo_unclear=200, update_fail_invalidate=10, update_inconsistent=200, create_blacklist=1, prop_mask=90),
    ("ramp", "sim3_track_mapped"): dict(),
    ("ramp", "perma_mapped"): dict(),
    ("step", "depthmap_update_sequence"):
        dict(stereo_err_search=90, stereo_err_interp=100, stereo_unclear=60, update_inconsistent=200),
    ("step", "depthmap_random_init_every_branch"):
        dict(stereo_err_search=20000, stereo_err_interp=10000, stereo_unclear=1000, update_inconsistent=9000,
             create_blacklist=10),
    ("step", "depthmap_individual_passes"): dict(stereo_unclear=30, update_inconsistent=7),
    ("step", "create_keyframe_and_finalize"):
        dict(stereo_err_search=30, stereo_err_interp=20, stereo_unclear=100, update_inconsistent=60, prop_mask=1000),
    ("step", "propagation_exposure"): dict(prop_mask=2000, prop_color=5000),
    ("step", "se3_eval_exposure"): dict(),
    ("step", "se3_track_scalar"):
        dict(stereo_err_search=1000, stereo_err_interp=1000, stereo_unclear=100, update_inconsistent=60),
    ("step", "bench_loop_with_keyframe_changes"):
        dict(stereo_err_search=1000, stereo_err_interp=1000, stereo_unclear=400, update_fail_invalidate=40,
             update_inconsistent=100, create_blacklist=20, prop_mask=2000),
    ("step", "sim3_eval_mapped"):
        dict(stereo_err_search=400, stereo_err_interp=700, stereo_unclear=300, update_fail_invalidate=40,
             update_inconsistent=100, create_blacklist=10, prop_mask=2000),
    ("step", "sim3_track_mapped"): dict(),
    ("step", "perma_mapped"): dict(),
    ("saturate", "depthmap_update_sequence"):
        dict(stereo_err_search=10000, stereo_err_interp=10000, stereo_unclear=40, update_inconsistent=10000),
    ("saturate", "depthmap_random_init_every_branch"):
        dict(stereo_err_search=20000, stereo_err_interp=10000, stereo_unclear=1000, update_inconsistent=5000,
             create_blacklist=10),
    ("saturate", "depthmap_individual_passes"):
        dict(stereo_err_search=3000, stereo_err_interp=2000, stereo_unclear=9, update_inconsistent=1000),
    ("saturate", "create_keyframe_and_finalize"):
        dict(stereo_err_search=7000, stereo_err_interp=4000, stereo_unclear=100, update_inconsistent=3000, create_blacklist=7,
             prop_mask=1000),
    ("saturate", "propagation_exposure"): dict(prop_mask=2000, prop_color=9000),
    ("saturate", "se3_eval_exposure"): dict(),
    ("saturate", "se3_track_scalar"): dict(stereo_err_search=4000, stereo_err_interp=7000, stereo_unclear=200),
    ("saturate", "bench_loop_with_keyframe_changes"):
        dict(stereo_err_search=6000, stereo_err_interp=10000, stereo_unclear=1000, update_fail_invalidate=70,
             update_inconsistent=100, create_blacklist=300, prop_mask=7000),
    ("saturate", "sim3_eval_mapped"):
        dict(stereo_err_search=2000, stereo_err_interp=4000, stereo_unclear=500, update_fail_invalidate=80,
             update_inconsistent=90, create_blacklist=200, prop_mask=6000),
    ("saturate", "sim3_track_mapped"): dict(),
    ("saturate", "perma_mapped"): dict(),
    ("dark", "depthmap_update_sequence"): dict(stereo_unclear=60, update_inconsistent=6),
    ("dark", "depthmap_random_init_every_branch"):
        dict(stereo_err_search=9000, stereo_err_interp=4000, stereo_unclear=2000, update_inconsistent=10000,
             create_blacklist=4),
    ("dark", "depthmap_individual_passes"): dict(stereo_unclear=30, update_inconsistent=7),
    ("dark", "create_keyframe_and_finalize"):
        dict(stereo_err_search=80, stereo_unclear=100, update_inconsistent=10, prop_mask=1000),
    ("dark", "propagation_exposure"): dict(prop_mask=2000),
    ("dark", "se3_eval_exposure"): dict(),
    ("dark", "se3_track_scalar"): dict(stereo_err_search=70, stereo_unclear=60, update_inconsistent=6),
    ("dark", "bench_loop_with_keyframe_changes"):
        dict(stereo_err_search=70, stereo_unclear=100, update_fail_invalidate=10, update_inconsistent=10, create_blacklist=10,
             prop_mask=100),
    ("dark", "sim3_eval_mapped"):
        dict(stereo_err_search=70, stereo_unclear=100, update_fail_invalidate=9, update_inconsistent=10, prop_mask=80),
    ("dark", "sim3_track_mapped"): dict(),
    ("dark", "perma_mapped"): dict(),
    ("ramp_forward", "depthmap_update_sequence"): dict(stereo_err_interp=1, stereo_unclear=100, update_inconsistent=200),
    ("ramp_forward", "depthmap_random_init_every_branch"):
        dict(stereo_err_search=10000, stereo_err_interp=4000, stereo_unclear=1000, update_inconsistent=10000,
             create_blacklist=5),
    ("ramp_forward", "depthmap_individual_passes"): dict(stereo_unclear=60, update_inconsistent=30),
    ("ramp_forward", "create_keyframe_and_finalize"):
        dict(stereo_unclear=100, update_inconsistent=5000, create_blacklist=5, prop_mask=1000),
    ("ramp_forward", "propagation_exposure"): dict(prop_mask=2000),
    ("ramp_forward", "se3_eval_exposure"): dict(),
    ("ramp_forward", "se3_track_scalar"): dict(stereo_unclear=90, update_inconsistent=90),
    ("ramp_forward", "bench_loop_with_keyframe_changes"):
        dict(stereo_err_interp=2, stereo_unclear=600, update_fail_invalidate=50, update_inconsistent=500, create_blacklist=100),
    ("ramp_forward", "sim3_eval_mapped"):
        dict(stereo_unclear=300, update_fail_invalidate=30, update_inconsistent=200, create_blacklist=9),
    ("ramp_forward", "sim3_track_mapped"): dict(),
    ("ramp_forward", "perma_mapped"): dict(),
}

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_PHOTOMETRY)
    return _gold


@pytest.mark.parametrize("schedule,case", PAIRS, ids=[f"{s}-{c}" for s, c in PAIRS])
def test_matches_reference_compiled_under_exposure(schedule, case):
    po.branch_counts_reset()
    pin.run_under_exposure(schedule, case, _load())
    got = po.branch_counts()
    low = {b: (got[b], n) for b, n in REACHES[(schedule, case)].items() if got[b] < n}
    assert not low, f"{schedule}/{case}: branches reached fewer times than stated (got, stated): {low}"


def test_every_photometric_counter_is_reached():
    """every counter this pin is about has a stated minimum under some schedule, the colour check of propagation among them; the
    negative-idepth -2 needs allowNegativeIdepths = 0 and is reached by that set of the settings pin"""
    assert set(REACHES) == set(PAIRS)
    reached = {b for want in REACHES.values() for b, n in want.items() if n > 0}
    want = {"stereo_err_search", "stereo_err_interp", "stereo_unclear", "update_fail_invalidate", "update_inconsistent",
            "create_blacklist", "prop_mask", "prop_color"}
    assert want <= reached, want - reached
    po.branch_counts_reset()
    pin.run_under_settings("allowNegativeIdepths=0", "depthmap_update_sequence", np.load(pin.GOLD_GLOBALS),
                           *motions.stream(motions.DEFAULT))
    assert po.branch_counts()["stereo_negative"] >= 100
    assert set(pin.UNREACHED_BY_DEFAULT_PHOTOMETRIC) <= reached | {"stereo_negative"}


def _default_key(schedule, key):
    """the key of the same observation in the constant-exposure records (ref_pin, ref_pin_motions, ref_pin_sim3)"""
    case = key.split("/", 2)[1]
    rest = key.split("/", 1)[1]
    motion = photometry.MOTION.get(schedule, motions.DEFAULT)
    if case in pin.SIM3_CASES:
        return pin.GOLD_SIM3, f"{motion}/{rest}"
    if motion != motions.DEFAULT:
        return pin.GOLD_MOTIONS, f"{motion}/{rest}"
    return pin.GOLD, rest


@pytest.mark.parametrize("schedule", list(photometry.SCHEDULES))
def test_each_schedule_changes_the_recorded_outputs(schedule):
    """the record of every schedule differs from the constant-exposure record somewhere in the depth map, the SE3 tracker and the
    Sim3 tracker: the exposure reached the reference's code"""
    g = _load()
    golds = {}
    differ = {}
    for key in (k for k in g.files if k.startswith(schedule + "/")):
        path, dk = _default_key(schedule, key)
        d = golds.setdefault(path, np.load(path))
        if dk in d.files:
            area = key.split("/")[1]
            differ.setdefault(area, []).append(not np.array_equal(g[key], d[dk]))
    assert {"depthmap_update_sequence", "se3_track_scalar", "sim3_track_mapped"} <= set(differ), sorted(differ)
    for area in ("se3_track_scalar", "bench_loop_with_keyframe_changes", "sim3_track_mapped"):
        assert any(differ[area]), (schedule, area)


def _stats(schedule, k):
    """se3_track_scalar's recorded statistics of frame k: lastResidual, pointUsage, good, bad, meanRes, a, b, diverged,
    trackingWasGood, initialTrackedResidual"""
    return _load()[f"{schedule}/se3_track_scalar/f{k}/stats"]


def test_tracker_outputs_leave_the_identity():
    """what the constant-exposure pins never show: under `step` and `saturate` the reference's final (a, b) leaves the identity
    (it replaces a by each evaluation's estimate, so it swings between the gain and 1) and its last evaluation has bad points;
    under `dark` frame 3 is not good without diverging, every other frame of every schedule is good"""
    for s in photometry.SCHEDULES:
        for k in range(1, 7):
            st = _stats(s, k)
            assert st[7] == 0, (s, k)
            assert st[8] == (0 if (s, k) == ("dark", photometry.DARK_FRAME) else 1), (s, k, st)
    st = _stats("step", 5)
    assert st[5] > 1.03 and st[3] > 1000, st
    st = _stats("saturate", 4)
    assert st[5] > 1.2 and st[6] < -10 and st[3] > 3000, st
    st = _stats("dark", photometry.DARK_FRAME)
    assert st[2] / (st[2] + st[3]) < 0.5, st


@pytest.mark.parametrize("schedule", list(photometry.SCHEDULES))
def test_wrong_affine_estimates_leave_bad_points(schedule):
    """se3_eval_exposure: of the two estimates other than the frame's true (g, o) -- the identity and pin_cases.FAR_AFFINE -- the
    one farther from the truth leaves more than 15 % of the warped points bad on every level, and the true (g, o) leaves
    fewer bad points at level 1 than it (no bad point at all where nothing clipped)"""
    g = _load()
    ident, true, far = pin.eval_affines(photometry.stream(schedule)[0])

    def counts(ab, lvl):
        tag = "" if ab == ident else f"a{ab[0]:g}_b{ab[1]:g}/"
        return g[f"{schedule}/se3_eval_exposure/{tag}L{lvl}/counts"]
    worst = max((ident, far), key=lambda ab: counts(ab, 1)[2])
    for lvl in (4, 3, 2, 1):
        c = counts(worst, lvl)
        assert c[2] > 0.15 * c[0], (lvl, worst, c)
    assert counts(true, 1)[2] < counts(worst, 1)[2]
