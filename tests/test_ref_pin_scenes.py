"""PIN of the oracle on scenes other than the smooth height field (tests/scenes.py: occluder, posts, stripes, flat, blank,
blank_const).

Every other pin renders synth.Sequence's height field: continuous depth, no occlusion, no repeated texture, no large flat area.
There the occlusion vote of regularizeDepthMap<true> and the occluded-source skip of propagateDepth never run (test below), and
doLineStereo's "no clear winner" exit runs only by chance.  This module runs on each textured scene the depth-map cases of
tests/pin_cases.py (DEPTH), the SE3 cases (TRACK), point_cloud, propagate_from_gt (the ground-truth map propagated to frame 8)
and the Sim3 / permaRef cases on keyframes the mapper finished; on `blank` and `blank_const` it runs empty_keyframe: random
init, mapping, fill-holes and the regularisers on a map of a few hundred pixels or none, and every tracker on a keyframe with
a handful of points or none.  Every observation is checked against tests/golden/ref_pin_scenes_320x240.npz, recorded from
oracle/_ref/liblsd_ref.so by python -m tests.golden.make_golden_ref_pin_scenes.

Non-vacuity: the C restatement's branch counters (pyoracle.BRANCHES) reach the minima of REACHES in each (scene, case)."""
import numpy as np
import pytest

from lsd_slam_b200 import synth
from oracle import pyoracle as po
from tests import scenes
from tests import pin_cases as pin

PAIRS = pin.SCENE_PAIRS

# (scene, case) -> {counter: at least this many runs} on the C restatement, about half the measured count.  se3_single_evaluation,
# point_cloud, sim3_track_mapped and perma_mapped run no depth-map pass; the Sim3 / permaRef cases count the mapping run that made
# their keyframes once per process, in sim3_eval_mapped.
REACHES = {
    ("occluder", "depthmap_update_sequence"): dict(epl_reject_grad=10000, epl_reject_angle=8000, stereo_unclear=60,
                                                   update_inconsistent=100),
    ("occluder", "depthmap_random_init_every_branch"): dict(reg_validity=30, fill_create=50, epl_reject_grad=10000,
                                                            epl_reject_angle=7000, stereo_unclear=1000, update_inconsistent=10000),
    ("occluder", "depthmap_individual_passes"): dict(reg_occlusion=8, epl_reject_grad=2000, epl_reject_angle=1000,
                                                     stereo_unclear=30, update_inconsistent=100),
    ("occluder", "create_keyframe_and_finalize"): dict(reg_occlusion=10, reg_validity=30, fill_create=2000, epl_reject_grad=10000,
                                                       epl_reject_angle=7000, prop_skip=40, stereo_unclear=100,
                                                       update_inconsistent=600),
    ("occluder", "se3_single_evaluation"): dict(),
    ("occluder", "se3_track_scalar"): dict(epl_reject_grad=10000, epl_reject_angle=6000, stereo_unclear=60, update_inconsistent=80),
    ("occluder", "point_cloud"): dict(),
    ("occluder", "propagate_from_gt"): dict(prop_skip=60, prop_color=70),
    ("occluder", "sim3_eval_mapped"): dict(reg_occlusion=10, reg_validity=30, fill_create=2000, epl_reject_grad=20000,
                                           epl_reject_angle=10000, prop_skip=90, stereo_unclear=100, update_inconsistent=300),
    ("occluder", "sim3_track_mapped"): dict(),
    ("occluder", "perma_mapped"): dict(),
    ("posts", "depthmap_update_sequence"): dict(epl_reject_grad=20000, epl_reject_angle=10000, stereo_unclear=100,
                                                update_inconsistent=900),
    ("posts", "depthmap_random_init_every_branch"): dict(reg_validity=5, fill_create=40, epl_reject_grad=10000,
                                                         epl_reject_angle=9000, stereo_unclear=1000, update_inconsistent=10000),
    ("posts", "depthmap_individual_passes"): dict(reg_occlusion=30, epl_reject_grad=3000, epl_reject_angle=1000, stereo_unclear=50,
                                                  update_inconsistent=700),
    ("posts", "create_keyframe_and_finalize"): dict(reg_occlusion=100, reg_validity=500, fill_create=4000, epl_reject_grad=10000,
                                                    epl_reject_angle=9000, prop_skip=600, stereo_unclear=100,
                                                    update_inconsistent=3000),
    ("posts", "se3_single_evaluation"): dict(),
    ("posts", "se3_track_scalar"): dict(epl_reject_grad=10000, epl_reject_angle=4000, stereo_unclear=100, update_inconsistent=1000),
    ("posts", "point_cloud"): dict(),
    ("posts", "propagate_from_gt"): dict(prop_skip=800, prop_color=400),
    ("posts", "sim3_eval_mapped"): dict(reg_occlusion=100, reg_validity=300, fill_create=4000, epl_reject_grad=20000,
                                        epl_reject_angle=9000, prop_skip=800, stereo_unclear=300, update_inconsistent=1000),
    ("posts", "sim3_track_mapped"): dict(),
    ("posts", "perma_mapped"): dict(),
    ("stripes", "depthmap_update_sequence"): dict(epl_reject_grad=2000, epl_reject_angle=300),
    ("stripes", "depthmap_random_init_every_branch"): dict(reg_validity=10, fill_create=1, epl_reject_grad=2000,
                                                           epl_reject_angle=200, stereo_unclear=5000, update_inconsistent=50000),
    ("stripes", "depthmap_individual_passes"): dict(epl_reject_grad=400, epl_reject_angle=50),
    ("stripes", "create_keyframe_and_finalize"): dict(fill_create=4000, epl_reject_grad=2000, epl_reject_angle=300),
    ("stripes", "se3_single_evaluation"): dict(),
    ("stripes", "se3_track_scalar"): dict(epl_reject_grad=2000, epl_reject_angle=5000, stereo_unclear=10, update_inconsistent=100),
    ("stripes", "point_cloud"): dict(),
    ("stripes", "propagate_from_gt"): dict(prop_color=1),
    ("stripes", "sim3_eval_mapped"): dict(reg_occlusion=40, reg_validity=400, fill_create=10000, epl_reject_grad=4000,
                                          epl_reject_angle=6000, prop_skip=100, stereo_unclear=300, update_inconsistent=400),
    ("stripes", "sim3_track_mapped"): dict(),
    ("stripes", "perma_mapped"): dict(),
    ("flat", "depthmap_update_sequence"): dict(epl_reject_grad=10000, epl_reject_angle=6000, stereo_unclear=50,
                                               update_inconsistent=300),
    ("flat", "depthmap_random_init_every_branch"): dict(fill_create=20, epl_reject_grad=10000, epl_reject_angle=6000,
                                                        stereo_unclear=1000, update_inconsistent=9000),
    ("flat", "depthmap_individual_passes"): dict(epl_reject_grad=2000, epl_reject_angle=1000, stereo_unclear=40,
                                                 update_inconsistent=200),
    ("flat", "create_keyframe_and_finalize"): dict(fill_create=1000, epl_reject_grad=10000, epl_reject_angle=6000,
                                                   stereo_unclear=100, update_inconsistent=400),
    ("flat", "se3_single_evaluation"): dict(),
    ("flat", "se3_track_scalar"): dict(epl_reject_grad=10000, epl_reject_angle=6000, stereo_unclear=70, update_inconsistent=10),
    ("flat", "point_cloud"): dict(),
    ("flat", "propagate_from_gt"): dict(),
    ("flat", "sim3_eval_mapped"): dict(fill_create=1000, epl_reject_grad=20000, epl_reject_angle=9000, stereo_unclear=100,
                                       update_inconsistent=20),
    ("flat", "sim3_track_mapped"): dict(),
    ("flat", "perma_mapped"): dict(),
    ("blank", "empty_keyframe"): dict(reg_occlusion=10, epl_reject_grad=70, epl_reject_angle=30, update_inconsistent=40),
    ("blank_const", "empty_keyframe"): dict(),
}
NEW_COUNTERS = ("reg_occlusion", "reg_validity", "fill_create", "epl_reject_grad", "epl_reject_angle")
# the depth-map counters the smooth height field never reaches under the default motion, and the cases of the default scene that
# show it: the GEOMETRY depth cases of tests/test_ref_pin.py and propagate_from_gt
UNREACHED_ON_THE_HEIGHT_FIELD = ("reg_occlusion", "prop_skip", "prop_color")

_gold = None


def _load():
    global _gold
    if _gold is None:
        _gold = np.load(pin.GOLD_SCENES)
    return _gold


@pytest.mark.parametrize("scene,case", PAIRS, ids=[f"{s}-{c}" for s, c in PAIRS])
def test_matches_reference_compiled_on_scene(scene, case):
    po.branch_counts_reset()
    pin.run_under_scene(scene, case, _load())
    got = po.branch_counts()
    low = {b: (got[b], n) for b, n in REACHES[(scene, case)].items() if got[b] < n}
    assert not low, f"{scene}/{case}: branches reached fewer times than stated (got, stated): {low}"


def test_every_new_counter_is_reached():
    assert set(REACHES) == set(PAIRS)
    reached = {b for want in REACHES.values() for b, n in want.items() if n > 0}
    assert set(NEW_COUNTERS) <= reached, set(NEW_COUNTERS) - reached
    for sc in ("occluder", "posts"):               # occluding edges under the default motion
        assert max(REACHES[(sc, c)].get("reg_occlusion", 0) for c in pin.DEPTH) > 0, sc
        assert REACHES[(sc, "propagate_from_gt")]["prop_skip"] > 0, sc
    assert REACHES[("stripes", "depthmap_random_init_every_branch")]["stereo_unclear"] >= 1000


# the counters of a successful observation (a depth formula and its subpixel outcome): every other counter is an exit or a decision
SUCCESS = ("depth_x", "depth_y", "subpixel_pre", "subpixel_post", "subpixel_none")


@pytest.mark.parametrize("case", pin.DEPTH)
def test_flat_patches_end_most_observations_at_the_gradient_check(case):
    """measured on the C restatement: on `flat` the epipolar-gradient rejection of makeAndCheckEPL is the most frequent of all
    exits and decisions of each depth-map case, and a larger share of the observations than on the default scene"""
    seq, frames = scenes.stream("flat")
    fn, fl, _ = pin.SCENE_CASES[case]
    po.set_globals(False)
    po.branch_counts_reset()
    fn(pin.Pin(case), fl, seq, frames)
    got = po.branch_counts()
    others = {b: n for b, n in got.items() if b not in SUCCESS + ("epl_reject_grad",)}
    assert got["epl_reject_grad"] > max(others.values()), (got["epl_reject_grad"], max(others.items(), key=lambda kv: kv[1]))
    po.branch_counts_reset()
    fn(pin.Pin(case), fl, synth.Sequence(320, 240, seed=1234), pin.scenes.Frames(synth.Sequence(320, 240, seed=1234)))
    dflt = po.branch_counts()
    po.set_globals(False)

    def share(c):
        return c["epl_reject_grad"] / (c["epl_reject_grad"] + c["depth_x"] + c["depth_y"])
    assert share(got) > share(dflt), (share(got), share(dflt))


def test_height_field_leaves_occlusion_unreached(seq_small, frames_small):
    """the claim this module rests on: on the default scene the depth-map cases never run the occlusion vote of
    regularizeDepthMap<true>, never skip an occluded source in propagateDepth and never drop one by its colour"""
    po.set_globals(False)
    po.branch_counts_reset()
    for c in pin.GEOMETRY:
        fn, fl, _ = pin.CASES[c]
        fn(pin.Pin(c), fl, seq_small, frames_small)
    pin.propagate_from_gt(pin.Pin("propagate_from_gt"), False, seq_small, frames_small)
    got = po.branch_counts()
    assert all(got[b] == 0 for b in UNREACHED_ON_THE_HEIGHT_FIELD), {b: got[b] for b in UNREACHED_ON_THE_HEIGHT_FIELD}
    assert got["reg_validity"] > 0 and got["fill_create"] > 0 and got["prop_merge"] > 0


def test_scenes_are_what_they_claim():
    """depth ratio across the near objects' edges, the posts' edges in frame 0, the stripe period, the flat fraction, the
    selected-pixel count of `blank`"""
    for name in ("occluder", "posts"):
        seq = scenes.sequence(name)
        for k in range(0, 21, 4):
            img, z = seq.render(k)
            near = scenes.near_mask(seq, k)
            if name == "occluder":
                assert 0.15 <= near.mean() <= 0.25, (k, near.mean())
            edge = near[:, 1:] != near[:, :-1]
            zn = np.where(near[:, 1:], z[:, 1:], z[:, :-1])[edge]
            zf = np.where(near[:, 1:], z[:, :-1], z[:, 1:])[edge]
            assert (zf / zn).min() >= 1.4, (name, k, (zf / zn).min())
    near = scenes.near_mask(scenes.sequence("posts"), 0)
    assert list(np.flatnonzero(np.diff(near[120].astype(int)))) == [31, 35, 58, 63]        # edges 31|32, 35|36, 58|59, 63|64
    assert list(np.flatnonzero(np.diff(near[:, 120].astype(int)))) == [3, 7, 15, 20]        # edges 3|4, 7|8, 15|16, 20|21
    seq = scenes.sequence("stripes")
    _, z = seq.render(0)
    period = scenes.STRIPE_PERIOD / z                  # texels -> px of frame 0 (a texel is 1 / z px at depth z)
    assert 4 <= period.min() and period.max() <= 8.5, (period.min(), period.max())
    row = seq.tex[seq.tex.shape[0] // 2] - seq.tex[seq.tex.shape[0] // 2].mean()

    def corr(lag):
        return float(np.corrcoef(row[lag:], row[:-lag])[0, 1])
    assert corr(scenes.STRIPE_PERIOD) > 0.9 and corr(scenes.STRIPE_PERIOD // 2) < -0.8 and np.abs(row).max() > 40
    seq = scenes.sequence("flat")
    for k in (0, 8, 20):
        assert 0.35 <= scenes.flat_mask(seq, k).mean() <= 0.45, k
    assert synth.semi_dense_fraction(seq.frame(0)) < 0.8 * synth.semi_dense_fraction(synth.Sequence(320, 240, seed=1234).frame(0))
    n = synth.semi_dense_fraction(scenes.sequence("blank").frame(0)) * 320 * 240
    assert 100 < n < 1024, n
    img = scenes.sequence("blank_const").frame(0)
    assert (img == img[0, 0]).all()


def test_empty_cases_are_empty():
    """what the reference did on the blank keyframes: a few hundred pixels drawn and a handful of points on `blank`, nothing
    on `blank_const`, where its SE3 evaluation and overlap are NaN (means over no point)"""
    g = _load()

    def rec(sc, what):
        return g[f"{sc}/empty_keyframe/{what}"]
    assert 100 < int(rec("blank", "selected")) < 1024 and 0 < int(rec("blank", "perma/n")) < 100
    assert int(rec("blank_const", "selected")) == 0 and int(rec("blank_const", "perma/n")) == 0
    assert all(int(rec("blank_const", f"point_cloud/L{lvl}")) == 0 for lvl in (1, 2, 3, 4))
    for lvl in (4, 3, 2, 1):                       # warpedSize, goodCount, badCount 0; pointUsage and every mean 0/0
        ev = rec("blank_const", f"se3_eval/L{lvl}")
        assert (ev[:3] == 0).all() and np.isnan(ev[3:10]).all(), lvl
    assert np.isnan(rec("blank_const", "perma/overlap")).all()
