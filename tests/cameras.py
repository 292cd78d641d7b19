"""Cameras other than synth.pinhole_K.  Every other stream of the suite has fx == fy and the principal point at the image centre
((w-1)/2, (h-1)/2): there a kernel that reads fx for fy (or fxi for fyi) gives the same bits, and the per-level principal point
(cx + 0.5) / 2^l - 0.5 (Frame.cpp:449-450) is exact at every level, so its float / double mixing never rounds.  Real cameras are
not like that: the K that UndistorterOpenCV hands to the system for the EuRoC calibration has fx != fy and its principal point
off centre.
CameraSequence renders the stream's scene through the camera below, its rays ((u - cx) / fx, (v - cy) / fy, 1), so that the
ground-truth depth is consistent with K:
  aspect    fx = 1.12 f0, fy = 0.90 f0, principal point centred: separates fx from fy and nothing else;
  offset    fx = fy = f0, principal point off centre by a non-dyadic amount in both axes: cx against cy;
  general   fx = 0.90 f0, fy = 1.10 f0, principal point moved the other way: both at once, and the one camera here whose
            level principal point depends on the precision of the level formula (level_cy_rounds);
  euroc640  (640x480 only) the float32 K of UndistorterOpenCV(EuRoC, 752x480, "full", 640x480).getK(): a wide view,
            fx = 0.54 f0 and fy = 0.64 f0 at that size, principal point (312.09, 248.80).
f0 = 525 W / 640, the focal length of synth.pinhole_K.  Every entry is a float32 value (lsdgpu_create and Frame take float).
The poses, the twist (synth.DEFAULT_XI) and the texture image are those of the default stream.  synth.Sequence.render maps the
world onto that texture through K's fx, cx and cy, so each camera lays it over the scene differently; the scene is still
static, and the 320x240 images keep a semi-dense density inside SURVEY 8d's 30-50 %."""
import numpy as np

from lsd_slam_b200 import synth
from tests import motions

F0_320 = np.float32(525.0 * 320 / 640)

# name -> (w, h, fx, fy, cx, cy), every value a float32
CAMERAS = {
    "aspect": (320, 240, np.float32(1.12 * F0_320), np.float32(0.90 * F0_320), np.float32(159.5), np.float32(119.5)),
    "offset": (320, 240, F0_320, F0_320, np.float32(190.37), np.float32(101.63)),
    "general": (320, 240, np.float32(0.90 * F0_320), np.float32(1.10 * F0_320), np.float32(131.81), np.float32(127.77)),
}
# (w, h, fx, fy, cx, cy) of UndistorterOpenCV(tests/golden/make_golden_opencv_undistort.EUROC, (752, 480), "full",
# (640, 480)).getK() (tests/test_ref_pin_cameras.py checks that it still is)
EUROC640 = (640, 480, np.float32(284.63577), np.float32(333.50217), np.float32(312.0926), np.float32(248.79613))
SMALL = tuple(CAMERAS)                  # the 320x240 cameras of the pin
# `general` under the vertical twist of tests/motions.py: the default twist's epipolar lines are all near horizontal, so only
# this stream reaches the y-dominant depth formula of doLineStereo, where the depth map reads fyi
VERTICAL = "general_vertical"


def level_c(c, level, double=True):
    """(c + 0.5) / 2^level - 0.5 (Frame.cpp:449-450) in double and rounded to float, as the reference does, or all in float"""
    c = np.float32(c)
    if double:
        return np.float32((np.float64(c) + 0.5) / (1 << level) - 0.5)
    return np.float32((c + np.float32(0.5)) / np.float32(1 << level) - np.float32(0.5))


def level_cy_rounds(name):
    """the levels at which the camera's cy comes out differently from the level formula in float and in double.  That needs
    cy + 0.5 to cross a power of two with the lowest bit of cy set: only then does the float sum round, where the double one is
    exact.  An off-centre value alone is not enough (101.63: no level differs)."""
    cy = (EUROC640 if name == "euroc640" else CAMERAS[name])[5]
    return [lv for lv in range(1, 5) if level_c(cy, lv) != level_c(cy, lv, double=False)]


def camera_K(name):
    w, h, fx, fy, cx, cy = EUROC640 if name == "euroc640" else CAMERAS[name]
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


class CameraSequence(synth.Sequence):
    """synth.Sequence of the default scene and motion seen through the camera K (3x3, float32)"""

    def __init__(self, K, w, h, seed=motions.SEED, xi=synth.DEFAULT_XI):
        super().__init__(w, h, seed=seed, xi=xi)
        self.K = np.ascontiguousarray(K, np.float32)
        fx, fy, cx, cy = (float(self.K[i, j]) for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
        self._rays = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], axis=-1)


def sequence(name, K=None):
    """the named camera's sequence (K: another camera at the same size instead, e.g. a perturbed one)"""
    if name == VERTICAL:
        return CameraSequence(camera_K("general") if K is None else K, 320, 240, xi=motions.MOTIONS["vertical"])
    w, h = (EUROC640 if name == "euroc640" else CAMERAS[name])[:2]
    return CameraSequence(camera_K(name) if K is None else K, w, h)


Frames = motions.Frames

_streams: dict = {}


def stream(name):
    """(sequence, lazily rendered frames) of the camera, shared by every test that reads it"""
    if name not in _streams:
        seq = sequence(name)
        _streams[name] = (seq, Frames(seq))
    return _streams[name]
