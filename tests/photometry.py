"""Exposure changes over the synthetic stream.  synth.Sequence renders every frame at the same brightness, so the trackers' affine
brightness model c1 = a * I_ref + b (SE3Tracker.cpp:952, Sim3Tracker.cpp:510) only ever estimates a gain near 1 and an offset
near 0, and the depth map, which compares raw intensities (doLineStereo, propagateDepth), never sees two frames disagree in
brightness.  ExposedSequence renders frame k as clip(rint(g_k * I_k + o_k), 0, 255) with the depth unchanged, with (g_k, o_k)
from one of these schedules (frame 0, the first keyframe, is always at (1, 0)):
  ramp          slow auto-exposure drift, (1 + 0.3 t, -15 t) with t = min(k, 20) / 20: no pixel clipped (frame 0 spans 62..197);
  step          an exposure jump to (1.3, 0) at frame STEP_FRAME: keyframe 0 and the frames tracked on it differ; at most 0.01 %
                of the pixels clipped to 255;
  saturate      (1.5, -10) from frame 2, after (1.25, -5) at frame 1 (frame 1 tracked from the identity at (1.5, -10) is not
                good): 5.4-5.6 % of the pixels clipped to 255 from frame 2;
  dark          frame DARK_FRAME at (0.6, -30), every other frame at (1, 0): there the reference returns trackingWasGood = 0
                without diverging; no pixel clipped;
  ramp_forward  ramp with the forward motion of tests/motions.py.
The reference's tracker (and so the oracle's) does not diverge on any frame a test reads; only the `dark` frame is not good."""
import numpy as np

from lsd_slam_b200 import synth
from tests import motions

STEP_FRAME = 3
DARK_FRAME = 3


def _ramp(k):
    t = min(k, 20) / 20.0
    return 1.0 + 0.3 * t, -15.0 * t


SCHEDULES = {
    "ramp": _ramp,
    "step": lambda k: (1.3, 0.0) if k >= STEP_FRAME else (1.0, 0.0),
    "saturate": lambda k: (1.5, -10.0) if k >= 2 else ((1.25, -5.0) if k == 1 else (1.0, 0.0)),
    "dark": lambda k: (0.6, -30.0) if k == DARK_FRAME else (1.0, 0.0),
    "ramp_forward": _ramp,
}
MOTION = {"ramp_forward": "forward"}          # schedule -> camera motion other than the default


class ExposedSequence(synth.Sequence):
    """synth.Sequence with frame k's image mapped by the schedule's exposure (g_k, o_k); depth and poses are unchanged"""

    def __init__(self, schedule, w=320, h=240):
        m = MOTION.get(schedule, motions.DEFAULT)
        super().__init__(w, h, seed=motions.SEED, xi=synth.DEFAULT_XI if m == motions.DEFAULT else motions.MOTIONS[m])
        self.schedule = schedule
        self.exposure = SCHEDULES[schedule]

    def render(self, k):
        img, depth = super().render(k)
        g, o = self.exposure(k)
        return np.clip(np.rint(g * img.astype(np.float64) + o), 0, 255).astype(np.uint8), depth

    def affine(self, k, ref=0):
        """the true (a, b) of c1 = a * I_ref + b between keyframe `ref` and frame k, clipping aside"""
        (g, o), (gr, orf) = self.exposure(k), self.exposure(ref)
        return g / gr, o - g / gr * orf


Frames = motions.Frames

_streams: dict = {}


def sequence(schedule, w=320, h=240):
    return ExposedSequence(schedule, w, h)


def stream(schedule):
    """(320x240 exposed sequence, lazily rendered frames) of the schedule, shared by every test that reads it"""
    if schedule not in _streams:
        seq = sequence(schedule)
        _streams[schedule] = (seq, Frames(seq))
    return _streams[schedule]
