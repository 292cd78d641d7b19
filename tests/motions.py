"""Camera motions other than the synthetic stream's default twist (synth.DEFAULT_XI: mostly sideways, hardly any motion along the
optical axis, almost no roll).  Under the default every epipolar line is close to horizontal and points the same way, the epipole
lies far outside the image, and propagation never lands two sources at inconsistent depths on one pixel.  The twists below (per
frame, [upsilon | omega], Sophus tangent order) make the depth map take the other branches:
  vertical  the y-dominant depth formula of doLineStereo;
  forward   epipole inside the image, search segments clipped at every border, depth ratios outside the rescale gate;
  backward  the same seen from the other side, the near-plane clamp, and propagation collisions;
  roll      epipolar lines at every angle.
The reference's tracker (and so the oracle's) converges on every frame of these streams that a test reads."""
import numpy as np

from lsd_slam_b200 import synth

SEED = 1234

MOTIONS = {
    "vertical": np.array([0.001, 0.004, 0.0005, 0.0008, 0.0004, 0.0002]),
    "forward": np.array([0.0005, 0.0005, 0.015, 0.0002, 0.0002, 0.0005]),
    "backward": np.array([0.0005, 0.0005, -0.015, 0.0002, 0.0002, 0.0005]),
    "roll": np.array([0.003, 0.002, 0.0005, 0.0003, 0.0003, 0.01]),
}


def sequence(name, w=320, h=240):
    return synth.Sequence(w, h, seed=SEED, xi=MOTIONS[name])


class Frames:
    """frame index -> (uint8 image, float32 z-depth) of one sequence, rendered lazily and cached"""

    def __init__(self, seq):
        self.seq, self._cache = seq, {}

    def __getitem__(self, k):
        if k not in self._cache:
            self._cache[k] = self.seq.render(k)
        return self._cache[k]


_streams: dict = {}


def stream(motion):
    """(320x240 sequence, lazily rendered frames) of the motion, shared by every test that reads it"""
    if motion not in _streams:
        seq = sequence(motion)
        _streams[motion] = (seq, Frames(seq))
    return _streams[motion]
