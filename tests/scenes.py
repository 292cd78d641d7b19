"""Scenes other than synth.Sequence's smooth height field.  The default scene's depth is continuous (z between about 1.5 and 2.5),
nothing in it occludes anything, and its blob texture has no repeated pattern and no large flat area.  So the depth-map decisions
that only come into play at a depth edge -- the occlusion vote of regularizeDepthMap<true> (DepthMap.cpp:826-834), the occluded
source of propagateDepth (:588-601) -- never run on it, doLineStereo's "no clear winner" exit (:1758-1762) runs only by chance,
and no map, tracker or point cloud is ever close to empty.  Each scene below keeps the default camera, the default twist and
320x240, so the pin's and the device's case functions run on it unchanged:
  occluder    a textured fronto-parallel box at z = 1 in front of part of the height field (about 2x the depth behind it),
              covering 15-25 % of every frame a test reads: occluding edges for the regularisers and for propagateDepth;
  posts       thin bars at z = 1, 4-5 px wide, whose edges lie on the device's tile borders in frame 0 (x = 31|32 and 63|64,
              y = 7|8 and 15|16): both the 5x5 regulariser window and the fill-holes halo straddle a depth edge at a CTA border;
  stripes     the height field with a texture periodic along x (STRIPE_PERIOD texels, 4.8-8 px in frame 0): the line stereo
              finds a second-best match close to the best;
  flat        the default texture flattened to a constant on about 40 % of the image, in patches much larger than the 5x5
              windows and a tracker tile: holes the fill-holes pass cannot close, epipolar gradients too small to search;
  blank       frame 0 constant except one textured patch smaller than a 1024-pixel random-init tile, no sensor noise: a map of a
              few hundred pixels;
  blank_const every frame constant: no pixel selected, an empty map, no tracker point, an empty cloud.
Every scene is static; the texture is attached to the world (synth.Sequence.render maps it through world X, Y), so it moves
with the scene from frame to frame."""
import numpy as np

from lsd_slam_b200 import synth
from tests import motions

Z_NEAR = 1.0                                   # the box and the posts
BOX = (-0.45, 0.05, -0.30, 0.14)               # world X0, X1, Y0, Y1 of the box at Z_NEAR
# the posts in frame 0's pixel columns / rows (inclusive); frame 0's camera is the world frame, so a pixel centre u lies on a post
# exactly when (u - cx) / f does at Z_NEAR
POST_COLS = ((32, 35), (59, 63))               # left edge 31|32, right edge 63|64
POST_ROWS = ((4, 7), (16, 20))                 # bottom edge 7|8, top edge 15|16
STRIPE_PERIOD = 12                             # texels along x; a texel is 1 / z px of frame 0, z in 1.5..2.5
FLAT_BLOCK = 80                                # texels per side of a flattened block (about 40 px of frame 0)
FLAT_SEED = 5
BLANK_PATCH = (300, 338, 222, 258)             # texel x0, x1, y0, y1 of blank's textured patch (about 19x18 px of frame 0)
BLANK_LEVEL = 120.0

NAMES = ("occluder", "posts", "stripes", "flat", "blank", "blank_const")


class SceneSequence(synth.Sequence):
    """synth.Sequence at 320x240 with the default twist and seed; a subclass changes the geometry (_near) or the texture"""

    def __init__(self, name, w=320, h=240, noise=1.0):
        super().__init__(w, h, seed=motions.SEED, xi=synth.DEFAULT_XI, noise=noise)
        self.name = name

    def _near(self, X, Y):
        """-> where the ray's point at Z_NEAR (world X, Y) lies on a near object (bool array); none by default"""
        return np.zeros(X.shape, bool)

    def _cast(self, k):
        X, Y, s = super()._cast(k)
        R, t = self.pose(k)
        c = -R.T @ t
        r = self._rays @ R
        sn = (Z_NEAR - c[2]) / r[..., 2]
        Xn, Yn = c[0] + sn * r[..., 0], c[1] + sn * r[..., 1]
        hit = self._near(Xn, Yn) & (sn < s)
        return np.where(hit, Xn, X), np.where(hit, Yn, Y), np.where(hit, sn, s)


class Occluder(SceneSequence):
    """the default scene with a textured fronto-parallel box at z = 1 in front of part of the view"""

    def _near(self, X, Y):
        return (X >= BOX[0]) & (X <= BOX[1]) & (Y >= BOX[2]) & (Y <= BOX[3])


def _post_span(lo, hi, c, f):
    return (lo - 0.5 - c) / f, (hi + 0.5 - c) / f


class Posts(SceneSequence):
    """thin vertical and horizontal bars at z = 1 across the whole view, edges on the device's tile borders in frame 0"""

    def _near(self, X, Y):
        f, cx, cy = float(self.K[0, 0]), float(self.K[0, 2]), float(self.K[1, 2])
        hit = np.zeros(X.shape, bool)
        for lo, hi in POST_COLS:
            a, b = _post_span(lo, hi, cx, f)
            hit |= (X > a) & (X < b)
        for lo, hi in POST_ROWS:
            a, b = _post_span(lo, hi, cy, f)
            hit |= (Y > a) & (Y < b)
        return hit


class Stripes(SceneSequence):
    """the height field with a texture periodic along x: a sine of STRIPE_PERIOD texels over the default texture's slow
    background, so that rows still differ a little"""

    def __init__(self, name, **kw):
        super().__init__(name, **kw)
        x = np.arange(self.tex.shape[1], dtype=np.float32)
        stripe = 60.0 * np.sin(2 * np.pi * x / STRIPE_PERIOD).astype(np.float32)
        self.tex = (0.25 * (self.tex - self.tex.mean()) + 128.0 + stripe[None, :]).astype(np.float32)


def flat_blocks(shape):
    """the flattened texel blocks of `flat`: about 40 % of the FLAT_BLOCK x FLAT_BLOCK blocks, seeded"""
    by, bx = shape[0] // FLAT_BLOCK, shape[1] // FLAT_BLOCK
    sel = np.random.default_rng(FLAT_SEED).random((by, bx)) < 0.4
    return np.kron(sel, np.ones((FLAT_BLOCK, FLAT_BLOCK), bool))


class Flat(SceneSequence):
    """the default texture set to its mean on flat_blocks"""

    def __init__(self, name, **kw):
        super().__init__(name, **kw)
        m = flat_blocks(self.tex.shape)
        self.tex = self.tex.copy()
        self.tex[m] = np.float32(self.tex.mean())


class Blank(SceneSequence):
    """a constant texture with the default texture kept on BLANK_PATCH (none if `const`), rendered without sensor noise"""

    def __init__(self, name, const=False, **kw):
        super().__init__(name, noise=0.0, **kw)
        tex = np.full(self.tex.shape, np.float32(BLANK_LEVEL))
        if not const:
            x0, x1, y0, y1 = BLANK_PATCH
            tex[y0:y1, x0:x1] = self.tex[y0:y1, x0:x1]
        self.tex = tex


def sequence(name, w=320, h=240):
    if name == "occluder":
        return Occluder(name, w=w, h=h)
    if name == "posts":
        return Posts(name, w=w, h=h)
    if name == "stripes":
        return Stripes(name, w=w, h=h)
    if name == "flat":
        return Flat(name, w=w, h=h)
    if name in ("blank", "blank_const"):
        return Blank(name, const=name == "blank_const", w=w, h=h)
    raise KeyError(name)


def near_mask(seq, k):
    """pixels of frame k that see the near object (box or posts)"""
    X, Y, s = synth.Sequence._cast(seq, k)
    Xn, Yn, sn = seq._cast(k)
    return sn < s


def flat_mask(seq, k):
    """pixels of frame k of `flat` whose texture lookup lies wholly inside the flattened blocks (rendered without noise)"""
    ind = SceneSequence("indicator", seq.w, seq.h, noise=0.0)
    ind.tex = flat_blocks(seq.tex.shape).astype(np.float32) * 255
    return ind.render(k)[0] == 255


Frames = motions.Frames

_streams: dict = {}


def stream(name):
    """(320x240 sequence, lazily rendered frames) of the scene, shared by every test that reads it"""
    if name not in _streams:
        seq = sequence(name)
        _streams[name] = (seq, Frames(seq))
    return _streams[name]
