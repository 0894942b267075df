"""Guided matching from known poses (K9, `csrc/guided_fast.cuh`) against a plain reference and an exact audit.

The engine and oracle/guided_fast_oracle.cpp restate the same geometry (the 3 x 3 product, the cross products, lineToEndPoints,
pixToBucket), so a convention they share cannot fail test_guided_fast.py.  This file adds two checks written from the reference's
source (matching/guidedMatching.hpp:353-460, guidedMatching.cpp:13-70) and not from either restatement:

* `reference()`: the algorithm in Python scalar floats (IEEE double, nothing fused; r1 / r2 rounded through float32, truncation by
  int()), brute force over every (i, j): i is a candidate of j when bucket(i) lies in [start(j), stop(j)); distanceRatio::update in
  ascending j and isValid with the product in double.  The association of F x is a parameter (ASSOCIATIONS);
* `audit()`: for every left i the buckets an evaluation of its line could give, from exact rationals of the line (of the double
  inputs, and of each association's double line), with both end points allowed where the exact residuals are both 0 (neither end
  clamped) or tie in float, and both truncations where a coordinate the reference rounds lies within its rounding bound of an
  integer; the same for every right j's start and stop (exact cross products of x +- n).  Each (i, j) is then a certain or a
  possible candidate, and a result passes when every left i's match, or its absence, is the fold over some candidate set C with
  certain <= C <= possible.

The scenes sit on the edges of this code: image sizes from 2 x 2 to 4000 x 3000, lines through the four corners and ending exactly
on 0, H - 1, inside (H - 1, H) and on H (x likewise), lines with a == 0 or b == 0, residuals that differ in double and tie in float,
ranges that are empty, wrap, start at bucket 0 or end at nb - 1, errorTh = 0, runs of right features without candidates between
ones with 1, 7, 8, 9 or many (the engine's 8-candidate chunks and its search over the candidate offsets), ties in the fold and
bd == distRatio * sbd exactly, every descriptor class (real-valued descriptors are dyadic, so their float sums are exact), views
with and without geometry positions.  Inputs where the reference is undefined (an epipole at infinity, a right feature exactly
at the epipole) are not in them."""
import ctypes as C
import functools
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import guided_fast as gfo
import test_guided_exact as tge
import test_guided_fast as tgf

GF_CAND_CHUNK = 8                  # guided_fast.cuh: consecutive candidates per 4-lane group and step
P3 = np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], np.float64)     # F (x, y, 1) = (1, x, y): the line is chosen by the left point
ID3 = np.eye(3)                                                     # F (x, y, 1) = (x, y, 1): a == 0 at x == 0, b == 0 at y == 0

# How F x is associated: "seq" (F(r,0) x + F(r,1) y) + F(r,2) for every row, what the kernel and the oracle compute; "halving"
# F(r,0) x + (F(r,1) y + F(r,2)) for every row, Eigen's scalar redux unroller on a strided row; "packet" rows 0 and 1 as "seq"
# and row 2 as "halving", Eigen's lazy 3 x 3 product assigned with SSE2 packets of 2 doubles (rows 0-1 a packet, row 2 the
# scalar tail).  See DESIGN.md (K9) for which one the engine uses and why.
ASSOCIATIONS = ("seq", "halving", "packet")
KERNEL_ASSOCIATION = "seq"


def _f32(v):
    return float(np.float32(v))


def _div(a, b):
    """IEEE a / b (Python raises on a division by 0)."""
    if b != 0:
        return a / b
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


# ---------------------------------------------------------------------------------------------- scenes
class FastScene:
    """One pair: left / right descriptors and positions, F (x_R^T F x_L = 0), epipole2 (not normalised), the right image size,
    errorTh and distRatio (already squared).  Positions: geometry positions (double) when `geometry`, else the float upload
    positions widened."""

    def __init__(self, name, kind, F, ep2, W, H, th, ratio, dl, xl, dr, xr, geometry, props=()):
        self.name, self.kind = name, kind
        self.F, self.ep2 = np.asarray(F, np.float64).reshape(3, 3), np.asarray(ep2, np.float64).reshape(3)
        self.W, self.H, self.th, self.ratio = int(W), int(H), float(th), float(ratio)
        self.dl, self.dr = np.ascontiguousarray(dl), np.ascontiguousarray(dr)
        xl, xr = np.asarray(xl, np.float64).reshape(-1, 2), np.asarray(xr, np.float64).reshape(-1, 2)
        self.xl, self.xr = np.ascontiguousarray(xl, np.float32), np.ascontiguousarray(xr, np.float32)
        if geometry:
            self.gl, self.gr = np.ascontiguousarray(xl), np.ascontiguousarray(xr)
            self.pl, self.pr = self.gl, self.gr
        else:
            self.gl = self.gr = None
            self.pl, self.pr = self.xl.astype(np.float64), self.xr.astype(np.float64)
        self.ml, self.mr, self.binary, self.props = len(self.dl), len(self.dr), kind == "bin", props
        self.nb = 2 * (self.W + self.H - 2)
        assert len(self.xl) == self.ml and len(self.xr) == self.mr

    @functools.cached_property
    def dist(self):
        """Regions::SquaredDescriptorDistance of every (i, j): exact integers (uchar, integer-valued fp32, binary) or exact dyadic
        float sums (real-valued fp32, and the mixed pair's fp32 expansion)."""
        ii, jj = np.meshgrid(np.arange(self.ml), np.arange(self.mr), indexing="ij")
        d = tge.distances(self, ii.ravel(), jj.ravel()).reshape(self.ml, self.mr) if self.ml and self.mr else np.zeros((self.ml, self.mr))
        if self.kind in ("real", "mixed"):
            a, b = self.dl.astype(np.float64)[:, None, :], self.dr.astype(np.float64)[None, :, :]
            assert np.array_equal(d, ((a - b) ** 2).sum(2)), f"{self}: a float descriptor sum is not exact"
        return d

    @functools.cached_property
    def classes(self):
        return classify(self)

    def __repr__(self):
        return self.name


def _descriptors(kind, owner, rng, ml):
    """Left descriptors and right ones (a noisy copy of left owner[j], or a fresh one where owner[j] < 0).  Real-valued ones are
    quarter steps in [0, 64): every partial float sum of their squared differences is exact."""
    if kind == "bin":
        dl = rng.integers(0, 256, (ml, 64), dtype=np.uint8)
        flips = np.packbits(rng.random((len(owner), 512)) < 0.05, axis=1, bitorder="little")
        dr = np.where((owner >= 0)[:, None], dl[np.maximum(owner, 0)] ^ flips, rng.integers(0, 256, (len(owner), 64), dtype=np.uint8))
        return dl, dr.astype(np.uint8)
    top = 256 if kind in ("u8", "f32") else 64
    dl = rng.integers(0, top, (ml, 128))
    noisy = np.clip(dl[np.maximum(owner, 0)] + rng.integers(-6, 7, (len(owner), 128)), 0, top - 1)
    dr = np.where((owner >= 0)[:, None], noisy, rng.integers(0, top, (len(owner), 128)))
    if kind == "u8":
        return dl.astype(np.uint8), dr.astype(np.uint8)
    dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    if kind in ("real", "mixed"):
        q = rng.integers(-1, 2, dr.shape).astype(np.float32) * 0.25
        dr = np.clip(dr + q, 0, top - 0.25).astype(np.float32)
    if kind == "real":
        dl = np.clip(dl + rng.integers(-1, 2, dl.shape).astype(np.float32) * 0.25, 0, top - 0.25).astype(np.float32)
    return dl, dr


def _cross(e, x, y):
    """Eigen's Vector3::cross(e, (x, y, 1)) in the number type of x, y."""
    return e[1] * 1 - e[2] * y, e[2] * x - e[0] * 1, e[0] * y - e[1] * x


def edge_scene(W, H, flip, kind="u8", geometry=True, seed=0):
    """F = P3, so left point (x, y) has the line (1, x, y) (negated when ep2(2) > 0).  Left points are chosen so the line ends
    exactly on ya = 0, H - 1, H - 1/2, H and xb = 0, W - 1, W - 1/2, W, passes through each corner, or has residuals that differ
    in double and tie in float; right features sit around the border near every end point, with the epipole inside the image, so
    that ranges of a few buckets start and stop all around every left bucket."""
    rng = np.random.default_rng(seed + 17 * W + H)
    s = -1.0 if flip else 1.0
    left = []
    for b in (1.0, -1.0, 0.5, -0.5, 2.0, -3.0, 0.25, -0.125):
        xa = 0.0 if s * b < 0 else W - 1.0                     # the vertical border the normalised line (s, s b, s c) meets
        for ya in (0.0, H - 1.0, H - 0.5, float(H), 0.5, H / 2.0):
            left.append((b, -(b * ya + xa)))
        for cx, cy in ((0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1)):
            left.append((b, -(cx + b * cy)))                   # through the corner: cx + b cy + c == 0
    for xb in (0.0, W - 1.0, W - 0.5, float(W), W / 2.0):
        for b in (1.0, -1.0, 4.0):
            left.append((b, -xb))                                # yb = 0 (or H - 1): x = -(b yb + c)
            left.append((b, -xb - b * (H - 1)))
    # residuals that differ in double and tie in float: a line of slope 2^-30 passing 1024 px beside the image, both end points
    # clamped to two corners of one side, r1 and r2 1024 and 1024 -+ 2^-30 (H - 1)
    for b in (2.0 ** -30, -2.0 ** -30):
        for c in (-(W - 1.0) - 1024, 1024.0, W - 1.0 + 1024, -1024.0):
            left.append((b, c))
    xl = np.array(left, np.float64)
    if not geometry:
        xl = xl[np.all(xl == xl.astype(np.float32), 1)]
    e = np.array([W / 2.0 + 0.375, H / 2.0 - 0.125, 1.0])
    ep2 = e * (2.0 if flip else -0.5)                            # ep2(2) > 0 makes the reference negate F and ep2
    # right features: near the border, around every left line's two end points and the corners, 0 .. 3 px inside
    pts = []
    for x, y in [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1)]:
        pts.append((x, y))
    for b, c in xl:
        a_, b_, c_ = s, s * b, s * c
        xa = 0.0 if b_ < 0 else W - 1.0
        yb = H - 1.0 if a_ < 0 else 0.0
        pts.append((xa, min(max(-(a_ * xa + c_) / b_, 0.0), H - 1.0)))
        pts.append((min(max(-(b_ * yb + c_) / a_, 0.0), W - 1.0), yb))
    pts = np.array(pts)
    xr = []
    for p in pts:
        d = e[:2] - p
        d = d / max(np.hypot(*d), 1e-9)
        for t in (0.0, 0.75, 2.5):
            q = p + t * d + rng.uniform(-1.0, 1.0, 2) * min(2.0, (min(W, H) - 1) / 2.0)
            xr.append(np.clip(q, 0.0, [W - 1.0, H - 1.0]))
    xr = np.round(np.array(xr) * 64) / 64
    xr = xr[np.hypot(xr[:, 0] - e[0], xr[:, 1] - e[1]) > 0]
    dists = rng.permutation(np.arange(10, 10 + 3 * len(xr)))[:len(xr)]
    dists[rng.choice(len(xr), len(xr) // 8, replace=False)] = 40          # ties of the best distance
    dl = np.zeros((len(xl), 128), np.uint8)
    dr = tge.at_distances(dists)
    if kind == "f32":
        dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    name = f"edge.{W}x{H}.{'flip' if flip else 'noflip'}.{kind}.{'geometry' if geometry else 'upload'}"
    return FastScene(name, kind, P3, ep2, W, H, 2.25, 0.64, dl, xl, dr, xr, geometry, props=("edge",))


def zero_coeff_scene():
    """F = I: line (x, y, 1): a == 0 at x == 0 (no end points), b == 0 at y == 0 (no end points), and ordinary lines."""
    W, H = 640, 480
    xl = np.array([[0.0, -0.002], [0.0, 0.003], [0.004, 0.0], [-0.001, 0.0], [0.0, 0.0], [-1 / 512, -1 / 256], [-1 / 300, -1 / 250],
                   [-1 / 600, -1 / 128], [-0.0025, -0.003]])
    e = np.array([320.25, 240.5, 1.0])
    rng = np.random.default_rng(4)
    xr = np.c_[rng.uniform(0, W - 1, 400), rng.uniform(0, H - 1, 400)]
    dr = tge.at_distances(rng.permutation(np.arange(5, 405)))
    return FastScene("zero_coeff", "u8", ID3, -e, W, H, 16.0, 0.64, np.zeros((len(xl), 128), np.uint8), xl, dr, xr, True,
                     props=("zero",))


def structure_scene(kind="u8", geometry=True, ratio=0.64):
    """F = [e]_x, the epipole far to the left: the left point p and a right point at p share their epipolar line.  Left features
    come in groups of identical positions (one bucket each), 48 px apart; each group has two or three right features on its line
    (candidates: the whole group), and filler right features between the groups have none.  Group sizes 1, 7, 8, 9, 100, ... put
    candidate runs on and across the 8-candidate chunks; the groups' distances hold ties of the best (matched only when
    distRatio > 1), sbd == bd, bd == distRatio * sbd exactly and bd between the float and the double product."""
    W, H = 1920, 1080
    e = np.array([-6000.5, 540.375, 1.0])
    Fx = np.array([[0, -e[2], e[1]], [e[2], 0, -e[0]], [-e[1], e[0], 0]])
    sizes = [1, 7, 8, 9, 100, 2, 16, 17, 3, 24, 5, 1, 9, 8, 7, 33, 2, 64, 6, 15]
    hits = tge.ratio_triples(ratio)[1]
    (be, se), (bf, sf) = hits["exact"][0], (hits["float"] or hits["exact"])[0]    # bd == ratio * sbd; float and double products split
    menus = [[10, 100, 400], [50, 50, 80], [40, 40], [be, se, se + 9], [be + 1, se], [max(be - 1, 0), se], [7, 7, 7], [300, 12, 90],
             [bf, sf], [max(bf - 1, 0), sf, sf + 3]]
    rng = np.random.default_rng(7)
    xl, xr, dists = [], [], []
    fill = 0
    for g, n in enumerate(sizes):
        p = (960.0 + 13.0 * g, 60.0 + 48.0 * g)
        xl += [p] * n
        for k in range(rng.integers(1, 6)):                             # fillers: no left feature within reach
            xr.append((700.0 + 5.0 * k, p[1] + 24.0)); dists.append(1 + fill % 3); fill += 1
        for k, d in enumerate(menus[g % len(menus)]):
            xr.append((p[0] + 37.0 * k - 20.0, p[1] + (p[1] - e[1]) * (37.0 * k - 20.0) / (p[0] - e[0]))); dists.append(d)
    xl = np.array(xl)[rng.permutation(len(xl))]
    dl = np.zeros((len(xl), 128), np.uint8)
    dr = tge.at_distances(dists)
    if kind == "f32":
        dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    return FastScene(f"structure.{kind}.{ratio}.{'geometry' if geometry else 'upload'}", kind, -Fx, e * 3.0, W, H, 4.0, ratio, dl, xl, dr,
                     np.array(xr), geometry, props=("structure",))


def random_scene(kind, W, H, e, th, seed, geometry=True, ml=160, mr=220, tag=""):
    """A general F = [e]_x A (A: a near-identity affine map), left points anywhere in the image and right ones near their epipolar
    lines; descriptors of the class `kind`, one noisy copy of each left descriptor on its line."""
    rng = np.random.default_rng(seed)
    A = np.array([[1.0 + rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(-9, 9)],
                  [rng.uniform(-0.05, 0.05), 1.0 + rng.uniform(-0.05, 0.05), rng.uniform(-9, 9)], [0.0, 0.0, 1.0]])
    e = np.asarray(e, np.float64)
    ex = np.array([[0, -1.0, e[1]], [1.0, 0, -e[0]], [-e[1], e[0], 0]])
    F = ex @ A
    xl = np.c_[rng.uniform(0, W - 1, ml), rng.uniform(0, H - 1, ml)]
    owner = rng.integers(0, ml, mr)
    q = (np.c_[xl[owner], np.ones(mr)] @ A.T)[:, :2]
    t = rng.uniform(-0.6, 0.6, mr)
    xr = np.clip(e[:2] + (q - e[:2]) * (1 + t[:, None]), [0, 0], [W - 1, H - 1]) + rng.uniform(-1.5, 1.5, (mr, 2))
    xr = xr[np.hypot(*(xr - e[:2]).T) > 1e-3]
    owner = owner[:len(xr)]
    desc_owner = np.where(rng.random(len(xr)) < 0.5, owner, -1)
    dl, dr = _descriptors(kind, desc_owner, rng, ml)
    sign = 1.0 if seed % 2 else -1.0                             # ep2(2) of either sign, F to match
    return FastScene(f"random.{kind}.{W}x{H}{tag}.{'geometry' if geometry else 'upload'}", kind, -sign * F, sign * e * 1.5, W, H, th,
                     0.64, dl, xl, dr, xr, geometry, props=("random",))


def tiny_scene(W, H, seed):
    """2 x 2 to 5 x 4 images: nb = 4 .. 14 buckets, every feature on or next to the border."""
    rng = np.random.default_rng(seed)
    e = np.array([(W - 1) / 2 + 0.125, (H - 1) / 2 - 0.0625, 1.0])
    xl = np.round(np.c_[rng.uniform(0, W - 1, 40), rng.uniform(0, H - 1, 40)] * 16) / 16
    xr = np.round(np.c_[rng.uniform(0, W - 1, 60), rng.uniform(0, H - 1, 60)] * 16) / 16
    xr = xr[np.hypot(*(xr - e[:2]).T) > 0]
    ex = np.array([[0, -1.0, e[1]], [1.0, 0, -e[0]], [-e[1], e[0], 0]])
    dl = np.zeros((40, 128), np.uint8)
    dr = tge.at_distances(rng.permutation(np.arange(3, 3 + len(xr))))
    return FastScene(f"tiny.{W}x{H}", "u8", ex, -e, W, H, 0.09, 0.64, dl, xl, dr, xr, True, props=("tiny",))


def association_scene():
    """Left lines that pass within 4 px of the bottom-right corner of a 4000 x 3000 image (both end points close to the corner and
    unclamped, so rounding noise picks one), with a general F = [e]_x A, kept where the "seq" and "halving" products put the left
    feature into different buckets; two right features near the corner whose range holds the "seq" bucket and not the "halving"
    one.  The two associations give different lists here."""
    W, H = 4000, 3000
    rng = np.random.default_rng(11)
    e = np.array([-5000.3, 1500.2, 1.0])
    A = np.array([[1.013, 0.021, 3.7], [-0.017, 0.991, -2.3], [0.0, 0.0, 1.0]])
    F = np.array([[0, -1.0, e[1]], [1.0, 0, -e[0]], [-e[1], e[0], 0]]) @ A
    Fl = [float(v) for v in F.reshape(9)]
    xl, xr = [], []
    for _ in range(4000):
        q = np.array([W - 1 - rng.uniform(0, 4), H - 1 - rng.uniform(0, 4)])
        p = np.linalg.solve(A, np.r_[e[:2] + rng.uniform(0.55, 0.95) * (q - e[:2]), 1.0])[:2]
        if not (0 <= p[0] <= W - 1 and 0 <= p[1] <= H - 1):
            continue
        bs = {a: _end_bucket(*_line(Fl, float(p[0]), float(p[1]), a), W, H) for a in ("seq", "halving")}
        if bs["seq"] < 0 or bs["seq"] == bs["halving"]:
            continue
        found = []
        for _ in range(200):
            r = e[:2] + rng.uniform(0.8, 0.999) * (q - e[:2]) + rng.uniform(-1, 1, 2)
            if not (0 <= r[0] <= W - 1 and 0 <= r[1] <= H - 1):
                continue
            rg = _right_range([e[0], e[1], 1.0], float(r[0]), float(r[1]), W, H, 0.25)
            if rg and rg[0] <= bs["seq"] < rg[1] and not rg[0] <= bs["halving"] < rg[1]:
                found.append(r)
                if len(found) == 2:
                    break
        if len(found) < 2:
            continue
        xl.append(p)
        xr += found
        if len(xl) == 12:
            break
    assert xl, "no left feature whose bucket depends on the association"
    # left k: 100 in component k; its two right features: distance 1 and 64 to it, at least 2 x 100^2 to every other left feature
    dl = np.zeros((len(xl), 128), np.uint8)
    dl[np.arange(len(xl)), np.arange(len(xl))] = 100
    dr = np.repeat(dl, 2, axis=0)
    dr[:, 127] = np.tile([1, 8], len(xl))
    return FastScene("association", "u8", -F, 2 * e, W, H, 0.25, 0.64, dl, np.array(xl), dr, np.array(xr), True, props=("association",))


@functools.lru_cache(maxsize=None)
def scenes():
    out = []
    for W, H in ((2, 2), (3, 2), (2, 5), (7, 4), (640, 480), (4000, 3000)):
        for flip in (False, True):
            out.append(edge_scene(W, H, flip))
    out.append(edge_scene(640, 480, False, kind="f32", geometry=False))
    out.append(edge_scene(1920, 1080, True, geometry=False))
    out.append(zero_coeff_scene())
    out += [structure_scene("u8"), structure_scene("f32", geometry=False), structure_scene("u8", ratio=1.5)]
    for k, kind in enumerate(("u8", "f32", "real", "mixed", "bin")):
        out.append(random_scene(kind, 640, 480, (300.5 + 7 * k, 200.25, 1.0), 9.0, 20 + k, geometry=(k % 2 == 0)))
    out.append(random_scene("u8", 4000, 3000, (-8000.5, 1400.0, 1.0), 16.0, 31, geometry=False, tag=".outside"))
    out.append(random_scene("u8", 1920, 1080, (960.5, 540.5, 1.0), 0.0, 32, tag=".th0"))
    out.append(random_scene("bin", 1920, 1080, (100.5, 1000.5, 1.0), 400.0, 33, tag=".wide"))
    out += [tiny_scene(2, 2, 1), tiny_scene(3, 2, 2), tiny_scene(5, 4, 3)]
    out.append(association_scene())
    return tuple(out)


# ---------------------------------------------------------------------------------------------- the reference, in Python floats
def _line(F, x, y, assoc):
    """F * Vec3(x, y, 1.) in the association `assoc` (F: 9 floats, row-major)."""
    out = []
    for r in range(3):
        v0, v1, v2 = F[3 * r] * x, F[3 * r + 1] * y, F[3 * r + 2] * 1.0
        out.append(v0 + (v1 + v2) if assoc == "halving" or (assoc == "packet" and r == 2) else (v0 + v1) + v2)
    return out


def _pix_to_bucket(x, y, W, H, mutation=None):
    """guidedMatching.cpp:13-22."""
    if y == 0:
        return x
    if x == W - 1:
        return W - 1 + y
    if y == H - 1:
        return 2 * W + H - 3 - x
    return 2 * (W + H - 2) - y - (1 if mutation == "left border off by one" else 0)


def _end_bucket(a, b, c, W, H, mutation=None):
    """lineToEndPoints (guidedMatching.cpp:24-70) and pixToBucket(x0.cast<int>()); -1: no end points (and a non-finite line,
    where the reference is undefined)."""
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return -1
    if b == 0:
        return -1
    x = 0.0 if b < 0 else float(W - 1)
    y = -(a * x + c) / b
    if y < 0:
        y = 0.0
    elif (y > H) if mutation == "> H" else (y >= H):
        y = float(H - 1)
    r1 = _f32(abs(a * x + b * y + c))
    x0 = (x, y)
    if a == 0:
        return -1
    y = float(H - 1) if a < 0 else 0.0
    x = -(b * y + c) / a
    if x < 0:
        x = 0.0
    elif x >= W:
        x = float(W - 1)
    r2 = _f32(abs(a * x + b * y + c))
    if r1 > r2:
        x0 = (x, y)
    return _pix_to_bucket(int(x0[0]), int(x0[1]), W, H, mutation)


def _normalised(sc, mutation=None):
    F = [float(v) for v in (sc.F.T if mutation == "F transposed" else sc.F).reshape(9)]
    e = [float(v) for v in sc.ep2]
    if e[2] > 0.0 and mutation != "sign normalisation dropped":
        F, e = [-v for v in F], [-v for v in e]
    e2 = e[2]
    return F, [_div(v, e2) for v in e]


def _right_range(e, x, y, W, H, th, mutation=None):
    """(bucketStart, bucketStop) of a right feature (guidedMatching.hpp:416-433), None where either line has no end points."""
    l0, l1, _ = _cross(e, x, y)
    s = _div(math.sqrt(th) if th >= 0 else math.nan, math.sqrt(l0 * l0 + l1 * l1))
    n0, n1 = l0 * s, l1 * s
    start = _end_bucket(*_cross(e, x - n0, y - n1), W, H, mutation)
    if start < 0:
        return None
    stop = _end_bucket(*_cross(e, x + n0, y + n1), W, H, mutation)
    return None if stop < 0 else (start, stop)


def left_buckets(sc, assoc=KERNEL_ASSOCIATION, mutation=None):
    F, _ = _normalised(sc, mutation)
    return np.array([_end_bucket(*_line(F, float(x), float(y), assoc), sc.W, sc.H, mutation) for x, y in sc.pl], np.int64)


def right_ranges(sc, mutation=None):
    _, e = _normalised(sc, mutation)
    return [_right_range(e, float(x), float(y), sc.W, sc.H, sc.th, mutation) for x, y in sc.pr]


def reference(sc, assoc=KERNEL_ASSOCIATION, mutation=None):
    """guidedMatchingFundamentalFast: matches[MATCH_DTYPE] in ascending i.  Brute force: i is a candidate of j when bucket(i) lies
    in [start(j), stop(j)) and stop(j) > start(j); each i folds its candidates in ascending j."""
    lb = left_buckets(sc, assoc, mutation)
    cand = np.zeros((sc.ml, sc.mr), bool)
    for j, rg in enumerate(right_ranges(sc, mutation)):
        if rg is None:
            continue
        s, t = rg
        if mutation == "stop inclusive":
            t += 1
        if t > s:
            cand[:, j] = (lb >= s) & (lb < t)
        elif mutation == "wrapping ranges accepted" and t < s:
            cand[:, j] = (lb >= 0) & ((lb >= s) | (lb < t))
    out = []
    for i in range(sc.ml):
        js = np.flatnonzero(cand[i])
        k = tge.fold(sc.dist[i, js].tolist(), js.tolist(), sc.ratio, mutation == "ratio product in float",
                     mutation == "largest j on ties") if len(js) else -1
        if k >= 0:
            out.append((i, k))
    return tge._matches(out)


# ---------------------------------------------------------------------------------------------- the exact audit
def _border_index(x, y, W, H):
    """The bucket of border pixel (x, y): its position on a clockwise walk of the border from (0, 0) - the top row, the right column,
    the bottom row, the left column, a corner counted on the first of these that reaches it."""
    if y == 0:
        return x
    if x == W - 1:
        return (W - 1) + y
    if y == H - 1:
        return (W - 1) + (H - 1) + (W - 1 - x)
    return 2 * (W - 1) + (H - 1) + (H - 1 - y)


def _truncations(v, tol, hi):
    """The integer parts the reference can give a coordinate whose exact value is v, rounded by at most tol, clamped to [0, hi]."""
    lo_i, hi_i = math.floor(v - tol), math.floor(v + tol)
    return set(range(max(lo_i, 0), min(hi_i, hi) + 1)) or {min(max(math.floor(v), 0), hi)}


_ROUND = Fraction(1, 1 << 49)      # four double roundings, with room


def _exact_ends(A, B, C, W, H, noisy):
    """Every bucket an evaluation of lineToEndPoints on the exact line (A, B, C) can give, where `noisy` says whether the double
    operations on it may round: the end point on the vertical border x = 0 (b < 0) or W - 1 and the one on the horizontal border
    y = H - 1 (a < 0) or 0, each clamped to the image; the one whose residual is smaller, and both when the exact residuals are
    both 0 (neither is clamped: the reference's choice is rounding noise) or tie after rounding to float; each coordinate truncated,
    both ways when it lies within the rounding bound of an integer.  -1: no end points."""
    if A == 0 or B == 0:
        return {-1}
    xa = 0 if B < 0 else W - 1
    yb = H - 1 if A < 0 else 0
    ya = -(A * xa + C) / B
    xb = -(B * yb + C) / A
    tol_y = _ROUND * (abs(A) * xa + abs(C)) / abs(B) if noisy else 0
    tol_x = _ROUND * (abs(B) * yb + abs(C)) / abs(A) if noisy else 0
    ya_c = 0 if ya < 0 else (H - 1 if ya >= H else ya)
    xb_c = 0 if xb < 0 else (W - 1 if xb >= W else xb)
    r1, r2 = abs(A * xa + B * ya_c + C), abs(A * xb_c + B * yb + C)
    tol_r = _ROUND * (abs(A) * W + abs(B) * H + abs(C)) if noisy else 0
    f1, f2 = _f32(float(r1)), _f32(float(r2))
    take0 = r1 <= r2 + tol_r or f1 <= f2
    take1 = r1 + tol_r > r2 and (f1 >= f2 or tol_r > 0)
    if r1 == 0 and r2 == 0:
        take0 = take1 = True
    out = set()
    if take0:
        ys = {int(ya_c)} if ya_c in (0, H - 1) and ya != ya_c else _truncations(ya_c, tol_y, H - 1)
        out |= {_border_index(xa, y, W, H) for y in ys}
    if take1:
        xs = {int(xb_c)} if xb_c in (0, W - 1) and xb != xb_c else _truncations(xb_c, tol_x, W - 1)
        out |= {_border_index(x, yb, W, H) for x in xs}
    return out


def _possible_left(sc):
    """Per left i, the set of buckets (-1: none) under any association: the exact line of the double inputs (whose sign and zero
    pattern every double evaluation must share, else every bucket is possible) and each association's double line, taken
    exactly."""
    F, _ = _normalised(sc)
    Fq = [Fraction(v) for v in F]
    allb = set(range(sc.nb)) | {-1}
    out = []
    for x, y in sc.pl:
        x, y = float(x), float(y)
        X, Y = Fraction(x), Fraction(y)
        L = [Fq[3 * r] * X + Fq[3 * r + 1] * Y + Fq[3 * r + 2] for r in range(3)]
        dbl = [_line(F, x, y, a) for a in ASSOCIATIONS]
        if not all(math.isfinite(v) for d in dbl for v in d):
            out.append(allb)
            continue
        exact = all(Fraction(v) == L[r] for d in dbl for r, v in enumerate(d))
        if any((v > 0) != (L[r] > 0) or (v == 0) != (L[r] == 0) for d in dbl for r, v in enumerate(d)):
            out.append(allb)
            continue
        P = _exact_ends(L[0], L[1], L[2], sc.W, sc.H, not exact)
        for d in dbl:
            P |= _exact_ends(Fraction(d[0]), Fraction(d[1]), Fraction(d[2]), sc.W, sc.H, True)
        out.append(P)
    return out


def _possible_right(sc):
    """Per right j, (starts, stops): the buckets of the lines ep2 x (x -+ n, 1), from the exact cross products of the double
    positions x -+ n (exact and as the reference rounds them) with n = l sqrt(errorTh) / |l| in double and one ulp either side."""
    _, e = _normalised(sc)
    eq = [Fraction(v) for v in e]
    out = []
    for x, y in sc.pr:
        x, y = float(x), float(y)
        l0, l1, _ = _cross(e, x, y)
        s = _div(math.sqrt(sc.th), math.sqrt(l0 * l0 + l1 * l1))
        ends = []
        for sign in (-1, 1):
            sets = set()
            for n0 in {l0 * s, math.nextafter(l0 * s, -math.inf), math.nextafter(l0 * s, math.inf)}:
                for n1 in {l1 * s, math.nextafter(l1 * s, -math.inf), math.nextafter(l1 * s, math.inf)}:
                    px, py = x + sign * n0, y + sign * n1                       # as the reference rounds x -+ n
                    for qx, qy in ((Fraction(px), Fraction(py)), (Fraction(x) + sign * Fraction(n0), Fraction(y) + sign * Fraction(n1))):
                        lq = _cross(eq, qx, qy)
                        sets |= _exact_ends(*lq, sc.W, sc.H, True)
            ends.append(sets)
        out.append(tuple(ends))
    return out


def classify(sc):
    """(certain, possible) candidate matrices [ml, mr]: certain when every allowed bucket of i, start and stop of j give
    start <= bucket < stop; possible when one combination does."""
    P, R = _possible_left(sc), _possible_right(sc)
    certain = np.zeros((sc.ml, sc.mr), bool)
    possible = np.zeros((sc.ml, sc.mr), bool)
    smin = np.array([min((v for v in s if v >= 0), default=10 ** 9) for s, _ in R])
    smax = np.array([max(s) if -1 not in s else 10 ** 9 for s, _ in R])
    tmin = np.array([min(t) if -1 not in t else -1 for _, t in R])
    tmax = np.array([max(t) for _, t in R])
    for i, Pi in enumerate(P):
        bs = [b for b in Pi if b >= 0]
        for b in bs:
            possible[i] |= (smin <= b) & (b < tmax)
        if len(Pi) == 1 and bs:
            certain[i] = (smax <= bs[0]) & (bs[0] < tmin)
    assert not (certain & ~possible).any()
    return certain, possible, P, R


def _reachable(d, cert, opt, ratio, got):
    """Is `got` (a j, or -1) the distanceRatio fold of some C with cert <= C <= cert + opt?  d: distance by j."""
    key = lambda j: (d[j], j)
    if got >= 0:
        if got not in cert and got not in opt:
            return False
        if any(key(j) < key(got) for j in cert):
            return False
        rest = [d[j] for j in cert if j != got]
        if rest:
            sbd = min(rest)                    # C = cert + {got}: the largest second distance any allowed C has
        else:
            extra = [d[j] for j in opt if j != got and key(j) > key(got)]
            if not extra:
                return False
            sbd = max(extra)
        return d[got] < ratio * sbd
    if len(cert) <= 1:
        return True                            # C = cert: fewer than two distances
    # No match: some C whose two smallest distances m1 <= m2 give m1 >= ratio * m2.  Every C holds the certain c1 <= c2, so m1 is c1
    # or an optional value <= c1; m2 is then the smallest other member C must or may hold: with m1 = c1, c2 or an optional value
    # in [c1, c2]; with an optional m1, c1 or another optional value in [m1, c1].  A smaller m2 only helps (ratio >= 0).
    c1, c2 = sorted(d[j] for j in cert)[:2]
    ov = [d[j] for j in opt]
    firsts = [(c1, None)] + [(v, k) for k, v in enumerate(ov) if v <= c1]
    for m1, k1 in firsts:
        hi = c2 if k1 is None else c1
        m2 = min([hi] + [v for k, v in enumerate(ov) if k != k1 and m1 <= v <= hi])
        if not m1 < ratio * m2:
            return True
    return False


def audit(result, sc):
    """One match per left feature in ascending i, and each left i's match (or none) reachable by the fold over a candidate set between
    its certain and its possible candidates."""
    i, j = np.asarray(result["i"], np.int64), np.asarray(result["j"], np.int64)
    assert np.all(np.diff(i) > 0), f"{sc}: not one match per left feature in ascending i"
    assert len(i) == 0 or (i[-1] < sc.ml and j.max() < sc.mr and i[0] >= 0), f"{sc}: index out of range"
    got = np.full(sc.ml, -1, np.int64)
    got[i] = j
    certain, possible, _, _ = sc.classes
    for r in range(sc.ml):
        cert = np.flatnonzero(certain[r]).tolist()
        opt = np.flatnonzero(possible[r] & ~certain[r]).tolist()
        assert _reachable(sc.dist[r], cert, opt, sc.ratio, int(got[r])), \
            f"{sc}: left {r} matched {got[r]}; certain candidates {cert[:8]}, possible {opt[:8]}"


# ---------------------------------------------------------------------------------------------- CPU tests
MUTATIONS = ("F transposed", "sign normalisation dropped", "> H", "stop inclusive", "wrapping ranges accepted", "largest j on ties",
             "ratio product in float", "left border off by one")


def _same(a, b):
    return len(a) == len(b) and np.array_equal(a["i"], b["i"]) and np.array_equal(a["j"], b["j"])


def test_scenes_reach_their_edges(record_property):
    """Each construction reaches the edge it names, decided in exact arithmetic."""
    seen = set()
    for sc in scenes():
        assert sc.ep2[2] != 0, sc
        F, e = _normalised(sc)
        eq = [Fraction(v) for v in e]
        for x, y in sc.pr:                                                      # no right feature at the epipole
            assert _cross(eq, Fraction(float(x)), Fraction(float(y)))[:2] != (0, 0), sc
        Fq = [Fraction(v) for v in F]
        W, H = sc.W, sc.H
        for x, y in sc.pl:
            X, Y = Fraction(float(x)), Fraction(float(y))
            A, B, Cc = (Fq[3 * r] * X + Fq[3 * r + 1] * Y + Fq[3 * r + 2] for r in range(3))
            if A == 0:
                seen.add("a == 0")
            if B == 0:
                seen.add("b == 0")
            if A == 0 or B == 0:
                continue
            for cx, cy, nm in ((0, 0, "corner 0,0"), (W - 1, 0, "corner W-1,0"), (0, H - 1, "corner 0,H-1"), (W - 1, H - 1, "corner W-1,H-1")):
                if A * cx + B * cy + Cc == 0:
                    seen.add(f"{nm}.{W}x{H}")
            ya = -(A * (0 if B < 0 else W - 1) + Cc) / B
            xb = -(B * (H - 1 if A < 0 else 0) + Cc) / A
            for v, lim, ax in ((ya, H, "ya"), (xb, W, "xb")):
                if v == 0:
                    seen.add(f"{ax} == 0")
                if v == lim - 1:
                    seen.add(f"{ax} == {ax}max - 1")
                if lim - 1 < v < lim:
                    seen.add(f"{ax} in (max - 1, max)")
                if v == lim:
                    seen.add(f"{ax} == max")
            dl = _line(F, float(x), float(y), KERNEL_ASSOCIATION)
            a, b, c = dl
            if b != 0 and a != 0:
                xa = 0.0 if b < 0 else W - 1.0
                y1 = min(max(-(a * xa + c) / b, 0.0), H - 1.0)
                yb = H - 1.0 if a < 0 else 0.0
                x1 = min(max(-(b * yb + c) / a, 0.0), W - 1.0)
                r1, r2 = abs(a * xa + b * y1 + c), abs(a * x1 + b * yb + c)
                if r1 != r2 and _f32(r1) == _f32(r2):
                    seen.add("r1 != r2 in double, equal in float")
        rr = right_ranges(sc)
        for rg in rr:
            if rg is None:
                continue
            s, t = rg
            seen.add("stop == start" if t == s else "stop < start" if t < s else "stop > start")
            if s == 0 and t > s:
                seen.add("start == 0")
            if t == sc.nb - 1:
                seen.add("stop == nb - 1")
        if sc.th == 0:
            seen.add("errorTh == 0")
        certain, possible, _, _ = sc.classes
        if "structure" in sc.props:
            counts = certain.sum(0)
            assert not (possible & ~certain).any(), sc
            for k in (1, 7, 8, 9):
                assert any(counts[j] == k and counts[j - 1] == 0 for j in range(1, sc.mr)), (sc, k)
            assert counts.max() >= 64 and (counts == 0).sum() > 20, sc
            starts = np.cumsum(np.r_[0, counts])
            assert any(starts[j] % GF_CAND_CHUNK and (starts[j] // GF_CAND_CHUNK != starts[j + 1] // GF_CAND_CHUNK) for j in range(sc.mr)), sc
            seen.add("candidate runs")
            rows = [sorted(sc.dist[r, certain[r]].tolist()) for r in range(sc.ml)]
            assert any(len(v) >= 3 and v[0] == v[1] == v[2] for v in rows), sc     # the best distance at several j
            assert any(len(v) == 2 and v[0] == v[1] for v in rows), sc             # the second best equal to the best
            assert any(len(v) >= 2 and v[0] == sc.ratio * v[1] for v in rows), sc  # bd == distRatio * sbd in double
            assert sc.ratio > 1 or any(len(v) >= 2 and (v[0] < sc.ratio * v[1]) != (v[0] < _f32(np.float32(sc.ratio) * np.float32(v[1])))
                                       for v in rows), sc
        seen.add(f"kind {sc.kind}")
        seen.add("geometry" if sc.gl is not None else "upload")
    record_property("edges", sorted(seen))
    want = {"a == 0", "b == 0", "ya == 0", "ya == yamax - 1", "ya in (max - 1, max)", "ya == max", "xb == 0", "xb == xbmax - 1",
            "xb in (max - 1, max)", "xb == max", "r1 != r2 in double, equal in float", "stop == start", "stop < start", "stop > start",
            "start == 0", "stop == nb - 1", "errorTh == 0", "candidate runs", "geometry", "upload"}
    want |= {f"kind {k}" for k in ("u8", "f32", "real", "mixed", "bin")}
    for W, H in ((2, 2), (640, 480), (4000, 3000)):
        want |= {f"corner {c}.{W}x{H}" for c in ("0,0", "W-1,0", "0,H-1", "W-1,H-1")}
    assert want <= seen, sorted(want - seen)


def test_reference_and_oracle_pass_audit():
    """The Python reference under every association and the oracle's compiled restatement pass the audit; the reference under the
    kernel's association equals the oracle bit for bit."""
    O = gfo.GuidedFastOracle("port")
    for sc in scenes():
        for a in ASSOCIATIONS:
            audit(reference(sc, a), sc)
        want = O.guided_fast(sc.dl, sc.pl, sc.dr, sc.pr, sc.F, sc.ep2, sc.W, sc.H, sc.th, sc.ratio, binary=sc.binary)
        audit(want, sc)
        assert _same(reference(sc), want), sc


def test_audit_rejects_wrong_results():
    """Each deliberate fault of the reference fails the audit on at least one scene."""
    caught = {m: [] for m in MUTATIONS}
    for m in MUTATIONS:
        for sc in scenes():
            try:
                audit(reference(sc, mutation=m), sc)
            except AssertionError:
                caught[m].append(sc.name)
    missed = [m for m, c in caught.items() if not c]
    assert not missed, f"faults the audit did not catch: {missed}"


def test_reachable_equals_enumeration():
    """The audit's existence check against every candidate set between the certain and the possible candidates, folded in ascending
    j: on a case where every allowed set keeps a match (certain {0, 1} at 1 and 10, optional {2, 3} at 5 and 6: no match is not
    reachable), and on random small cases with ties, for each outcome (no match, or any j)."""
    import itertools
    d = {0: 1.0, 1: 10.0, 2: 5.0, 3: 6.0}
    assert not _reachable(d, [0, 1], [2, 3], 0.64, -1) and _reachable(d, [0, 1], [2, 3], 0.64, 0)
    rng = np.random.default_rng(3)
    for _ in range(3000):
        n = int(rng.integers(1, 7))
        d = {j: float(v) for j, v in enumerate(rng.integers(1, 12, n))}
        role = rng.integers(0, 3, n)                                   # 0: certain, 1: optional, 2: not a candidate
        cert, opt = np.flatnonzero(role == 0).tolist(), np.flatnonzero(role == 1).tolist()
        ratio = float(rng.choice([0.0, 0.5, 0.64, 1.0, 1.5]))
        outcomes = set()
        for k in range(len(opt) + 1):
            for S in itertools.combinations(opt, k):
                js = sorted(cert + list(S))
                outcomes.add(tge.fold([d[j] for j in js], js, ratio))
        for got in [-1] + list(range(n)):
            assert _reachable(d, cert, opt, ratio, got) == (got in outcomes), (d, cert, opt, ratio, got, outcomes)


def _realistic():
    """test_guided_fast.py's two-view grid (geometry positions) and a list of pairs of its multi-view scene."""
    out = []
    for kind in ("u8", "bin"):
        for geom, W, H, sign in tgf.GRID:
            s = tgf.two_view(kind, geom, 600, W, H, seed=5)
            out.append((f"two_view.{kind}.{geom}.{W}x{H}.{sign}", FastScene("t", kind, sign * s["F"], sign * s["ep2"], W, H, 16.0, 0.64,
                                                                               s["dl"], s["ul"], s["dr"], s["ur"], True)))
    cams, views = tgf.multi_view(12, 1000)
    rng = np.random.default_rng(2)
    pairs = [(a, b) for a in range(12) for b in range(12) if a != b]
    for k in rng.permutation(len(pairs))[:40]:
        a, b = pairs[k]
        F, e = tgf.fundamental(cams[a], cams[b])
        out.append((f"multi_view.{a}.{b}", FastScene("m", "u8", F, e, cams[b].W, cams[b].H, 16.0, 0.64, views[a][0], views[a][2],
                                                     views[b][0], views[b][2], True)))
    return out


def test_association_sensitivity(record_property):
    """The reference under "seq", "halving" and "packet": the left features whose bucket differs and the match lists that differ,
    on the edge scenes and on realistic scenes (recorded as test properties); the association scene shows that the choice
    changes a list."""
    counts = {}
    for group, items in (("edge", [(sc.name, sc) for sc in scenes()]), ("realistic", _realistic())):
        for other in ("halving", "packet"):
            feats = lists = total_feats = total_lists = 0
            for name, sc in items:
                b0, b1 = left_buckets(sc, KERNEL_ASSOCIATION), left_buckets(sc, other)
                feats += int((b0 != b1).sum())
                total_feats += sc.ml
                lists += not _same(reference(sc, KERNEL_ASSOCIATION), reference(sc, other))
                total_lists += 1
            counts[(group, other)] = (feats, lists)
            record_property(f"{group}.{KERNEL_ASSOCIATION}_vs_{other}.left_features_in_another_bucket", f"{feats} of {total_feats}")
            record_property(f"{group}.{KERNEL_ASSOCIATION}_vs_{other}.match_lists_that_differ", f"{lists} of {total_lists}")
    sc = next(s for s in scenes() if s.name == "association")
    assert not _same(reference(sc, "seq"), reference(sc, "halving"))
    assert (left_buckets(sc, "seq") != left_buckets(sc, "halving")).all()


# ---------------------------------------------------------------------------------------------- GPU tests
def _upload(ctx, base, keep):
    """Both views of every scene under ids base + 2 k, base + 2 k + 1; geometry positions where the scene has them."""
    from alicevision_b200 import matching
    ids = []
    for k, sc in enumerate(scenes()):
        ids.append((base + 2 * k, base + 2 * k + 1))
        for vid, d, xy, g in ((base + 2 * k, sc.dl, sc.xl, sc.gl), (base + 2 * k + 1, sc.dr, sc.xr, sc.gr)):
            code = matching.BIN if sc.binary else matching._dtype_code(d, False)
            keep.append((d, xy))
            matching._check(ctx.lib.b200m_upload_view(ctx._h, C.c_uint32(vid), d.ctypes.data_as(C.c_void_p), C.c_int(len(d)),
                                                      C.c_int(d.shape[1]), C.c_int(code), xy.ctypes.data_as(C.c_void_p)),
                            "b200m_upload_view")
            if g is not None:
                ctx.set_view_geometry(vid, g)
    ctx.lib.b200m_wait_uploads(ctx._h)
    return ids


@pytest.mark.gpu
def test_gpu_one_pair_equals_reference():
    """matching.guidedMatchingFundamentalFast on every scene: equal to the reference bit for bit and audited."""
    from alicevision_b200 import Regions, matching
    ctx = matching.Context(0)
    try:
        errs = ctx.exactness_errors()
        for sc in scenes():
            L, R = Regions(sc.dl, sc.xl, binary=sc.binary), Regions(sc.dr, sc.xr, binary=sc.binary)
            got = matching.guidedMatchingFundamentalFast(sc.F, sc.ep2, L, R, sc.W, sc.H, sc.th, sc.ratio, xy_left=sc.gl, xy_right=sc.gr,
                                                         ctx=ctx)
            assert _same(got, reference(sc)), (sc, len(got), len(reference(sc)))
            audit(got, sc)
        assert ctx.exactness_errors() == errs
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_pair_lists_equal_reference(monkeypatch):
    """Context.guided_match_fast_pairs over one list per (errorTh, distRatio, kernel class) holding all of its scenes (image sizes and
    geometry positions mixed): at the default bound of left features per batch, where each list runs as one batch (as many launches
    as a list of its first pair alone), and with a bound of 64, which splits every list of two or more pairs and more than 64 left
    features into several batches (more launches): every result equal to the reference bit for bit and audited."""
    from alicevision_b200 import matching
    sc_all = scenes()
    groups = {}
    for k, sc in enumerate(sc_all):
        groups.setdefault((sc.th, sc.ratio, tge._KCLASS[sc.kind]), []).append(k)
    assert max(sum(sc_all[k].kind == "mixed" for k in ks) for ks in groups.values()) <= 1    # one fp32 expansion per list at most
    split = 0
    for cap in (None, 64):
        if cap:
            monkeypatch.setenv("B200M_GUIDED_FAST_LEFT_CAP", str(cap))      # read when a context is created
        ctx = matching.Context(0)
        keep = []
        try:
            ids = _upload(ctx, 0x1000, keep)
            errs = ctx.exactness_errors()
            for (th, ratio, _), ks in sorted(groups.items()):
                args = lambda ks_: ([ids[k] for k in ks_], [sc_all[k].F for k in ks_], [sc_all[k].ep2 for k in ks_],
                                    [(sc_all[k].W, sc_all[k].H) for k in ks_], th, ratio)
                ctx.guided_match_fast_pairs(*args(ks[:1]))
                one_batch = ctx.last_launches()
                got = ctx.guided_match_fast_pairs(*args(ks))
                launches = ctx.last_launches()
                for k in ks:
                    assert _same(got[ids[k]], reference(sc_all[k])), (sc_all[k], cap)
                    audit(got[ids[k]], sc_all[k])
                if cap is None:
                    assert launches == one_batch, (th, ratio, ks, launches, one_batch)
                elif len(ks) > 1 and sum(sc_all[k].ml for k in ks) > cap:     # (a pair larger than the bound runs alone)
                    assert launches > one_batch, (th, ratio, ks, launches, one_batch)
                    split += 1
            assert ctx.exactness_errors() == errs
        finally:
            ctx.close()
    assert split >= 3, split
