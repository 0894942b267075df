"""Guided matching (K7 `guided_pairs_kernel`, and the position-only `guided_positions_pairs_kernel`) against an exact reference.

The oracles restate the reference's 3 x 3 error arithmetic (FundamentalError.hpp:52-64, HomographyError.hpp:23-31) without Eigen, as the
kernels do, so a convention shared by all of them (F applied to the wrong side, the homography transfer in the wrong direction, `<=`
for `<`) would pass every engine-vs-oracle comparison.  This file decides every (left i, right j) independently:

* an outward-rounded interval, evaluated in numpy along the reference's operation sequence, encloses both the exact error of the double
  positions and the double the reference computes: a pair is a definite pass (hi < errorTh), a definite fail (lo >= errorTh, or a
  division by an exact 0 / a NaN input, which IEEE arithmetic turns into inf or NaN) or ambiguous.  Ambiguous pairs (and a sample of
  the others) are checked against the exact rational error written from the definitions (the squared distance of x_r to the
  epipolar line F x_l; the squared transfer error of x_r against H x_l);
* the audits then state what a correct result must be, allowing every choice of the ambiguous pairs: K7's distanceRatio fold
  (guidedMatching.hpp:77-118, the ratio product in double) over the gate in ascending j, and the position-only minimum (the first j
  of an exact tie, the phantom (0, 0) of an empty row at errorTh = +inf; guidedMatching.hpp:37-70).

The scenes sit where these kernels can go wrong: errors exactly on errorTh and one ulp either side, errors that double rounding
decides, degenerate models and thresholds, ratio products exactly on bd or split by float rounding, survivor counts on the edges of
K7's 32-wide steps, 8-deep drains and 1024-position tiles, and every descriptor class for both models.  The CPU part checks that the
oracles pass the audits and that the audits reject deliberately wrong results; the GPU part (run with -m gpu on an H100) audits the
three engine calls and compares them with the oracles bit for bit."""
import ctypes as C
import functools
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle
from oracle import guided_fast as gfo
from oracle import guided_positions as gpo

DBL_MAX = float(np.finfo(np.float64).max)
GM_STEP, GM_TILE = 32, 1024                 # guided.cuh: a warp tests 32 right positions per step; GM_TILE positions per shared tile
F_RECT = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)      # rectified pair: err = (y_l - y_r)^2
H_POW2 = np.array([[4, 0, 128], [0, 2, -64], [0, 0, 2]], np.float64)    # x_r = (2 x + 64, y - 32): every operation exact
R_DEFAULT = 0.64                            # distRatio as guidedMatching receives it (already squared)


# ---------------------------------------------------------------------------------------------- outward-rounded intervals
_TINY, _HUGE = 2.0 ** -450, 2.0 ** 450      # where the error-free transformations below are exact (no overflow, no underflow)


def _safe(*xs):
    ok = True
    for x in xs:
        a = np.abs(x)
        ok = ok & ((a == 0) | ((a >= _TINY) & (a <= _HUGE)))
    return ok


def _sum_err(a, b, s):
    """TwoSum: (a + b) - s exactly."""
    bb = s - a
    return (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a
    h = c - (c - a)
    return h, a - h


def _prod_err(a, b, p):
    """Dekker's TwoProduct: a * b - p exactly, for operands and product inside _safe."""
    ah, al = _split(a)
    bh, bl = _split(b)
    return ((ah * bh - p) + ah * bl + al * bh) + al * bl


class Iv:
    """[lo, hi] holds the exact value of the expression on the double inputs and the double the reference computes from them.
    ex: lo == hi, so both are lo; und: the reference's double is certainly +-inf or NaN (a NaN input, or a division by an exact 0);
    bad: no enclosure (an end point became NaN, or a divisor interval holds 0): the value is unknown."""

    def __init__(self, lo, hi, und, bad):
        self.lo, self.hi, self.und, self.bad = lo, hi, und, bad
        self.ex = (lo == hi) & ~und & ~bad

    @staticmethod
    def point(x):
        x = np.asarray(x, np.float64)
        return Iv(x, x, np.isnan(x), np.zeros(x.shape, bool))


def _round(a, b, corners, und=None, nonneg=False):
    """The result of one operation from its corners [(round-to-nearest value c, sign of exact - c, NaN when unknown)]: the operation
    is monotone in each operand on the box, so its exact range and the reference's double (rounding is monotone) lie between the
    smallest and the largest corner, each widened by one ulp unless the error-free transformation shows that no corner of that value
    was rounded across it (the exact corner is within half an ulp of c)."""
    und = (a.und | b.und) if und is None else und
    vals = [c for c, _ in corners]
    with np.errstate(invalid="ignore"):
        lo, hi = np.minimum.reduce(vals), np.maximum.reduce(vals)
        lo_ok = np.logical_and.reduce([(c > lo) | (e >= 0) for c, e in corners])
        hi_ok = np.logical_and.reduce([(c < hi) | (e <= 0) for c, e in corners])
        nan = np.isnan(lo) | np.isnan(hi)
        lo2 = np.where(lo_ok, lo, np.nextafter(lo, -np.inf))
        hi2 = np.where(hi_ok, hi, np.nextafter(hi, np.inf))
        if nonneg:                          # squares, their sums and quotients by a positive: neither value can be negative
            lo2 = np.maximum(lo2, 0.0)
    return Iv(lo2, hi2, und, (a.bad | b.bad | nan) & ~und)


def _known(sign, ok):
    return np.where(ok, sign, np.nan)


def _add(x, y):
    s = x + y
    return s, _known(np.sign(_sum_err(x, y, s)), np.isfinite(s) & _safe(x, y, s))


def _mul(x, y):
    p = x * y
    return p, _known(np.sign(_prod_err(x, y, p)), np.isfinite(p) & _safe(x, y, p))


def _div(x, y):
    """exact - q = (x - q y) / y; the residual x - q y of a correctly rounded quotient is a double, (x - fl(q y)) - err(q y) exactly."""
    q = x / y
    pe = q * y
    r = (x - pe) - _prod_err(q, y, pe)
    return q, _known(np.sign(r) * np.sign(y), np.isfinite(q) & _safe(x, y, q, pe))


def iv_add(a, b, nonneg=False):
    with np.errstate(all="ignore"):
        return _round(a, b, [_add(a.lo, b.lo), _add(a.hi, b.hi)], nonneg=nonneg)


def iv_sub(a, b):
    with np.errstate(all="ignore"):
        return _round(a, b, [_add(a.lo, -b.hi), _add(a.hi, -b.lo)])


def iv_mul(a, b):
    with np.errstate(all="ignore"):
        return _round(a, b, [_mul(a.lo, b.lo), _mul(a.lo, b.hi), _mul(a.hi, b.lo), _mul(a.hi, b.hi)])


def iv_sq(a):
    with np.errstate(all="ignore"):
        l2, h2 = _mul(a.lo, a.lo), _mul(a.hi, a.hi)
        straddle = (a.lo < 0) & (a.hi > 0)
        zero = (np.where(straddle, 0.0, l2[0]), np.where(straddle, 0.0, l2[1]))   # an interval holding 0 squares down to 0
        return _round(a, a, [l2, h2, zero], nonneg=True)


def iv_div(a, b, nonneg=False):
    zero = (b.lo <= 0) & (b.hi >= 0)
    with np.errstate(all="ignore"):
        corners = [_div(a.lo, b.lo), _div(a.lo, b.hi), _div(a.hi, b.lo), _div(a.hi, b.hi)]
    und = a.und | b.und | (zero & b.ex)     # an exact 0 divisor: the reference's double is +-inf or NaN
    r = _round(a, b, corners, und=und, nonneg=nonneg)
    r.bad = r.bad | (zero & ~und)
    r.ex = r.ex & ~r.bad
    return r


def enclose(model, M, pl, pr):
    """Intervals of the error of every (left i, right j) for double positions pl [m_l, 2], pr [m_r, 2], in the reference's operation
    order: F_x row r = (M(r,0) x + M(r,1) y) + M(r,2); F: dot = (F_x0 y0 + F_x1 y1) + F_x2, err = dot^2 / (F_x0^2 + F_x1^2);
    H: d = y - F_x.head<2>() / F_x2, err = d0^2 + d1^2."""
    P = Iv.point
    x, y = P(pl[:, :1]), P(pl[:, 1:2])
    f = [iv_add(iv_add(iv_mul(P(M[r, 0]), x), iv_mul(P(M[r, 1]), y)), P(M[r, 2])) for r in range(3)]
    y0, y1 = P(pr[None, :, 0]), P(pr[None, :, 1])
    if model == 0:
        nrm = iv_add(iv_sq(f[0]), iv_sq(f[1]), nonneg=True)
        dot = iv_add(iv_add(iv_mul(f[0], y0), iv_mul(f[1], y1)), f[2])
        return iv_div(iv_sq(dot), nrm, nonneg=True)
    d0, d1 = iv_sub(y0, iv_div(f[0], f[2])), iv_sub(y1, iv_div(f[1], f[2]))
    return iv_add(iv_sq(d0), iv_sq(d1), nonneg=True)


def decide(iv, th):
    """+1: err < th for the exact value and the reference's double; -1: neither (NaN never passes); 0: undecided."""
    shape = np.broadcast(iv.lo, iv.hi).shape
    if math.isnan(th):
        return np.full(shape, -1, np.int8)
    ok = ~iv.und & ~iv.bad
    return np.where(ok & (iv.hi < th), 1, np.where(iv.und | (ok & (iv.lo >= th)), -1, 0)).astype(np.int8)


def exact_error(model, M, x, y):
    """The error of right point y for left point x from its definition, in rationals (None where it is undefined): the squared
    distance of y to the line l = M x, (l . y)^2 / (l0^2 + l1^2), or the squared distance of y to the point M x."""
    if not (np.all(np.isfinite(M)) and np.all(np.isfinite(x)) and np.all(np.isfinite(y))):
        return None
    Mq = [[Fraction(float(v)) for v in row] for row in M]
    xh = (Fraction(float(x[0])), Fraction(float(x[1])), Fraction(1))
    yh = (Fraction(float(y[0])), Fraction(float(y[1])), Fraction(1))
    l = [sum(Mq[r][c] * xh[c] for c in range(3)) for r in range(3)]
    if model == 0:
        n = l[0] ** 2 + l[1] ** 2
        return None if n == 0 else sum(l[c] * yh[c] for c in range(3)) ** 2 / n
    if l[2] == 0:
        return None
    return (yh[0] - l[0] / l[2]) ** 2 + (yh[1] - l[1] / l[2]) ** 2


# ---------------------------------------------------------------------------------------------- descriptor distances
GAMMA_36 = 36 * 2.0 ** -24 / (1 - 36 * 2.0 ** -24)      # a sum of 32 squared differences per lane and three lane sums, in float


def distances(sc, ii, jj):
    """Regions::SquaredDescriptorDistance of left ii / right jj (double): exact integers for uchar and integer-valued fp32 (stored as
    uchar), popcount^2 for binary, and for real fp32 (and the mixed pair's fp32 expansion) the reference's four SSE lanes,
    s_k += (a - b)^2 over t ascending, ((s0 + s1) + s2) + s3, every operation rounded to float."""
    ii, jj = np.asarray(ii, np.int64), np.asarray(jj, np.int64)
    a, b = sc.dl[ii], sc.dr[jj]
    if sc.kind == "bin":
        h = np.unpackbits(a ^ b, axis=1).sum(1).astype(np.float64)
        return h * h
    if sc.kind in ("u8", "f32"):
        d = a.astype(np.int64) - b.astype(np.int64)
        return (d * d).sum(1).astype(np.float64)
    a, b = a.reshape(-1, 32, 4), b.reshape(-1, 32, 4)
    s = np.zeros((len(ii), 4), np.float32)
    for t in range(32):
        d = a[:, t] - b[:, t]
        s = s + d * d
    v = (((s[:, 0] + s[:, 1]) + s[:, 2]) + s[:, 3]).astype(np.float64)
    d64 = a.astype(np.float64) - b.astype(np.float64)       # exact: the operands are within a factor 2^29 of each other
    exact = (d64 * d64).sum((1, 2))
    assert np.all(np.abs(v - exact) <= GAMMA_36 * exact), "the four-lane float sum left its error bound"
    return v


# ---------------------------------------------------------------------------------------------- scenes
class Scene:
    """One (left view, right view, model, errorTh, distRatio).  Positions: geometry positions (double) when gl / gr are set, else the
    float upload positions widened.  The classification of every pair is computed once."""

    def __init__(self, name, model, M, th, ratio, kind, dl, xl, dr, xr, geometry=False, props=()):
        self.name, self.model, self.M, self.th, self.ratio, self.kind = name, model, np.asarray(M, np.float64), float(th), ratio, kind
        self.dl, self.dr = np.ascontiguousarray(dl), np.ascontiguousarray(dr)
        xl, xr = np.asarray(xl, np.float64).reshape(-1, 2), np.asarray(xr, np.float64).reshape(-1, 2)
        if geometry:
            self.gl, self.gr = np.ascontiguousarray(xl), np.ascontiguousarray(xr)
            self.pl, self.pr = self.gl, self.gr
        else:
            self.gl = self.gr = None
        self.xl, self.xr = np.ascontiguousarray(xl, np.float32), np.ascontiguousarray(xr, np.float32)
        if not geometry:
            self.pl, self.pr = self.xl.astype(np.float64), self.xr.astype(np.float64)
        self.props = props
        self.ml, self.mr = len(self.dl), len(self.dr)
        assert self.ml <= 2048 and self.mr <= 2055 and len(self.xl) == self.ml and len(self.xr) == self.mr
        self.binary = kind == "bin"

    @functools.cached_property
    def iv(self):
        return enclose(self.model, self.M, self.pl, self.pr)

    @functools.cached_property
    def cls(self):
        """K7's gate: err < errorTh."""
        return decide(self.iv, self.th)

    @functools.cached_property
    def pos_th(self):
        """The position-only scan needs err < errorTh and err < min, min starting at DBL_MAX."""
        return self.th if not self.th > DBL_MAX else DBL_MAX

    @functools.cached_property
    def cls_pos(self):
        return decide(self.iv, self.pos_th)

    def lohi(self):
        return np.broadcast_to(self.iv.lo, (self.ml, self.mr)), np.broadcast_to(self.iv.hi, (self.ml, self.mr))

    def __repr__(self):
        return self.name


def _greedy_squares(d):
    """Components <= 255 whose squares sum to d."""
    out = []
    while d:
        c = min(255, math.isqrt(d))
        out.append(c)
        d -= c * c
    assert len(out) <= 128
    return out


def at_distances(dists, dtype=np.uint8):
    """Right descriptors whose squared distance to the all-zero left descriptor is exactly dists[k]."""
    out = np.zeros((len(dists), 128), np.uint8)
    for k, d in enumerate(dists):
        c = _greedy_squares(int(d))
        out[k, :len(c)] = c
    return out.astype(dtype)


def _pred(x, f32):
    return float(np.nextafter(np.float32(x), np.float32(0))) if f32 else float(np.nextafter(x, 0.0))


def _succ(x, f32):
    return float(np.nextafter(np.float32(x), np.float32(np.inf))) if f32 else float(np.nextafter(x, np.inf))


def threshold_scene(model, th, geometry):
    """Errors exactly on errorTh (rejected: the gate is err < errorTh), one ulp of the position below and above.  F: F_RECT, left
    rows at y = 0, +-s, 3 s with s = sqrt(errorTh), right points s, one ulp below and above away; H: H_POW2, right points at the exact
    transfer plus the same offsets along x and y.  One left feature of each has no right point within reach but one on the threshold.  The right descriptors put the best distances on the points exactly on the
    threshold, so admitting one changes the result."""
    s = math.sqrt(th)
    f32 = not geometry
    offs = [0.0, s, -s, _pred(s, f32), -_pred(s, f32), _succ(s, f32), -_succ(s, f32), 2 * s, -3 * s]
    dist_of = {0: 400, 1: 1, 2: 2, 3: 100, 4: 200, 5: 3, 6: 4, 7: 9, 8: 16}
    if model == 0:
        yl = [0.0, s, -s, 0.0, 3 * s]                                       # 3 s: the one point within reach sits on the threshold
        xl = np.array([[10.0 * k, y] for k, y in enumerate(yl)])
        xr = np.array([[5.0 * k, o] for k, o in enumerate(offs)])
        dists = [dist_of[k] for k in range(len(offs))]
        M = F_RECT
    else:
        xl = np.array([[-32.0, 32.0], [-31.0, 33.0], [-30.0, 34.0]])          # transfers (0, 0), (2, 1), (4, 2)
        proj = np.c_[2 * xl[:, 0] + 64, xl[:, 1] - 32]
        xr, dists = [], []
        for p in proj:
            for k, o in enumerate(offs):
                for ax in (0, 1):
                    xr.append(p + (o if ax == 0 else 0.0, o if ax == 1 else 0.0))
                    dists.append(dist_of[k] + 20 * ax)
        xl = np.r_[xl, [[-20.0, 50.0]]]                                    # transfer (24, 18): one point, on the threshold
        xr.append((24.0 + s, 18.0))
        dists.append(5)
        xr = np.array(xr)
        M = H_POW2
    if not geometry:
        xl, xr = xl.astype(np.float32), xr.astype(np.float32)
    dl = np.zeros((len(xl), 128), np.uint8)
    return Scene(f"threshold.{'FH'[model]}.{th}.{'geometry' if geometry else 'upload'}", model, M, th, 0.64, "u8", dl, xl,
                 at_distances(dists), xr, geometry, props=("threshold",))


def rounding_scene(model, seed):
    """Geometry positions around 1e6 .. 1e7 with right points 2 px from the epipolar line (F) or from the transfer (H) up to a few
    1e-9 px: double rounding decides some of them (ambiguous pairs).  errorTh = 4.  The near-threshold points carry the best descriptor
    distances."""
    rng = np.random.default_rng(seed)
    if model == 0:
        A = np.array([[1.0 / 3, 0.2, 1.7e5], [0.1, 0.7, -3.1e5], [0, 0, 1]])
        M = np.linalg.inv(A).T @ F_RECT                   # the epipolar lines of A-mapped rows
    else:
        M = np.array([[0.7, 0.11, 2.3e5], [-0.13, 0.9, 1.1e5], [1e-9, -2e-9, 1.0]])
    ml, per = 24, 6
    xl = np.c_[rng.uniform(1e6, 1e7, ml), 3e6 + 1e5 * np.arange(ml)]
    xr, dists = [], []
    for i in range(ml):
        if model == 0:
            base = A @ np.array([rng.uniform(1e6, 1e7, per), np.full(per, xl[i, 1]), np.ones(per)])
            line = M @ np.array([xl[i, 0], xl[i, 1], 1.0])
            n = line[:2] / np.hypot(line[0], line[1])
            p = base[:2].T
        else:
            h = M @ np.array([xl[i, 0], xl[i, 1], 1.0])
            p = np.tile(h[:2] / h[2], (per, 1))
            ang = rng.uniform(0, 2 * np.pi, per)
            n = np.c_[np.cos(ang), np.sin(ang)]
        t = 2.0 + np.r_[rng.uniform(-4e-9, 4e-9, 3), -0.5, 0.5, 1.5]    # three near the threshold, two inside, one outside
        xr.extend(p + t[:, None] * n)
        dists.extend([3 + i % 5, 5 + i % 3, 7, 60, 90, 1])
    xr = np.array(xr)
    dl = np.zeros((ml, 128), np.uint8)
    return Scene(f"rounding.{'FH'[model]}", model, M, 4.0, 0.64, "u8", dl, xl, at_distances(dists), xr, True, props=("rounding",))


def random_descriptors(kind, owner, rng, ml):
    """Left descriptors and right ones: a noisy copy of the left descriptor of owner[j] (or a fresh one where owner[j] < 0)."""
    if kind == "bin":
        dl = rng.integers(0, 256, (ml, 64), dtype=np.uint8)
        flips = np.packbits(rng.random((len(owner), 512)) < 0.05, axis=1, bitorder="little")
        dr = np.where((owner >= 0)[:, None], dl[np.maximum(owner, 0)] ^ flips, rng.integers(0, 256, (len(owner), 64), dtype=np.uint8))
        return dl, dr.astype(np.uint8)
    dl = rng.integers(0, 256, (ml, 128)).astype(np.uint8)
    noisy = np.clip(dl[np.maximum(owner, 0)].astype(np.int32) + rng.integers(-12, 13, (len(owner), 128)), 0, 255)
    dr = np.where((owner >= 0)[:, None], noisy, rng.integers(0, 256, (len(owner), 128))).astype(np.uint8)
    if kind == "u8":
        return dl, dr
    dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    if kind == "f32":
        return dl, dr
    dr = dr + rng.uniform(-0.5, 0.5, dr.shape).astype(np.float32)     # real fp32 right view
    if kind == "real":
        dl = dl + rng.uniform(-0.5, 0.5, dl.shape).astype(np.float32)
    return dl, dr                                                         # "mixed": integer-valued left, real right


def class_scene(kind, model, th=4.0, seed=0, M=None, geometry=False, ml=37, mr=300, tag=None):
    """Random scene of one descriptor class: left rows spaced 8 px apart, each right point within 2.5 px of the epipolar line (F,
    through an affine map of the right image: a general F) or of the transfer (H_POW2) of a random left point; one right descriptor
    per left feature is a noisy copy of its descriptor, the others are fresh."""
    rng = np.random.default_rng(seed + 101 * model + 7 * ("u8", "f32", "real", "mixed", "bin").index(kind))
    xl = np.c_[rng.uniform(0, 512, ml), 8.0 * np.arange(ml) + 4]
    owner = rng.integers(0, ml, mr)
    if model == 0:
        A = np.array([[1.0, 0.25, 3.0], [0.125, 1.0, -2.0], [0, 0, 1]])
        rect = np.c_[rng.uniform(0, 512, mr), xl[owner, 1] + rng.uniform(-2.5, 2.5, mr), np.ones(mr)]
        xr = (rect @ A.T)[:, :2]
        Mm = np.linalg.inv(A).T @ F_RECT if M is None else M
    else:
        xr = np.c_[2 * xl[owner, 0] + 64, xl[owner, 1] - 32] + rng.uniform(-1.8, 1.8, (mr, 2))
        Mm = H_POW2 if M is None else M
    desc_owner = np.full(mr, -1)
    for i in range(ml):                                                   # one noisy copy per left feature, in its gate
        js = np.flatnonzero(owner == i)
        if len(js):
            desc_owner[rng.choice(js)] = i
    dl, dr = random_descriptors(kind, desc_owner, rng, ml)
    name = f"class.{kind}.{'FH'[model]}" + (f".{tag}" if tag else "")
    return Scene(name, model, Mm, th, R_DEFAULT, kind, dl, xl, dr, xr, geometry, props=("class",))


def epipole_scene():
    """F = [t]_x, t = (64, 32, 1): the left point (64, 32) is the epipole, F x = 0 exactly, err = 0 / 0 (NaN) for every right point."""
    F = np.array([[0, -1, 32], [1, 0, -64], [-32, 64, 0]], np.float64)
    xl = np.array([[64, 32], [0, 0], [128, 96], [65, 32], [64, 32]], np.float64)
    xr = [[2.0 * k, 1.0 * k] for k in range(1, 12)]                 # on the line of (0, 0): 32 X - 64 Y = 0
    xr += [[64 + 2.0 * k, 32 + 1.0 * k + 0.25] for k in range(6)]
    xr += [[128 - k, 96 + 0.5 * k] for k in range(6)]
    xr = np.array(xr)
    return Scene("degenerate.epipole", 0, F, 4.0, 1.0, "u8", np.zeros((5, 128), np.uint8), xl,
                 at_distances(list(range(1, len(xr) + 1))), xr, props=("epipole",))


def w_scene(geometry):
    """H with w = x / 64 - 1: w = 0 at x = 64 (the transfer is inf / NaN), w < 0 at x = 32 (x_r = -(2x, 2y) / 0.5)."""
    H = np.array([[2, 0, 0], [0, 2, 0], [0.015625, 0, -1]], np.float64)
    xl = np.array([[64, 8], [32, 8], [128, 16], [64, 16], [16, 4]], np.float64)
    h = np.c_[xl, np.ones(5)] @ H.T
    proj = h[:, :2] / np.where(h[:, 2:] == 0, 1, h[:, 2:])
    xr = np.concatenate([proj + o for o in ([0, 0], [0.5, 0.5], [1.5, 0], [-1, -1], [3, 0])])
    return Scene(f"degenerate.w.{'geometry' if geometry else 'upload'}", 1, H, 4.0, 1.0, "u8", np.zeros((5, 128), np.uint8), xl,
                 at_distances(list(range(1, len(xr) + 1))), xr, geometry, props=("w",))


def ratio_triples(r):
    """(bd, sbd) integer distances for ratio r (already squared): "exact" bd == fl(r * sbd) in double; "float": the float and the
    double product of r and sbd fall on different sides of bd; each with its integer neighbours bd - 1, bd + 1."""
    sbd = np.arange(1, 1 << 22, dtype=np.float64)
    pd = r * sbd
    pf = (np.float32(r) * sbd.astype(np.float32)).astype(np.float64)
    hits = {}
    ex = np.flatnonzero((pd == np.floor(pd)) & (pd <= sbd))
    hits["exact"] = [(int(pd[k]), int(sbd[k])) for k in ex[:2]] + ([(0, 0)] if r == 0 or r > 1 else [])
    c = np.ceil(np.minimum(pf, pd))
    fl = np.flatnonzero((c < np.maximum(pf, pd)) & (c <= sbd))
    hits["float"] = [(int(c[k]), int(sbd[k])) for k in fl[:2]]
    out = []
    for bd, s in hits["exact"] + hits["float"]:
        for b in (bd - 1, bd, bd + 1):
            if 0 <= b <= s and (b, s) not in out:
                out.append((b, s))
    return out, hits


def ratio_scene(r):
    """Rows of F_RECT (y = 16 i): each left row sees exactly the right points on its row.  A row per (bd, sbd) of ratio_triples
    (the sbd point first, then the bd point, then a third point farther than sbd), a row of two equal distances (duplicate
    right descriptors: bd == sbd, the first j wins), and a row with a single candidate (sbd = DBL_MAX: never kept)."""
    rows, hits = ratio_triples(r)
    cand = [[s, b, s + 7] for b, s in rows] + [[50, 50, 80], [0]]
    xl = np.array([[0.0, 16.0 * i] for i in range(len(cand))])
    xr, dists = [], []
    for i, c in enumerate(cand):
        for k, d in enumerate(c):
            xr.append([3.0 * k, 16.0 * i])
            dists.append(d)
    sc = Scene(f"ratio.{r}", 0, F_RECT, 4.0, r, "u8", np.zeros((len(xl), 128), np.uint8), xl, at_distances(dists), np.array(xr),
               props=("ratio",))
    sc.hits = hits
    return sc


def structure_scene(mr, ml=13, kind="u8"):
    """F_RECT rows y = 16 i; right point j lies on exactly one left row (err = 0, every other row sees err >= 256).  With 2055 right
    points: row 0 has 7 survivors in step 0, row 1 8, row 2 9 and row 3 all 32 of their steps; row 4 has 7 waiting survivors followed by a
    full step (39 queued); row 5 straddles the tile boundary 1024, row 6 the boundary 2048; row 7 has one survivor every 97 positions
    (steps with none in between); the rest of the positions go to rows 8 .. 12.  Smaller right views keep the first mr positions.  The
    best descriptor of a row sits on a step boundary (j % 32 == 31) or on a tile boundary (j % 1024 == 0)."""
    owner = np.full(2055, -1)
    for row, (a, b) in enumerate([(0, 7), (32, 40), (64, 73), (96, 128)]):
        owner[a:b] = row
    owner[160:167] = 4
    owner[192:224] = 4
    owner[1016:1032] = 5
    owner[2040:2055] = 6
    free = np.flatnonzero(owner < 0)
    owner[free[free % 97 == 0]] = 7
    free = np.flatnonzero(owner < 0)
    owner[free] = 8 + free % (ml - 8)
    owner = owner[:mr]
    j = np.arange(mr)
    dists = 5000 + (j * 7919) % 90000
    dists = np.where(j % GM_STEP == GM_STEP - 1, 10 + j % 50, dists)
    dists = np.where((j % GM_TILE == 0) & (j > 0), 5, dists)
    xl = np.c_[np.arange(ml) * 3.0, 16.0 * np.arange(ml)]
    xr = np.c_[j * 0.5, 16.0 * owner]
    dr = at_distances(dists)
    dl = np.zeros((ml, 128), np.uint8)
    if kind == "f32":
        dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    return Scene(f"structure.{mr}.{kind}", 0, F_RECT, 4.0, R_DEFAULT, kind, dl, xl, dr, xr, props=("structure",))


def allpass_scene():
    """errorTh = +inf: every right point passes the gate of every left feature (2055 candidates per row)."""
    rng = np.random.default_rng(5)
    ml, mr = 9, 2055
    dl = rng.integers(0, 256, (ml, 128)).astype(np.uint8)
    dr = rng.integers(0, 256, (mr, 128)).astype(np.uint8)
    dr[::300] = np.clip(dl[:7].astype(int) + 3, 0, 255)                 # one near copy for each of the first 7 left features
    return Scene("structure.allpass", 0, F_RECT, np.inf, R_DEFAULT, "u8", dl, rng.uniform(-1e3, 1e3, (ml, 2)), dr,
                 rng.uniform(-1e3, 1e3, (mr, 2)), props=("allpass",))


@functools.lru_cache(maxsize=None)
def scenes():
    out = []
    for model in (0, 1):
        for th in (4.0, 2.25, 2.0 ** -20):
            for geometry in (False, True):
                out.append(threshold_scene(model, th, geometry))
        out.append(rounding_scene(model, 3 + model))
        for kind in ("u8", "f32", "real", "mixed", "bin"):
            out.append(class_scene(kind, model, geometry=(kind == "real")))
        for th in (0.0, -1.0, math.nan, math.inf, 1e300):
            out.append(class_scene("u8", model, th=th, seed=9, ml=21, mr=120, tag=f"th{th}"))
        for name, M in (("zero", np.zeros((3, 3))), ("nan", np.full((3, 3), np.nan))):
            for th in (4.0, math.inf):
                out.append(class_scene("u8", model, th=th, seed=11, M=M, ml=10, mr=40, tag=f"{name}.{th}"))
    out.append(class_scene("u8", 0, seed=13, ml=301, mr=1500, tag="large"))
    out.append(epipole_scene())
    out += [w_scene(False), w_scene(True)]
    out += [ratio_scene(r) for r in (0.0, 0.36, 0.64, 1.0, 1.5)]
    out += [structure_scene(mr) for mr in (1, 2, 31, 32, 33, 1023, 1024, 1025, 2055)]
    out.append(structure_scene(1025, kind="f32"))
    out.append(allpass_scene())
    return tuple(out)


# ---------------------------------------------------------------------------------------------- audits
def _rows(result):
    i, j = np.asarray(result["i"], np.int64), np.asarray(result["j"], np.int64)
    return i, j


def fold(ds, js, ratio, f32_ratio=False, last_on_ties=False):
    """distanceRatio (guidedMatching.hpp:77-118) over candidates in the given order: the kept j or -1."""
    bd = sbd = DBL_MAX
    idx = -1
    for d, j in zip(ds, js):
        if d < bd or (last_on_ties and d == bd):
            idx, sbd, bd = j, bd, d
        elif d < sbd:
            sbd = d
    if sbd == DBL_MAX:
        return -1
    prod = float(np.float32(ratio) * np.float32(sbd)) if f32_ratio else ratio * sbd
    return idx if bd < prod else -1


def k7_expected_definite(sc, D):
    """The expected j (or -1) of every row from its definite passes alone, vectorised: the smallest distance, the first j on ties;
    sbd = the second value of the multiset; kept iff two candidates and bd < distRatio * sbd in double."""
    ii, jj = np.nonzero(D)
    want = np.full(sc.ml, -1, np.int64)
    if len(ii) == 0:
        return want
    d = distances(sc, ii, jj)
    o = np.lexsort((jj, d, ii))
    ii, jj, d = ii[o], jj[o], d[o]
    first = np.flatnonzero(np.r_[True, ii[1:] != ii[:-1]])
    count = np.bincount(ii, minlength=sc.ml)
    rows = ii[first]
    two = count[rows] >= 2
    f2 = first[two]
    keep = d[f2] < sc.ratio * d[f2 + 1]
    want[rows[two][keep]] = jj[f2][keep]
    return want


def audit_guided(result, sc):
    """K7: the engine's (i, j) - or no match - of every left i is a distanceRatio outcome of its definite passes D and some subset of its
    ambiguous pairs A (|A| <= 4), in ascending j; exactly the outcome of D when A is empty.  One match per i, ascending i."""
    i, j = _rows(result)
    assert np.all(np.diff(i) > 0), f"{sc}: not one match per left feature in ascending i"
    assert len(i) == 0 or (i[-1] < sc.ml and np.all(j < sc.mr)), f"{sc}: index out of range"
    got = np.full(sc.ml, -1, np.int64)
    got[i] = j
    D, A = sc.cls == 1, sc.cls == 0
    want = k7_expected_definite(sc, D)
    amb_rows = np.flatnonzero(A.any(1))
    plain = np.ones(sc.ml, bool)
    plain[amb_rows] = False
    bad = np.flatnonzero(plain & (got != want))
    assert len(bad) == 0, f"{sc}: left {bad[:5].tolist()} matched {got[bad[:5]].tolist()}, expected {want[bad[:5]].tolist()}"
    for r in amb_rows:
        a = np.flatnonzero(A[r])
        assert len(a) <= 4, f"{sc}: row {r} has {len(a)} undecided pairs"
        d_js = np.flatnonzero(D[r])
        outcomes = set()
        for k in range(len(a) + 1):
            for S in itertools.combinations(a.tolist(), k):
                js = np.sort(np.r_[d_js, np.array(S, np.int64)]).astype(np.int64)
                outcomes.add(fold(distances(sc, np.full(len(js), r), js), js.tolist(), sc.ratio))
        assert got[r] in outcomes, f"{sc}: left {r} matched {got[r]}, possible {sorted(outcomes)}"


def audit_positions(result, sc):
    """Position-only: the engine's j of every left i is a definite or ambiguous pass whose interval reaches down to the smallest
    upper end over the definite passes, no definite pass before it is certainly <= it and none after it certainly < it (the first j of
    an exact tie); a row with a definite pass has a match; and (0, 0) stands for every unmatched row when errorTh = +inf.  Sorted
    by (i, j), no duplicates (IndMatch::getDeduplicated)."""
    i, j = _rows(result)
    pairs = list(zip(i.tolist(), j.tolist()))
    assert pairs == sorted(set(pairs)), f"{sc}: not sorted and de-duplicated"
    lo, hi = sc.lohi()
    c = sc.cls_pos
    inf = sc.th == math.inf

    def check(plist, phantom_removed):
        rows = {}
        for a, b in plist:
            assert a not in rows, f"{sc}: two matches for left {a}"
            assert 0 <= a < sc.ml and 0 <= b < sc.mr, f"{sc}: index out of range"
            rows[a] = b
        unmatched = any(r not in rows for r in range(sc.ml))
        if phantom_removed:
            assert inf and unmatched, f"{sc}: (0, 0) without an unmatched row at errorTh = +inf"
        elif inf and unmatched:
            assert (0, 0) in plist, f"{sc}: no (0, 0) for the unmatched rows at errorTh = +inf"
        for r in range(sc.ml):
            Dr = np.flatnonzero(c[r] == 1)
            if r not in rows:
                assert len(Dr) == 0, f"{sc}: left {r} unmatched with definite passes {Dr[:5].tolist()}"
                continue
            jj = rows[r]
            assert c[r, jj] >= 0, f"{sc}: left {r} matched {jj}, which fails the gate"
            if len(Dr):
                assert lo[r, jj] <= hi[r, Dr].min(), f"{sc}: left {r} matched {jj}, not the minimum"
                before, after = Dr[Dr < jj], Dr[Dr > jj]
                assert not np.any(hi[r, before] <= lo[r, jj]), f"{sc}: left {r} matched {jj}, an earlier j is as small"
                assert not np.any(hi[r, after] < lo[r, jj]), f"{sc}: left {r} matched {jj}, a later j is smaller"

    tries = [(pairs, False)]
    if (0, 0) in pairs:
        tries.append(([p for p in pairs if p != (0, 0)], True))
    errors = []
    for plist, removed in tries:
        try:
            check(plist, removed)
            return
        except AssertionError as e:
            errors.append(str(e))
    raise AssertionError(" / ".join(errors))


# ---------------------------------------------------------------------------------------------- oracles and a faulty model
def oracle_guided(sc):
    if sc.gl is None:
        return oracle.best().guided_match(sc.dl, sc.xl, sc.dr, sc.xr, sc.M, sc.th, sc.ratio, binary=sc.binary, model=sc.model)
    return gfo.best().guided_match(sc.dl, sc.gl, sc.dr, sc.gr, sc.M, sc.th, sc.ratio, binary=sc.binary, model=sc.model)


def oracle_positions(sc):
    return gpo.GuidedPositionsOracle().guided_match_positions(sc.pl, sc.pr, sc.M, sc.th, sc.model)


MUTATIONS = ("F transposed", "H inverted", "<= at the threshold", "float ratio product", "last j on ties",
             "survivor dropped at a step boundary", "survivor dropped at a tile boundary")


def _double_error(model, M, pl, pr):
    with np.errstate(all="ignore"):
        x, y = pl[:, :1], pl[:, 1:]
        f = [(M[r, 0] * x + M[r, 1] * y) + M[r, 2] for r in range(3)]
        if model == 0:
            dot = (f[0] * pr[None, :, 0] + f[1] * pr[None, :, 1]) + f[2]
            return (dot * dot) / (f[0] * f[0] + f[1] * f[1])
        d0, d1 = pr[None, :, 0] - f[0] / f[2], pr[None, :, 1] - f[1] / f[2]
        return d0 * d0 + d1 * d1


def simulate(sc, mutation=None):
    """Both guided matchings in numpy doubles with one deliberate fault (or none): (K7 matches, position-only matches)."""
    M = sc.M
    if mutation == "F transposed":
        M = M.T
    elif mutation == "H inverted":
        M = np.linalg.inv(M)
    err = _double_error(sc.model, M, sc.pl, sc.pr)
    le = mutation == "<= at the threshold"
    with np.errstate(invalid="ignore"):
        gate = err <= sc.th if le else err < sc.th
        gate_p = (err <= sc.pos_th if le else err < sc.pos_th) & (err < DBL_MAX)
    j = np.arange(sc.mr)
    if mutation == "survivor dropped at a step boundary":
        gate[:, j % GM_STEP == GM_STEP - 1] = False
        gate_p[:, j % GM_STEP == GM_STEP - 1] = False
    if mutation == "survivor dropped at a tile boundary":
        gate[:, (j % GM_TILE == 0) & (j > 0)] = False
        gate_p[:, (j % GM_TILE == 0) & (j > 0)] = False
    last = mutation == "last j on ties"
    k7 = []
    for r in range(sc.ml):
        js = np.flatnonzero(gate[r])
        if len(js):
            b = fold(distances(sc, np.full(len(js), r), js), js.tolist(), sc.ratio, mutation == "float ratio product", last)
            if b >= 0:
                k7.append((r, b))
    pos = set()
    for r in range(sc.ml):
        js = np.flatnonzero(gate_p[r])
        if len(js):
            e = err[r, js]
            k = np.flatnonzero(e == e.min())
            pos.add((r, int(js[k[-1] if last else k[0]])))
        elif sc.pos_th == DBL_MAX:
            pos.add((0, 0))
    return _matches(k7), _matches(sorted(pos))


def _matches(ij):
    m = np.zeros(len(ij), oracle.MATCH_DTYPE)
    if ij:
        a = np.array(ij, np.int64)
        m["i"], m["j"] = a[:, 0], a[:, 1]
    return m


def _same(a, b):
    return len(a) == len(b) and np.array_equal(a["i"], b["i"]) and np.array_equal(a["j"], b["j"])


# ---------------------------------------------------------------------------------------------- CPU tests
def test_interval_arithmetic_encloses_exact_values():
    """Every enclosure holds the exact rational error: all undecided pairs of every scene and a sample of the others; exact points
    stay points (an error exactly on errorTh is decided)."""
    rng = np.random.default_rng(1)
    checked = 0
    for sc in scenes():
        lo, hi = sc.lohi()
        und, bad = np.broadcast_to(sc.iv.und, lo.shape), np.broadcast_to(sc.iv.bad, lo.shape)
        amb = np.argwhere(sc.cls == 0)
        defi = np.argwhere(~und & ~bad)
        sample = defi[rng.choice(len(defi), min(len(defi), 40), replace=False)] if len(defi) else defi
        for r, k in np.concatenate([amb, sample]):
            if und[r, k] or bad[r, k]:
                continue
            E = exact_error(sc.model, sc.M, sc.pl[r], sc.pr[k])
            if E is None:
                continue
            assert Fraction(float(lo[r, k])) <= E, (sc, r, k)
            assert hi[r, k] == math.inf or E <= Fraction(float(hi[r, k])), (sc, r, k)
            checked += 1
        assert np.all(lo[~und & ~bad] <= hi[~und & ~bad]), sc
    assert checked > 1000


def test_scenes_reach_their_edges(record_property):
    """Each scene contains what it was built for, computed from the interval classification.  The undecided pairs of the rounding
    scenes - whose exact and double decisions may differ - are reported with their exact decisions (test properties)."""
    for sc in scenes():
        lo, hi = sc.lohi()
        ex = np.broadcast_to(sc.iv.ex, lo.shape)
        if "threshold" in sc.props:
            on = ex & (lo == sc.th)
            assert on.sum() >= 2 and np.all(sc.cls[on] == -1), sc                   # err == errorTh exactly: a definite fail
            assert ((sc.cls == 1) & (lo > sc.th / 2)).any(), sc                      # errors just below errorTh pass
            assert ((sc.cls == -1) & (lo > sc.th) & (lo < 2 * sc.th)).any(), sc     # and just above fail
            assert not (sc.cls == 0).any(), sc
        if "rounding" in sc.props:
            amb = np.argwhere(sc.cls == 0)
            assert len(amb) > 0, sc
            assert (np.count_nonzero(sc.cls == 0, axis=1) <= 4).all(), sc
            exact_pass = sum(exact_error(sc.model, sc.M, sc.pl[r], sc.pr[k]) < Fraction(sc.th) for r, k in amb)
            record_property(f"{sc.name}.undecided", len(amb))
            record_property(f"{sc.name}.undecided_exactly_below_errorTh", exact_pass)
        if "epipole" in sc.props:
            assert np.all(sc.iv.und[0]) and np.all(sc.iv.und[4]) and (sc.cls[1:4] == 1).any(), sc
        if "w" in sc.props:
            und = np.broadcast_to(sc.iv.und, lo.shape)
            assert und[0].all() and und[3].all(), sc                                 # w == 0
            assert (sc.cls[1] == 1).sum() >= 3, sc                                   # w < 0 still transfers
        if sc.name.startswith(("class.u8.F.zero", "class.u8.H.zero", "class.u8.F.nan", "class.u8.H.nan")):
            assert np.all(sc.cls == -1) and np.all(sc.cls_pos == -1), sc
        if "ratio" in sc.props:
            assert sc.hits["exact"] or sc.ratio in (0.0, 1.0, 1.5), sc
            D = sc.cls == 1
            counts = D.sum(1)
            assert (counts == 1).any() and not (sc.cls == 0).any(), sc
            bd_sbd = []
            for r in np.flatnonzero(counts >= 2):
                d = np.sort(distances(sc, np.full(counts[r], r), np.flatnonzero(D[r])))
                bd_sbd.append((d[0], d[1]))
            assert any(b == s for b, s in bd_sbd), sc                                # duplicate distances
            assert any(b == sc.ratio * s for b, s in bd_sbd), sc                    # bd == fl(distRatio * sbd)
            if sc.ratio in (0.36, 0.64):
                assert any((b < sc.ratio * s) != (b < float(np.float32(sc.ratio) * np.float32(s))) for b, s in bd_sbd), sc
        if "structure" in sc.props and sc.mr == 2055:
            D = sc.cls == 1
            steps = [np.add.reduceat(D[r], np.arange(0, sc.mr, GM_STEP)) for r in range(sc.ml)]
            seen = set(np.concatenate(steps).tolist())
            assert {0, 7, 8, 9, 32} <= seen, sc
            assert any(D[r, :GM_TILE].any() and D[r, GM_TILE:2 * GM_TILE].any() for r in range(sc.ml)), sc
            assert any(D[r, GM_TILE - 8:GM_TILE].any() and D[r, GM_TILE:GM_TILE + 8].any() for r in range(sc.ml)), sc
            assert any(any(a == 7 and b == 32 for a, b in zip(s[:-1], s[1:])) for s in steps), sc     # 39 in the queue
        if "structure" in sc.props:
            assert sc.ml % 8 != 0 and not (sc.cls == 0).any(), sc
        if "allpass" in sc.props:
            assert np.all(sc.cls == 1), sc
    names = {sc.name for sc in scenes()}
    assert {f"structure.{m}.u8" for m in (1, 2, 31, 32, 33, 1023, 1024, 1025, 2055)} <= names
    assert {f"class.{k}.{m}" for k in ("u8", "f32", "real", "mixed", "bin") for m in "FH"} <= names


def test_oracle_passes_audits():
    """The oracles (compiled descriptor distances when the reference is built; the position-only loop) pass both audits on every
    scene, and so does the fault-free numpy model the rejection test perturbs."""
    for sc in scenes():
        want, want_p = oracle_guided(sc), oracle_positions(sc)
        audit_guided(want, sc)
        audit_positions(want_p, sc)
        k7, pos = simulate(sc)
        assert _same(k7, want) and _same(pos, want_p), sc


def test_audits_reject_wrong_results():
    """Each deliberate fault is caught by an audit on at least one scene: F transposed, H inverted, `<=` at errorTh, the ratio product
    in float, the last j of a tie, a survivor lost on a 32-wide step boundary and one lost on a 1024-position tile boundary."""
    caught = {m: [] for m in MUTATIONS}
    for m in MUTATIONS:
        for sc in scenes():
            if (m == "F transposed" and sc.model != 0) or (m == "H inverted" and sc.model != 1):
                continue
            if m == "H inverted" and not (np.all(np.isfinite(sc.M)) and abs(np.linalg.det(sc.M)) > 0):
                continue
            k7, pos = simulate(sc, m)
            for audit, res in ((audit_guided, k7), (audit_positions, pos)):
                try:
                    audit(res, sc)
                except AssertionError:
                    caught[m].append((sc.name, audit.__name__))
    missed = [m for m, c in caught.items() if not c]
    assert not missed, f"faults no audit caught: {missed}"
    for m in ("<= at the threshold", "last j on ties"):
        assert {a for _, a in caught[m]} == {"audit_guided", "audit_positions"}, (m, caught[m])


# ---------------------------------------------------------------------------------------------- GPU tests
def _regions(sc):
    from alicevision_b200 import Regions
    return Regions(sc.dl, sc.xl, binary=sc.binary), Regions(sc.dr, sc.xr, binary=sc.binary)


@pytest.mark.gpu
def test_gpu_guided_matching_one_pair():
    """matching.guidedMatching (b200m_guided_match_model, a list of one) on every scene: audited, and equal to the oracle."""
    from alicevision_b200 import matching
    ctx = matching.Context(0)
    try:
        for sc in scenes():
            L, R = _regions(sc)
            got = matching.guidedMatching(sc.M, L, R, sc.th, sc.ratio, ctx=ctx, model=sc.model, xy_left=sc.gl, xy_right=sc.gr)
            audit_guided(got, sc)
            assert _same(got, oracle_guided(sc)), sc
    finally:
        ctx.close()


_KCLASS = {"u8": "u8", "f32": "u8", "real": "f32", "bin": "bin", "mixed": "mixed"}


def _expected_launches(group, cap):
    """K7's launches for a list: per kernel class, batches of whole pairs up to `cap` left features (a larger pair runs alone), 4
    launches per batch (guided_pairs_kernel, the two of the scan, the emit) and one fp32 expansion per mixed pair."""
    launches = 0
    for k in set(_KCLASS.values()):
        n = l = 0
        for sc in group:
            if _KCLASS[sc.kind] != k:
                continue
            if n and l + sc.ml > cap:
                launches += 4
                n = l = 0
            n += 1
            l += sc.ml
        launches += 4 if n else 0
    return launches + sum(sc.kind == "mixed" for sc in group)


def _upload_all(ctx, keep):
    """Every scene's two views, with ids 2 k + 1 and 2 k + 2 for scene k; geometry positions where the scene has them."""
    from alicevision_b200 import matching
    ids = {}
    for k, sc in enumerate(scenes()):
        ids[sc.name] = (2 * k + 1, 2 * k + 2)
        for vid, d, xy, g in ((2 * k + 1, sc.dl, sc.xl, sc.gl), (2 * k + 2, sc.dr, sc.xr, sc.gr)):
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
@pytest.mark.parametrize("cap", [None, 16])
def test_gpu_guided_lists(monkeypatch, cap):
    """Context.guided_match_pairs over one list per (model, distRatio) holding all of its scenes with their own errorTh - at the default
    left bound, and with a bound of 16 left features per batch, which splits every list into several batches (last_launches() counts
    them) - and Context.guided_match_positions_pairs (undecorated) over one list per model: every result audited and equal to its
    oracle."""
    from alicevision_b200 import matching
    if cap:
        monkeypatch.setenv("B200M_GUIDED_LEFT_CAP", str(cap))
    groups = {}
    for sc in scenes():
        groups.setdefault((sc.model, sc.ratio), []).append(sc)
    ctx = matching.Context(0)
    keep = []
    split = False
    try:
        ids = _upload_all(ctx, keep)
        for (model, ratio), group in sorted(groups.items()):
            got = ctx.guided_match_pairs([ids[sc.name] for sc in group], [sc.M for sc in group], [sc.th for sc in group], ratio, model)
            launches = ctx.last_launches()
            assert ctx.last_records() == sum(len(g) for g in got)
            for sc, g in zip(group, got):
                audit_guided(g, sc)
                assert _same(g, oracle_guided(sc)), sc
            assert launches == _expected_launches(group, cap or (1 << 21)), (model, ratio, launches)
            if cap and sum(sc.ml for sc in group) > cap:                      # the list ran in more batches than at the default bound
                assert launches > _expected_launches(group, 1 << 21), (model, ratio)
                split = True
        for model in (0, 1):
            group = [sc for sc in scenes() if sc.model == model]
            got = ctx.guided_match_positions_pairs([ids[sc.name] for sc in group], [sc.M for sc in group], [sc.th for sc in group], model,
                                                   decorate=False)
            for sc, g in zip(group, got):
                audit_positions(g, sc)
                assert _same(g, oracle_positions(sc)), sc
        assert split == bool(cap)
    finally:
        ctx.close()
