"""K10 against an independent high-precision reference: the a-contrario RANSAC arithmetic checked in mpmath, not in acransac_math.h.

The engine and both oracle builds share alicevision_b200/csrc/acransac_math.h, so the engine-vs-oracle tests cannot see a wrong term
in that header.  Here every quantity is recomputed in mpmath at DPS significant digits from the raw inputs (the pixel coordinates,
the image sizes, the double coefficients a primitive is given), with the exact preconditioner s = 1 / sqrt(w h):

* CPU: the header's primitives through the oracle's C entry points (the cubic solver, both null spaces, fit7 / fit4, the epipolar
  and homography errors, the preconditioner, both unnormalisers, the 3 x 3 inverse, both logalpha0, the float logc tables), and
  ``audit()`` of the port's result on every scene of test_acransac.py and test_acransac_h.py;
* GPU: ``audit()`` of the engine's results on the same scenes, on every pair of the 500-pair lists, on the skip-off runs, and on
  adversarial scenes that also go through the engine-vs-oracle protocol.

Bounds.  u = 2^-53 is the unit roundoff of binary64 and gamma(k) = k u / (1 - k u) the usual bound of k chained roundings.  A
bound "c u x" counts the roundings along the longest chain of the double computation (c) against the sum of the absolute values
it rounds (x, evaluated in mp); each constant is derived where it is defined.  The residual checks of ``audit()`` carry the bound
as an interval per correspondence, so no tolerance is a bare constant.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
from mpmath import mp

import test_acransac as tf
import test_acransac_h as th
from oracle import acransac as acr_oracle
from oracle import acransac_h as acrh

DPS = 40
mp.dps = DPS
U = 2.0 ** -53                  # binary64 unit roundoff
UF = 2.0 ** -24                 # binary32 unit roundoff (the logc tables are float sums)
FLT_EPSILON = 2.0 ** -23
INF = mp.inf
# An mp singular value below this fraction of the matrix norm is an exact zero of a rank-deficient system: exactly degenerate inputs
# give singular values at the 10^-DPS level of the mp computation, every other input here gives ones above 10^-20.
MP_ZERO = mp.mpf(10) ** (-DPS // 2)


def gamma(k: int) -> float:
    return k * U / (1 - k * U)


def M(x) -> mp.mpf:
    return mp.mpf(float(x))   # exact: every double is an mpf


def mpmat(a) -> mp.matrix:
    a = np.asarray(a, np.float64)
    return mp.matrix([[M(v) for v in row] for row in a.reshape(a.shape[0], -1)])


def fro(A) -> mp.mpf:
    return mp.sqrt(sum(x * x for x in A))


@pytest.fixture(scope="module")
def pf():
    return acr_oracle.AcransacOracle("port")


@pytest.fixture(scope="module")
def ph():
    return acrh.AcransacHOracle("port")


# ------------------------------------------------------------------------------------------------------------ mp reference pieces
def norm_mp(w: int, h: int):
    """The exact preconditioner of preconditionerFromImageSize: (s, tx, ty) = (1 / sqrt(w h), -w s / 2, -h s / 2)."""
    s = 1 / mp.sqrt(w * h)   # w h as a Python int: exact
    return s, -mp.mpf(w) / 2 * s, -mp.mpf(h) / 2 * s


def nmat(n) -> mp.matrix:
    s, tx, ty = n
    return mp.matrix([[s, 0, tx], [0, s, ty], [0, 0, 1]])


def null_mp(A: mp.matrix):
    """(singular values, orthonormal basis of the exact null space as rows, rank) of A in mp."""
    _, S, V = mp.svd_r(A, full_matrices=True)
    sv = [S[i] for i in range(len(S))]
    top = max(sv) if sv else mp.mpf(0)
    rank = sum(1 for x in sv if x > MP_ZERO * top)
    return sv, [[V[r, c] for c in range(V.cols)] for r in range(rank, V.rows)], rank


def dist_to_span(v, basis) -> mp.mpf:
    """|(I - B^T B) v| for a unit vector v and orthonormal rows B."""
    r = list(v)
    for b in basis:
        d = mp.fsum(x * y for x, y in zip(v, b))
        r = [x - d * y for x, y in zip(r, b)]
    return fro(r)


def unit_dist(a, b) -> mp.mpf:
    """min(|a/|a| - b/|b||, |a/|a| + b/|b||): the distance of two vectors up to scale and sign."""
    na, nb = fro(a), fro(b)
    x = [p / na for p in a]
    y = [q / nb for q in b]
    return min(fro([p - q for p, q in zip(x, y)]), fro([p + q for p, q in zip(x, y)]))


def epipolar_rows(c) -> mp.matrix:
    """encodeEpipolarEquation of the correspondences c (k x 4) in mp."""
    return mp.matrix([[M(x2) * M(x1), M(x2) * M(y1), M(x2), M(y2) * M(x1), M(y2) * M(y1), M(y2), M(x1), M(y1), 1]
                      for x1, y1, x2, y2 in np.asarray(c, np.float64).reshape(-1, 4)])


def dlt_rows(c) -> mp.matrix:
    rows = []
    for x1, y1, x2, y2 in np.asarray(c, np.float64).reshape(-1, 4):
        X1, Y1, X2, Y2 = M(x1), M(y1), M(x2), M(y2)
        rows.append([X1, Y1, 1, 0, 0, 0, -X2 * X1, -X2 * Y1, -X2])
        rows.append([0, 0, 0, X1, Y1, 1, -Y2 * X1, -Y2 * Y1, -Y2])
    return mp.matrix(rows)


# Householder null space (acr::nullspace<R>): R reflections, each from a norm over at most 9 entries and applied with a 9-term dot
# product and an update: at most 2 * 9 + 4 roundings per reflection, so the computed Q is within R (2 * 9 + 4) u of an orthogonal
# matrix and A^T is within the same multiple of u (times |A|) of an exact Q R (backward stability).  The product A N checked below
# adds a 9-term dot product (9 roundings).
def c_householder(R: int) -> int:
    return R * (2 * 9 + 4)


def nullspace_bound(R: int, A: mp.matrix, sv) -> tuple[float, mp.mpf]:
    """(the bound on |A n| / |A|_F for a computed unit column n, the bound on its angle to the exact null space): a vector with
    |A n| <= eps |A| lies within eps |A| / sigma_r of the null space (sigma_r the smallest non-zero singular value), i.e. eps kappa(A)."""
    eps = (c_householder(R) + 9) * U
    nz = [x for x in sv if x > MP_ZERO * max(sv)]
    return eps, eps * fro([A[i, j] for i in range(A.rows) for j in range(A.cols)]) / min(nz)


# ------------------------------------------------------------------------------------------------------------ 1. the cubic solver
def _poly(r, lead=1.0):
    """Double coefficients, ascending, of lead * prod(x - r_i), each rounded once from the exact mp expansion."""
    x = [mp.mpf(1)]
    for ri in r:
        ri = mp.mpf(ri)
        x = [(x[i - 1] if i else 0) - ri * (x[i] if i < len(x) else 0) for i in range(len(x) + 1)]
    return np.array([float(lead * v) for v in x], np.float64)   # x[i]: the coefficient of x^i


def _cubic_families():
    rng = np.random.default_rng(7)
    fam = {}
    fam["distinct"] = np.array([_poly(sorted(rng.uniform(-5, 5, 3)), float(rng.choice([-1, 1]) * rng.uniform(0.1, 10))) for _ in range(24)]
                               + [_poly([-1e3, 0.5, 2.0]), _poly([1e-3, 2e-3, 7.0]), _poly([-3.0, -2.9999, 4.0])])
    # integer coefficients with an exact double root: CR2 == CQ3 holds in double (R < 0 for (x - 1)^2 (x - 4), R > 0 with the signs
    # flipped)
    fam["double_exact"] = np.array([_poly(r, lead) for r, lead in (([1, 1, 4], 1.0), ([-1, -1, -4], 1.0), ([2, 2, -1], 1.0), ([-2, -2, 1], 1.0),
                                                                    ([3, 3, 1], 2.0), ([0.5, 0.5, 3], 1.0), ([-0.5, -0.5, -3], -4.0))])
    fam["triple"] = np.array([[-8.0, 12.0, -6.0, 1.0], [27.0, 27.0, 9.0, 1.0], [-16.0, 24.0, -12.0, 2.0], [1.0, 3.0, 3.0, 1.0]])
    # (x - 1)^2 (x - 4) with c moved by a few ulps either side: the discriminant changes sign within rounding
    base = np.array([-4.0, 9.0, -6.0, 1.0])
    near = []
    for k in range(-12, 13):
        p = base.copy()
        p[0] = base[0] + k * np.spacing(4.0)
        near.append(p)
        q = base.copy()
        q[1] = base[1] + k * np.spacing(9.0)
        near.append(q)
    fam["near_double"] = np.array(near)
    fam["one_real"] = np.array([[1.0, 1.0, 1.0, 1.0], [-1.0, 1.0, -1.0, 1.0], [5.0, 0.5, 0.25, 2.0], [1e-3, 3.0, 0.0, 1.0],
                                [-2.0, 1e-8, 0.0, 1.0], [7.0, -2.0, 3.0, -0.5]])
    fam["tiny_leading"] = np.array([[1.0, -3.0, 2.0, 1e-12], [1.0, -3.0, 2.0, -1e-9], [2.0, 1.0, -1.0, 1e-15], [3.0, -1.0, 2.0, 1e-6]])
    fam["zero_constant"] = np.array([[0.0, 1.0, 2.0, 3.0], [-0.0, -1.0, 2.0, 1.0], [0.0, 0.0, 0.0, 1.0], [-0.0, 5.0, -4.0, 1e-9]])
    return fam


CUBIC_FAMILIES = _cubic_families()
# The solver's own error.  a, b, c carry one rounding; q and r five more (their largest terms are a^2, 3 |b| and 2 |a|^3, 9 |a b|,
# 27 |c|); Q, R one; sqrt(Q), sq3, R / sq3, acos (< 1 ulp), theta / 3, cos (< 1 ulp) and the final product and difference six:
# about 16 roundings on quantities of size T = |a| / 3 + 2 sqrt(|Q|) + (2 |R|)^(1/3) (the terms the last line adds) or T^2, T^3 in q, r.  A
# root of multiplicity 1 at distance d from the nearest other root moves by that relative error times T / d; a root of a cluster
# moves by at most T sqrt(that error) (the square-root law of a double root).  C_CUBIC = 64 doubles the count of 16 twice, for the
# cancellations in q and r, whose terms are up to 9 times |q| or |r|.
C_CUBIC = 64


def cubic_roots_mp(P):
    """The exact roots (complex mpc) of the polynomial with the double coefficients P (ascending), and the monic a, b, c."""
    p3 = M(P[3])
    a, b, c = M(P[2]) / p3, M(P[1]) / p3, M(P[0]) / p3
    return monic_roots([a, b, c]), (a, b, c)


def monic_roots(coef):
    """The complex roots of x^m + coef[0] x^(m-1) + ... + coef[-1] as the eigenvalues of the companion matrix at 3 DPS digits: a
    root of multiplicity 3 is then still accurate to DPS digits (the cube root of 10^(-3 DPS)), where polyroots' iteration fails."""
    m = len(coef)
    with mp.workdps(3 * DPS):
        C = mp.matrix(m, m)
        for j in range(m):
            C[0, j] = -coef[j]
        for i in range(1, m):
            C[i, i - 1] = 1
        ev = mp.eig(C, left=False, right=False)
    return [mp.mpc(x) for x in ev]


def cubic_root_bounds(roots, abc):
    """Per exact root: the distance within which the solver's root may lie (see C_CUBIC)."""
    a, b, c = abc
    q = a * a - 3 * b
    r = 2 * a ** 3 - 9 * a * b + 27 * c
    # |A| + |B| of the one-root branch are at most (2 |R|)^(1/3) + 2 sqrt(|Q|) (A^3 = |R| + sqrt(R^2 - Q^3) and B = Q / A)
    T = abs(a) / 3 + 2 * mp.sqrt(abs(q) / 9) + mp.cbrt(2 * abs(r) / 54) + mp.mpf(2) ** -1074
    e = C_CUBIC * U
    out = []
    for i, r in enumerate(roots):
        d = min(abs(r - x) for j, x in enumerate(roots) if j != i)
        out.append(e * T * min(max(1, 2 * T / d) if d > 0 else INF, 2 / math.sqrt(e)))
    return out


@pytest.mark.parametrize("family", sorted(CUBIC_FAMILIES))
def test_solve_cubic(pf, family):
    """SolveCubicPolynomial: bit for bit the compiled reference's, and every root within its conditioning of an exact mp root of the
    same double coefficients; a root count of 1 against 3 (or 3 against 1) only where two exact roots lie within that bound of each
    other (the discriminant's sign is decided by rounding); P[0] == +-0 returns no root."""
    Ps = CUBIC_FAMILIES[family]
    got = [pf.solve_cubic(P) for P in Ps]
    want = acr_oracle.reference_output(f"solve_cubic_{family}",
                                       lambda: tuple(acr_oracle.AcransacOracle("ref").solve_cubic(P) for P in Ps), acr_oracle.current("ref"))
    for P, g, w in zip(Ps, got, want):
        w = np.asarray(w, np.float64).reshape(-1)
        assert g.size == w.size and np.array_equal(g.view(np.uint64), w.view(np.uint64)), (family, P, g, w)
    for P, x in zip(Ps, got):
        if P[0] == 0:
            assert x.size == 0, (family, P)
            continue
        roots, abc = cubic_roots_mp(P)
        bnd = cubic_root_bounds(roots, abc)
        # finite: near a double root R / sq3 can round past +-1, and acos would return NaN; these families must not get there
        assert x.size in (1, 3) and np.isfinite(x).all(), (family, P, x)
        for xi in x:   # every returned root is near an exact root
            assert min(abs(M(xi) - r) - bd for r, bd in zip(roots, bnd)) <= 0, (family, P, x, roots)
        for r, bd in zip(roots, bnd):
            if abs(r.imag) > bd:
                continue   # a complex root: not expected in the output
            hit = min(abs(M(xi) - r) for xi in x)
            if hit > bd:   # a real root missed: only a cluster member whose partner was returned may be
                assert x.size == 1 and any(abs(r - o) <= 2 * bd for o in roots if o is not r), (family, P, x, roots)
        if x.size == 3:   # three roots reported: the exact ones are real, or a complex pair within the bound of the real axis
            assert all(abs(r.imag) <= bd for r, bd in zip(roots, bnd)), (family, P, x, roots)
            # the acos branch sorts its roots; the CR2 == CQ3 and triple-root branches return theirs in a fixed order
            assert x[0] <= x[1] <= x[2] or family in ("double_exact", "triple"), (family, P, x)


def test_cubic_families_reach_every_branch():
    """The families reach the four branches of the solver: triple root, CR2 == CQ3, three real roots by acos, one real root."""
    def branch(P):
        a, b, c = P[2] / P[3], P[1] / P[3], P[0] / P[3]
        q = a * a - 3.0 * b
        r = 2.0 * a * a * a - 9.0 * a * b + 27.0 * c
        CR2, CQ3 = 729.0 * r * r, 2916.0 * q * q * q
        return ("triple" if r / 54 == 0 and q / 9 == 0 else "equal" if CR2 == CQ3 else "acos" if CR2 < CQ3 else "one"), float(np.sign(r))
    seen = {f: {branch(P)[0] for P in Ps if P[0] != 0} for f, Ps in CUBIC_FAMILIES.items()}
    assert seen["triple"] == {"triple"} and seen["double_exact"] == {"equal"} and seen["one_real"] == {"one"}
    assert {"equal", "acos", "one"} <= seen["near_double"] and seen["distinct"] == {"acos"}
    assert {branch(P)[1] for P in CUBIC_FAMILIES["double_exact"]} == {-1.0, 1.0}   # R < 0 and R > 0 in the CR2 == CQ3 branch


# ------------------------------------------------------------------------------------------------------------ 2. null spaces
def _systems(R: int):
    rng = np.random.default_rng(11 + R)
    out = []
    for _ in range(6):
        out.append(("random", rng.normal(size=(R, 9))))
    for _ in range(3):
        A = rng.normal(size=(R, 9))
        A[-1] = A[0]                                  # a duplicated row
        out.append(("duplicated", A))
    c = rng.integers(-16, 17, (7 if R == 7 else 4, 4)) / 16.0
    c[:, 1] = 0.25 * c[:, 0] - 0.125                  # every point of image I on one line (dyadic: exact, as is every product)
    c[:, 3] = -0.5 * c[:, 2] + 0.0625                 # every point of image J on one line
    A = np.array(mpmat_to_float(epipolar_rows(c) if R == 7 else dlt_rows(c)))
    out.append(("collinear", A))
    A = rng.normal(size=(R, 9))
    A[1] = A[0] * (1 + 2 ** -40)                      # nearly duplicated
    out.append(("near_duplicate", A))
    A = rng.normal(size=(R, 9)) * np.array([1e-6] * 4 + [1.0] * 5)   # badly scaled columns
    out.append(("scaled", A))
    return out


def mpmat_to_float(A: mp.matrix):
    """The exact products as doubles: rows of data, so that the system the header sees and the one mp sees are the same."""
    return [[float(A[i, j]) for j in range(A.cols)] for i in range(A.rows)]


@pytest.mark.parametrize("R", [7, 8])
def test_nullspace(pf, ph, R):
    """acr::nullspace<R>: orthonormal columns; |A n| <= eps |A|; each column within eps kappa(A) of the exact mp null space (which is
    larger for rank-deficient systems: duplicated rows, collinear points)."""
    for kind, A in _systems(R):
        N = pf.nullspace7(A) if R == 7 else ph.nullspace8(A).reshape(1, 9)
        Am = mpmat(A)
        sv, basis, rank = null_mp(Am)
        eps, ang = nullspace_bound(R, Am, sv)
        assert len(basis) >= 9 - R and (rank < R) == (kind in ("duplicated", "collinear")), (R, kind, rank)
        Nm = [[M(v) for v in row] for row in N]
        # orthonormality: the computed Q is within c_householder(R) u of orthogonal (see c_householder)
        for i in range(len(Nm)):
            for j in range(len(Nm)):
                d = mp.fsum(x * y for x, y in zip(Nm[i], Nm[j])) - (1 if i == j else 0)
                assert abs(d) <= 2 * c_householder(R) * U, (R, kind, i, j, d)
        nA = fro([Am[i, j] for i in range(Am.rows) for j in range(Am.cols)])
        for n in Nm:
            An = fro([mp.fsum(Am[i, j] * n[j] for j in range(9)) for i in range(Am.rows)])
            assert An <= eps * nA, (R, kind, An / nA)
            assert dist_to_span([x / fro(n) for x in n], basis) <= ang + 2 * c_householder(R) * U, (R, kind)


# ------------------------------------------------------------------------------------------------------------ 3. fit7 / fit4
def det_bound(cm: float = 0.0) -> float:
    """|det F| / |F|_F^3 of a computed 7-point model.  det(f1 + a f2) is the cubic at the computed root: its coefficients sum 18 triple
    products of unit-basis entries each (2 roundings per product, 17 additions: gamma(21) times 18 (1 + |a|)^3 <= 18 2^(3/2) |F|^3),
    and the solver leaves a residual of C_CUBIC u on that scale; cm (the model's rounding after fitting, relative) adds 3 cm through
    the adjugate, and the engine's normalised points (C_POINT u on each side) 6 C_POINT u."""
    return (gamma(21) + C_CUBIC * U) * 18 * 2 ** 1.5 + 3 * cm + 6 * C_POINT * U


# A model found by the engine comes from a sample drawn in some order, whose Householder basis the audit does not know.  In a basis
# where det(f2) is small the cubic's leading coefficient is small, and SolveCubicPolynomial loses the other roots to the cancellation
# of the tiny_leading family (seen on the 500-pair list: a model 2.3e-9 from the exact one of its sample, |det| / |F|^3 = 1.8e-11;
# refitting the same 7 points in other orders gives the same spread).  So the audit bounds the determinant by the solver's
# square-root law instead: a root within T sqrt(C_CUBIC u) on the scale T >= |a| of its cubic moves a unit model by at most
# sqrt(C_CUBIC u), and |det| by at most 3 times that (|adj| <= 1 for a unit model), and it checks that the model is the exact rank-2
# member its own determinant places it nearest to.
AUDIT_DET_BOUND = 3 * math.sqrt(C_CUBIC * U)


def fit7_mp(c7, cm: float = 0.0, det_model=None):
    """The exact 7-point models of 7 correspondences: [(unit model as 9 mpf, bound on the distance of a computed model)], the
    models of the real roots of det(G1 + a G2) (and G2 when the cubic's leading coefficient vanishes), G1, G2 an orthonormal mp
    basis of the null space.  Also returns the rank of the epipolar system.

    Bound.  The header's basis f1, f2 spans a plane within ang = eps kappa(A) (nullspace_bound(7)) of the exact one, and its model's
    determinant is within det_bound() of 0.  Both are independent of the basis the header happened to pick.  In the exact basis, the
    model is then G(a + delta_a) up to ang (1 + |a|), where p(a) = det G(a) changes by at most num = ang (1 + |a|) |adj G|_F +
    det_bound |G|^3, so delta_a <= num / |p'(a)|, or sqrt(2 num / |p''(a)|) by the square-root law where p'(a) vanishes.  The model
    lies within 2 (ang (1 + |a|) + delta_a) / |G| of the exact one (the factor 2 covers the first-order expansion).  det_model: the
    audit's measured |det| / |F|^3 of the model, used in place of det_bound when larger (see AUDIT_DET_BOUND)."""
    A = epipolar_rows(c7)
    sv, basis, rank = null_mp(A)
    eps, ang = nullspace_bound(7, A, sv)
    if rank < 7:
        return [], rank, ang
    G1, G2 = basis
    det = lambda t: mp.det(mp.matrix([[G1[3 * i + j] + t * G2[3 * i + j] for j in range(3)] for i in range(3)]))  # noqa: E731
    ts = [mp.mpf(v) for v in (-1, 0, 1, 2)]
    coef = mp.lu_solve(mp.matrix([[t ** k for k in range(4)] for t in ts]), mp.matrix([det(t) for t in ts]))
    c = [coef[k] for k in range(4)]
    out = []
    rts = monic_roots([c[2] / c[3], c[1] / c[3], c[0] / c[3]]) if abs(c[3]) > MP_ZERO else monic_roots([c[1] / c[2], c[0] / c[2]])
    for r in rts:
        r = mp.mpc(r)
        if abs(r.imag) > MP_ZERO:
            continue
        a = r.real
        G = [G1[k] + a * G2[k] for k in range(9)]
        Gm = mp.matrix([[G[3 * i + j] for j in range(3)] for i in range(3)])
        adj = fro([Gm[(i + 1) % 3, (j + 1) % 3] * Gm[(i + 2) % 3, (j + 2) % 3] - Gm[(i + 1) % 3, (j + 2) % 3] * Gm[(i + 2) % 3, (j + 1) % 3]
                   for i in range(3) for j in range(3)])
        dp = abs(c[1] + 2 * c[2] * a + 3 * c[3] * a * a)
        d2 = abs(2 * c[2] + 6 * c[3] * a)
        num = ang * (1 + abs(a)) * adj + (det_bound(cm) if det_model is None else max(det_bound(cm), 2 * det_model)) * fro(G) ** 3
        da = min(num / dp if dp > 0 else INF, mp.sqrt(2 * num / d2) if d2 > 0 else INF)
        out.append((G, 2 * (ang * (1 + abs(a)) + da) / fro(G)))
    if abs(c[3]) <= MP_ZERO * max(abs(x) for x in c):
        out.append((list(G2), 2 * ang))
    return out, rank, ang


def _check_fit7(F_list, c7, what):
    """Every computed model is within its bound of an exact model (so within that bound of rank 2); every exact model set apart from
    the others by more than the bounds is returned."""
    models, rank, ang = fit7_mp(c7)
    A = epipolar_rows(c7)
    nA = fro([A[i, j] for i in range(A.rows) for j in range(A.cols)])
    for F in F_list:
        f = [M(v) for v in np.asarray(F).ravel()]
        nf = fro(f)
        # every model satisfies the 7 epipolar equations up to the null space's backward error (independent of the root's accuracy,
        # since both f1 and f2 do), plus 2 roundings of f1 + a f2
        An = fro([mp.fsum(A[i, j] * f[j] for j in range(9)) for i in range(7)])
        assert An <= ((c_householder(7) + 9) * U + gamma(2)) * nA * nf, (what, An / (nA * nf))
        if rank < 7:
            assert dist_to_span([x / nf for x in f], null_mp(A)[1]) <= ang, what
            continue
        d = [unit_dist(f, G) - b for G, b in models]
        assert d and min(d) <= 0, (what, [float(x) for x in d])
    if rank == 7:
        units = [np.asarray(F).ravel() / np.linalg.norm(F) for F in F_list]
        for i, (G, b) in enumerate(models):
            apart = all(unit_dist(G, H) > 2 * (b + bb) for j, (H, bb) in enumerate(models) if j != i)
            if apart and b < 1:   # a bound of 1 or more says little (unit vectors up to sign are at most sqrt(2) apart)
                assert any(unit_dist([M(v) for v in x], G) <= b for x in units), (what, "exact model not returned", float(b))


def _fit7_samples():
    rng = np.random.default_rng(21)
    out = [("known_answer", np.c_[np.array([[0, 0, 0, 1, 1, 1, 2], [0, 1, 2, 0, 1, 2, 0]], float).T,
                                  np.array([[0, 0, 0, 1, 1, 1, 2], [1, 2, 3, 1, 2, 3, 1]], float).T])]
    for k in range(8):
        out.append((f"random{k}", rng.uniform(-1, 1, (7, 4))))
    for k in range(4):   # 7 points of a real two-view scene, normalised as the kernel does
        c = tf.two_view_scene(40, 1.0, 500 + k, noise=0.0)[:7]
        out.append((f"scene{k}", _normalise(c, tf.WH)))
    c = rng.uniform(-1, 1, (7, 4))
    c[6] = c[5] + 1e-9                                  # two nearly coincident correspondences
    out.append(("near_duplicate", c))
    c = tf.two_view_scene(40, 1.0, 600, planar=True, noise=0.0)[:7]
    out.append(("planar", _normalise(c, tf.WH)))          # 7 points of a plane: a 3-D null space up to the scene's rounding
    c = rng.uniform(-1, 1, (7, 4))
    c[6] = c[0]
    out.append(("duplicate", c))                          # exactly degenerate
    return out


def _normalise(c, wh):
    n1 = (1 / math.sqrt(wh[0] * wh[1]), -wh[0] / 2, -wh[1] / 2)
    n2 = (1 / math.sqrt(wh[2] * wh[3]), -wh[2] / 2, -wh[3] / 2)
    return np.c_[(c[:, 0] + n1[1]) * n1[0], (c[:, 1] + n1[2]) * n1[0], (c[:, 2] + n2[1]) * n2[0], (c[:, 3] + n2[2]) * n2[0]]


@pytest.mark.parametrize("name,c7", _fit7_samples(), ids=[s[0] for s in _fit7_samples()])
def test_fit7(pf, name, c7):
    _check_fit7(pf.fit7(c7), c7, name)


def fit4_mp(c4):
    """(the exact DLT null vector or None when the null space is larger, the bound on a computed one's distance to it (up to scale
    and sign), the exact null space, its bound)."""
    L = dlt_rows(c4)
    sv, basis, rank = null_mp(L)
    _, ang = nullspace_bound(8, L, sv)
    return (basis[0] if rank == 8 else None), ang, basis


def _fit4_samples():
    rng = np.random.default_rng(31)
    out = []
    grid = np.array([[x, y] for x in (0.0, 1.0, 2.0) for y in (0.0, 1.0, 2.0)])
    Hgt = [np.eye(3), np.array([[1, 0, -4], [0, 1, 5], [0, 0, 1.0]]), np.array([[1, -2, 3], [4, 5, -6], [-7, 8, 1.0]])]
    for g, H in enumerate(Hgt):   # homographyKernel_test's ground truths on 4 grid points in general position
        for q, idx in enumerate(([0, 2, 6, 8], [0, 4, 5, 7], [1, 3, 5, 8])):
            x1 = grid[idx]
            p = np.c_[x1, np.ones(4)] @ H.T
            out.append((f"known_answer{g}_{q}", np.c_[x1, p[:, :2] / p[:, 2:]], H))
    for k in range(6):
        out.append((f"random{k}", rng.uniform(-1, 1, (4, 4)), None))
    c = rng.uniform(-1, 1, (4, 4))
    c[3, :2] = c[1, :2] + 1e-7 * (c[2, :2] - c[1, :2]) + (c[2, :2] - c[1, :2]) * 0.5   # three image-I points nearly collinear
    out.append(("near_collinear", c, None))
    c = rng.uniform(-1, 1, (4, 4))
    c[3] = c[1]
    out.append(("duplicate", c, None))
    c = rng.uniform(-1, 1, (4, 4))
    c[:, 1] = 0.5 * c[:, 0]
    c[:, 3] = -0.25 * c[:, 2] + 0.5
    out.append(("collinear", c, None))
    return out


@pytest.mark.parametrize("name,c4,Hgt", _fit4_samples(), ids=[s[0] for s in _fit4_samples()])
def test_fit4(ph, name, c4, Hgt):
    """fit4: the model equals the exact DLT null vector up to scale and sign within eps kappa(L); for a degenerate sample it lies in
    the larger exact null space.  The known answers also recover the ground truth."""
    H = ph.fit4(c4).ravel()
    h = [M(v) for v in H]
    v, ang, basis = fit4_mp(c4)
    # the computed vector is unit within the Householder bound, so its distance to a subspace bounds the angle
    if v is None:
        assert dist_to_span([x / fro(h) for x in h], basis) <= ang, name
    else:
        assert unit_dist(h, v) <= ang, (name, float(unit_dist(h, v)), float(ang))
    if Hgt is not None:
        assert unit_dist(h, [M(x) for x in Hgt.ravel()]) <= ang, name


# ------------------------------------------------------------------------------------------------------------ 4. residuals
def epi_mp(F, c):
    """Exact (d, L) of the epipolar error d^2 / L of correspondence c = (x1, y1, x2, y2) under F (9 mpf)."""
    x1, y1, x2, y2 = (M(v) for v in c)
    l = [F[3 * r] * x1 + F[3 * r + 1] * y1 + F[3 * r + 2] for r in range(3)]
    return l[0] * x2 + l[1] * y2 + l[2], l[0] ** 2 + l[1] ** 2


def epi_bound(F, c, e_exact):
    """The header's epipolar error is within this of the exact one (same double inputs).  l_r: two products and two additions,
    |delta l_r| <= gamma(3) (|F| |x1|)_r; d: gamma(3) more on |l| |x2|, so |delta d| <= gamma(6) D with D = |x2|^T |F| |x1|; L: the
    l_r errors, two squares and an addition; the quotient one more rounding.  Returned as the interval of d^2 / L."""
    x1, y1, x2, y2 = (abs(M(v)) for v in c)
    a = [abs(F[3 * r]) * x1 + abs(F[3 * r + 1]) * y1 + abs(F[3 * r + 2]) for r in range(3)]
    D = a[0] * x2 + a[1] * y2 + a[2]
    d, L = epi_mp(F, c)
    dd = gamma(6) * D
    l0, l1 = F[0] * M(c[0]) + F[1] * M(c[1]) + F[2], F[3] * M(c[0]) + F[4] * M(c[1]) + F[5]
    dL = 2 * (abs(l0) * gamma(3) * a[0] + abs(l1) * gamma(3) * a[1]) + (gamma(3) * a[0]) ** 2 + (gamma(3) * a[1]) ** 2 + gamma(2) * L
    lo = max(abs(d) - dd, 0) ** 2 / (L + dL) * (1 - gamma(3))
    hi = (abs(d) + dd) ** 2 / (L - dL) * (1 + gamma(3)) if L > dL else INF
    return lo, hi


def _class(x) -> str:
    return "nan" if math.isnan(x) else "inf" if math.isinf(x) else "finite"


def test_epipolar_error(pf):
    """FundamentalEpipolarDistanceError against mp: random F and points; a point on its line (d = 0, e = 0); a point at the epipole
    (l0 = l1 = 0: inf when d != 0, NaN when d == 0 too)."""
    rng = np.random.default_rng(41)
    for k in range(40):
        F = rng.normal(size=9) * (10.0 ** rng.integers(-3, 4))
        c = rng.uniform(-2, 2, (25, 4)) * (10.0 ** rng.integers(-2, 3))
        e = pf.errors(F, c)
        Fm = [M(v) for v in F]
        for ci, ei in zip(c, e):
            lo, hi = epi_bound(Fm, ci, None)
            assert lo <= M(ei) <= hi, (k, ci, ei, lo, hi)
    # integer data: every product and sum is exact, so the classes are the exact ones
    F = np.array([1.0, 0, -2, 0, 1, -3, 2, 5, 1])          # F (2, 3, 1) = (0, 0, 20): (2, 3) is the epipole of its own line
    cases = [((1.0, 1.0, 0.0, 0.0), None), ((2.0, 3.0, 5.0, 7.0), "inf"), ((1.0, 2.0, 2.0, 0.0), None)]
    Fz = np.array([1.0, 0, -2, 0, 1, -3, 0, 0, 0])           # l2 = 0 at the epipole as well: 0 / 0
    for ci, cls in cases:
        d, L = epi_mp([M(v) for v in F], ci)
        e = pf.errors(F, np.array([ci]))[0]
        want = "nan" if L == 0 and d == 0 else "inf" if L == 0 else "finite"
        assert _class(e) == want and (cls is None or cls == want), (ci, e)
        if want == "finite":
            assert M(e) == d * d / L or abs(M(e) - d * d / L) <= gamma(3) * d * d / L, (ci, e)
    on = np.array([[1.0, 1.0, 4.0, 2.0]])                   # l = F (1, 1, 1) = (-1, -2, 8): (4, 2) lies on it, d = 0 exactly
    assert pf.errors(F, on)[0] == 0.0 and epi_mp([M(v) for v in F], on[0])[0] == 0
    e = pf.errors(Fz, np.array([[2.0, 3.0, 5.0, 7.0]]))[0]
    assert math.isnan(e)


def homog_mp(H, c):
    """Exact (u, v, w) of H (x1, y1, 1)."""
    x1, y1 = M(c[0]), M(c[1])
    return [H[3 * r] * x1 + H[3 * r + 1] * y1 + H[3 * r + 2] for r in range(3)]


def homog_bound(H, c, du=None):
    """Interval of the header's HomographyAsymmetricError |x2 - (u, v) / w|^2 for the exact (u, v, w) and |delta (u, v, w)| <= du
    (default: the evaluation's own gamma(3) (|H| |x1|), two products and two additions); the quotient, the difference, the squares
    and the sum add one rounding each (gamma(4) on the result once the intervals are formed).  (0, inf) when w's interval holds 0."""
    x2, y2 = M(c[2]), M(c[3])
    u, v, w = homog_mp(H, c)
    if du is None:
        a = [abs(H[3 * r]) * abs(M(c[0])) + abs(H[3 * r + 1]) * abs(M(c[1])) + abs(H[3 * r + 2]) for r in range(3)]
        du = [gamma(3) * x for x in a]
    if abs(w) <= du[2]:
        return mp.mpf(0), INF
    comps = []
    for num, dn, x in ((u, du[0], x2), (v, du[1], y2)):
        qs = [(num + sn * dn) / (w + sw * du[2]) for sn in (-1, 1) for sw in (-1, 1)]
        lo, hi = min(qs), max(qs)
        if lo <= x <= hi:
            comps.append((mp.mpf(0), max(x - lo, hi - x)))
        else:
            comps.append((min(abs(x - lo), abs(x - hi)), max(abs(x - lo), abs(x - hi))))
    lo = (comps[0][0] ** 2 + comps[1][0] ** 2) * (1 - gamma(4))
    hi = (comps[0][1] ** 2 + comps[1][1] ** 2) * (1 + gamma(4))
    return lo, hi


def test_homography_error(ph):
    """HomographyAsymmetricError against mp: random H and points; w = 0 gives inf (u or v != 0) or NaN (u = v = 0, or an infinite
    and a NaN component), the class of the double expression."""
    rng = np.random.default_rng(43)
    for k in range(40):
        H = rng.normal(size=9) * (10.0 ** rng.integers(-3, 4))
        c = rng.uniform(-2, 2, (25, 4)) * (10.0 ** rng.integers(-2, 3))
        e = ph.errors(H, c)
        Hm = [M(v) for v in H]
        for ci, ei in zip(c, e):
            lo, hi = homog_bound(Hm, ci)
            assert lo <= M(ei) <= hi, (k, ci, ei, lo, hi)
    H = np.array([1.0, 2, 3, -1, 1, 0, 1, 1, -3])           # w = x + y - 3: zero on the line x + y = 3 (integers: exact)
    for ci in ((1.0, 2.0, 0.0, 0.0), (2.0, 1.0, 5.0, 5.0), (0.0, 3.0, 1.0, 1.0), (-3.0, 6.0, 0.0, 0.0)):
        u, v, w = homog_mp([M(x) for x in H], ci)
        assert w == 0
        cu = "nan" if u == 0 else "inf"
        cv = "nan" if v == 0 else "inf"
        want = "nan" if "nan" in (cu, cv) else "inf"
        assert _class(ph.errors(H, np.array([ci]))[0]) == want, (ci, u, v)


# ------------------------------------------------------------------------------------------------------------ 5. normalisation
SIZES = [(1, 1), (1, 7), (1001, 777), (1280, 960), (641, 1923), (8000, 50), (50, 8000), (20000, 15000), (46340, 46340)]
# w h < 2^31: the kernel forms w h as an int (preconditionerFromImageSize), so image sizes past that are outside its domain; the
# engine refuses them (test_acransac_h.py::test_gpu_bad_arguments).
assert all(w * h < 2 ** 31 for w, h in SIZES)


@pytest.mark.parametrize("w,h", SIZES)
def test_precondition(pf, w, h):
    """s = 1 / sqrt(w h) within 2 u (a square root and a division of an exact product); tx = (-.5f w) s within 3 u (the float
    product is exact below 2^24, then s's 2 u and one more rounding); a normalised coordinate s x + tx within 5 u (|s x| + |tx|)
    (s's 2 u, one product, one addition, and tx's 3 u)."""
    rng = np.random.default_rng(w * 31 + h)
    x = np.r_[rng.uniform(-2 * w, 3 * w, 50), 0.0, w, -1e9, 1e12, 0.5]
    y = np.r_[rng.uniform(-2 * h, 3 * h, 50), 0.0, h, 1e9, -1e12, 0.5]
    (s, tx, ty), xs, ys = pf.precondition(w, h, x, y)
    S, TX, TY = norm_mp(w, h)
    assert abs(M(s) - S) <= 2 * U * S
    assert abs(M(tx) - TX) <= 3 * U * abs(TX) and abs(M(ty) - TY) <= 3 * U * abs(TY)
    for X, Xn, T in ((x, xs, TX), (y, ys, TY)):
        for a, b in zip(X, Xn):
            exact = S * M(a) + T
            assert abs(M(b) - exact) <= 5 * U * (S * abs(M(a)) + abs(T)), (w, h, a, b)


WH4 = [(1280, 960, 1200, 900), (1, 1, 1, 1), (1001, 777, 641, 1923), (8000, 50, 50, 8000), (20000, 15000, 1280, 960), (3, 16, 16, 1)]


def _unnorm_err_bound(Nl, Fm, Nr):
    """Componentwise |Nl| |F| |Nr|: the sum of absolute values of the terms a 3 x 3 x 3 product rounds."""
    return [[mp.fsum(abs(Nl[i, a]) * abs(Fm[a, b]) * abs(Nr[b, j]) for a in range(3) for b in range(3)) for j in range(3)] for i in range(3)]


@pytest.mark.parametrize("wh", WH4)
def test_unnormalize(pf, wh):
    """UnnormalizerT: F <- N2^T F N1 within gamma(12) |N2^T| |F| |N1| componentwise: two chained 3-term products (gamma(6)) on N
    entries that carry 3 u each (s 2 u, tx 3 u), i.e. 6 u more on every term."""
    rng = np.random.default_rng(sum(wh))
    for _ in range(8):
        F = rng.normal(size=(3, 3))
        got = pf.unnormalize(wh, F)
        N1, N2 = nmat(norm_mp(*wh[:2])), nmat(norm_mp(*wh[2:]))
        Fm = mpmat(F)
        want = N2.T * Fm * N1
        bnd = _unnorm_err_bound(N2.T, Fm, N1)
        for i in range(3):
            for j in range(3):
                assert abs(M(got[i, j]) - want[i, j]) <= gamma(12) * bnd[i][j], (wh, i, j, got[i, j], want[i, j])


@pytest.mark.parametrize("wh", WH4)
def test_unnormalize_h(ph, wh):
    """UnnormalizerI: H <- N2^-1 H N1 within gamma(24) |N2^-1| |H| |N1|: N2^-1 by inverse3 carries 10 u per entry (N2's 3 u, cofactor
    products 2 u, the determinant 3 u, the reciprocal and the product 2 u), N1 3 u, and the two products 6 u; doubled for the products
    of perturbations and rounded up to 24."""
    rng = np.random.default_rng(sum(wh) + 1)
    for _ in range(8):
        H = rng.normal(size=(3, 3))
        got = ph.unnormalize(wh, H)
        N1, N2 = nmat(norm_mp(*wh[:2])), nmat(norm_mp(*wh[2:]))
        Hm = mpmat(H)
        N2i = N2 ** -1
        want = N2i * Hm * N1
        bnd = _unnorm_err_bound(N2i, Hm, N1)
        for i in range(3):
            for j in range(3):
                assert abs(M(got[i, j]) - want[i, j]) <= gamma(24) * bnd[i][j], (wh, i, j, got[i, j], want[i, j])


def test_inverse3(ph):
    """acr::inverse3 against mp: C(i, j) within gamma(2) of the sum of |products| it subtracts; det within gamma(3) of sum |C M| plus
    the cofactor errors; R = C^T / det within those relative errors plus 2 u (reciprocal and product)."""
    rng = np.random.default_rng(47)
    mats = [rng.normal(size=(3, 3)) for _ in range(20)] + [np.diag([1e-8, 1.0, 1e8]), np.array([[1, 2, 3], [4, 5, 6], [7, 8, 10.0]])]
    for w, h in SIZES:
        s = 1 / math.sqrt(w * h)
        mats.append(np.array([[s, 0, -w / 2 * s], [0, s, -h / 2 * s], [0, 0, 1]]))
    for A in mats:
        got = ph.inverse3(A)
        Am = mpmat(A)
        want = Am ** -1
        Cabs = [[abs(Am[(j + 1) % 3, (i + 1) % 3] * Am[(j + 2) % 3, (i + 2) % 3]) + abs(Am[(j + 1) % 3, (i + 2) % 3] * Am[(j + 2) % 3, (i + 1) % 3])
                 for j in range(3)] for i in range(3)]   # Cabs[i][j]: the terms of cofactor C(j, i)
        det = mp.det(Am)
        kdet = mp.fsum(Cabs[0][i] * abs(Am[i, 0]) for i in range(3)) / abs(det)   # condition of the first-column expansion
        rel_det = gamma(5) * kdet
        for i in range(3):
            for j in range(3):
                b = gamma(2) * Cabs[i][j] / abs(det) + abs(want[i, j]) * (rel_det + gamma(2)) + gamma(2) * gamma(5) * kdet * Cabs[i][j] / abs(det)
                assert abs(M(got[i, j]) - want[i, j]) <= b * (1 + 4 * rel_det), (A, i, j)


@pytest.mark.parametrize("wh", WH4)
def test_logalpha0_and_error_unnormalisation(pf, ph, wh):
    """logalpha0 of both kernels and unormalizeError against mp.
    F: log10(2 sqrt(w2^2 + h2^2) / (w2 h2) / s2) = log10(2 sqrt(w2^2 + h2^2) / sqrt(w2 h2)); the double argument carries the square root,
    two divisions and s2's 2 u (5 u), so the result is within 5 u / ln 10 plus log10's own 2 ulp.
    H: log10(pi / (w2 h2) / s2^2) = log10(pi) exactly for every size; the argument carries pi's rounding, the division, s2^2 (5 u)
    and the last division (8 u).
    unormalizeError(v) = sqrt(v) / s2 within 4 u (sqrt, division, s2's 2 u)."""
    w2, h2 = wh[2], wh[3]
    S = norm_mp(w2, h2)[0]
    la_f = mp.log10(2 * mp.sqrt(mp.mpf(w2) ** 2 + mp.mpf(h2) ** 2) / (mp.mpf(w2) * h2) / S)
    la_h = mp.log10(mp.pi)
    got_f, got_h = pf.logalpha0(wh), ph.logalpha0(wh)
    assert abs(M(got_f) - la_f) <= 5 * U / math.log(10) + 4 * U * abs(la_f), (wh, got_f, la_f)
    assert abs(M(got_h) - la_h) <= 8 * U / math.log(10) + 4 * U * abs(la_h), (wh, got_h, la_h)
    for v in (0.0, 1e-30, 2.5e-7, 0.3, 4.0, 1e10):
        for got in (pf.unnormalize_error(wh, v), ph.unnormalize_error(wh, v)):
            want = mp.sqrt(M(v)) / S
            assert abs(M(got) - want) <= 4 * U * want, (wh, v, got)


# ------------------------------------------------------------------------------------------------------------ 6. logc tables
def logc_running_bound(terms_a, terms_b, partial):
    """Running error bound of the float sum r_k = fl(r_{k-1} + fl(l10[a_k] - l10[b_k])), each l10 = (float)log10(m) rounded once:
    per step the two logs' roundings, the subtraction and the addition, u_f times the magnitudes involved (partial: the computed
    sums, which are the table entries)."""
    out, acc = [], mp.mpf(0)
    for a, b, p in zip(terms_a, terms_b, partial):
        la, lb = mp.log10(a), mp.log10(b)
        acc += UF * (abs(la) + abs(lb) + abs(la - lb) * (1 + UF) + abs(M(p)) * (1 + UF)) + 2 * UF * UF * (abs(la) + abs(lb))
        out.append(acc)
    return out


@pytest.mark.parametrize("n", [8, 9, 100, 1000, 8192])
@pytest.mark.parametrize("k", [4, 7])
def test_logc_tables_exact(ph, n, k):
    """logc_n[j] and logc_k[m] against the exact log10 C(n, j) and log10 C(m, k), within the running bound of their float sums
    (j, m <= n; both tables are 0 at and beyond the degenerate ends, as makelogcombi's logcombi returns)."""
    lcn, lck = ph.logc(k, n)
    ln10 = mp.log(10)
    lg = [mp.loggamma(m + 1) for m in range(n + 1)]
    half = n // 2
    bnd = logc_running_bound([n - i + 1 for i in range(1, half + 1)], list(range(1, half + 1)), lcn[1:half + 1])
    for j in range(1, n):
        jj = min(j, n - j)
        exact = (lg[n] - lg[j] - lg[n - j]) / ln10
        assert abs(M(lcn[j]) - exact) <= bnd[jj - 1], (n, j, float(lcn[j]), exact)
    assert lcn[0] == 0 and lcn[n] == 0
    for m in range(n + 1):
        if m <= k:
            assert lck[m] == 0
            continue
        kk = min(k, m - k)
        partial = np.cumsum(np.float32([np.float32(math.log10(m - i + 1)) - np.float32(math.log10(i)) for i in range(1, kk + 1)]), dtype=np.float32)
        b = logc_running_bound([m - i + 1 for i in range(1, kk + 1)], list(range(1, kk + 1)), partial)[-1]
        exact = (lg[m] - lg[k] - lg[m - k]) / ln10
        assert abs(M(lck[m]) - exact) <= b, (m, k, float(lck[m]), exact)


# ------------------------------------------------------------------------------------------------------------ 7. the audit
class Audit:
    """What audit() established, for the tests that want to look further (the rounding-level set, the kind of sample)."""

    def __init__(self):
        self.rounding_level: list[int] = []
        self.sample = "none"


def _prep(corr, wh):
    n1, n2 = norm_mp(*wh[:2]), norm_mp(*wh[2:])
    P = []
    for x1, y1, x2, y2 in np.asarray(corr, np.float64):
        X = [M(v) for v in (x1, y1, x2, y2)]
        p = (n1[0] * X[0] + n1[1], n1[0] * X[1] + n1[2], n2[0] * X[2] + n2[1], n2[0] * X[3] + n2[2])
        # |N| |x|: the magnitudes the engine's normalisation rounds (5 u each, test_precondition)
        a = (n1[0] * abs(X[0]) + abs(n1[1]), n1[0] * abs(X[1]) + abs(n1[2]), n2[0] * abs(X[2]) + abs(n2[1]), n2[0] * abs(X[3]) + abs(n2[2]))
        P.append((p, a))
    return n1, n2, P


# Rounding counts of the audit's residual intervals.  The engine scored its normalised model Mn on its rounded normalised points
# (5 u (|N| |x|) each, test_precondition); a valid result comes back unnormalised, within gamma(12) (F) or gamma(24) (H) of
# |N2^T| |Mn| |N1| (test_unnormalize*), and mapping it back to the normalised frame multiplies those terms by |N^-1| |N| <= 3
# componentwise on |N| |x| (|N^-1| |N| = [1 0 2|t|; 0 1 2|t|; 0 0 1] and |N| |x| >= |t|), i.e. by at most 9 on a point pair.
C_POINT = 5
C_MODEL = {"F": 12 * 9, "H": 24 * 9}


def _residual_intervals(model, Mn, P, valid, n2):
    """Per correspondence: (lo, hi) of the engine's squared residual, the exact residual, and rho (the algebraic residual over |Mn|
    |x1h| |x2h|, the quantity the minimal solver drives to its null space's backward error)."""
    cm = C_MODEL[model] * U if valid else 0.0
    nM = fro(Mn)
    out = []
    for p, a in P:
        x1, y1, x2, y2 = p
        a1 = (a[0], a[1], mp.mpf(1))
        nx1 = mp.sqrt(x1 * x1 + y1 * y1 + 1)
        nx2 = mp.sqrt(x2 * x2 + y2 * y2 + 1)
        if not all(mp.isfinite(v) for v in p):
            out.append((INF, INF, mp.nan, INF))
            continue
        q = [abs(Mn[3 * r]) * a1[0] + abs(Mn[3 * r + 1]) * a1[1] + abs(Mn[3 * r + 2]) for r in range(3)]
        l = [Mn[3 * r] * x1 + Mn[3 * r + 1] * y1 + Mn[3 * r + 2] for r in range(3)]
        if model == "F":
            D = q[0] * a[2] + q[1] * a[3] + q[2]
            d = l[0] * x2 + l[1] * y2 + l[2]
            L = l[0] ** 2 + l[1] ** 2
            # d: gamma(6) evaluation + 2 C_POINT u on the points + the model's cm; l0, l1: gamma(3) + C_POINT u + cm / 3 (only the rows
            # 0 and 1 of |N2^-T| |N2^T|, which are the identity's)
            dd = (gamma(6) + 2 * C_POINT * U + cm) * D
            dl = [(gamma(3) + C_POINT * U + cm / 3) * q[r] for r in range(2)]
            Llo = (max(abs(l[0]) - dl[0], 0) ** 2 + max(abs(l[1]) - dl[1], 0) ** 2) * (1 - gamma(2))
            Lhi = ((abs(l[0]) + dl[0]) ** 2 + (abs(l[1]) + dl[1]) ** 2) * (1 + gamma(2))
            e = d * d / L if L > 0 else (INF if d != 0 else mp.nan)
            lo = max(abs(d) - dd, 0) ** 2 / Lhi * (1 - gamma(1)) if Lhi > 0 else INF
            hi = (abs(d) + dd) ** 2 / Llo * (1 + gamma(1)) if Llo > 0 else INF
            rho = abs(d) / (nM * nx1 * nx2)
        else:
            t2 = (abs(n2[1]), abs(n2[2]))
            du = [(gamma(3) + C_POINT * U) * q[0] + cm * (q[0] + 2 * t2[0] * q[2]),
                  (gamma(3) + C_POINT * U) * q[1] + cm * (q[1] + 2 * t2[1] * q[2]),
                  (gamma(3) + C_POINT * U + cm) * q[2]]
            u_, v_, w_ = l
            if abs(w_) <= du[2]:
                lo, hi = mp.mpf(0), INF
            else:
                comps = []
                for num, dn, x, ax in ((u_, du[0], x2, a[2]), (v_, du[1], y2, a[3])):
                    qs = [(num + sn * dn) / (w_ + sw * du[2]) for sn in (-1, 1) for sw in (-1, 1)]
                    qlo, qhi = min(qs), max(qs)
                    xlo, xhi = x - C_POINT * U * ax, x + C_POINT * U * ax
                    dlo = max(xlo - qhi, qlo - xhi, 0)
                    dhi = max(abs(xhi - qlo), abs(qhi - xlo))
                    comps.append((dlo, dhi))
                lo = (comps[0][0] ** 2 + comps[1][0] ** 2) * (1 - gamma(4))
                hi = (comps[0][1] ** 2 + comps[1][1] ** 2) * (1 + gamma(4))
            e = (x2 - u_ / w_) ** 2 + (y2 - v_ / w_) ** 2 if w_ != 0 else INF
            rho = mp.sqrt((u_ - x2 * w_) ** 2 + (v_ - y2 * w_) ** 2) / (nM * nx1 * nx2)
        out.append((lo, hi, e, rho))
    return out


def _nfa_tools(model, n, wh, n2, logc):
    s = 7 if model == "F" else 4
    dim = 1 if model == "F" else 2
    w2, h2 = wh[2], wh[3]
    la0 = mp.log10(2 * mp.sqrt(mp.mpf(w2) ** 2 + mp.mpf(h2) ** 2) / (mp.mpf(w2) * h2) / n2[0]) if model == "F" else mp.log10(mp.pi)
    dla0 = (5 if model == "F" else 8) * U / math.log(10) + 4 * U * abs(la0)   # test_logalpha0_and_error_unnormalisation
    loge0 = mp.log10((3 if model == "F" else 1) * (n - s))
    lcn, lck = logc

    def nfa(e, k):
        """mpNFA(k) at the squared residual e, and the bound of the engine's double evaluation: per rank the log10 argument sqrt(e) +
        FLT_EPSILON carries 2 roundings (2 u / ln 10 on the log) and log10 itself 2 ulp; la0 its dla0; the NFA sum of 4 terms and one
        product 4 roundings of the magnitudes."""
        if e == INF or mp.isnan(e):
            return INF, mp.mpf(0)
        lg = mp.log10(mp.sqrt(e) + FLT_EPSILON)
        la = la0 + dim * lg
        v = loge0 + la * (k - s) + M(lcn[k]) + M(lck[k])
        tol = (k - s) * (dla0 + dim * (2 * U / math.log(10) + 4 * U * abs(lg))) + 4 * U * (abs(loge0) + abs(la) * (k - s) + abs(M(lcn[k])) + abs(M(lck[k])))
        return v, tol
    return s, nfa


def audit(result: dict, corr, wh, precision: float, model: str, logc=None) -> Audit:
    """Recomputes in mp what an a-contrario RANSAC result claims (A1..A6 of the module's checks).  result: the engine's or the
    oracle's dict ("valid", "inliers", "F" or "H", "error_max", "min_nfa"); corr: n x 4 pixels; wh = (wI, hI, wJ, hJ); model "F" or
    "H"; logc: the float tables (logc_n, logc_k) the NFA uses (pinned to makelogcombi bit for bit elsewhere)."""
    rep = Audit()
    corr = np.asarray(corr, np.float64).reshape(-1, 4)
    n = corr.shape[0]
    s = 7 if model == "F" else 4
    valid = bool(result["valid"])
    inl = np.asarray(result["inliers"], np.int64)
    nfa_g, em = float(result["min_nfa"]), float(result["error_max"])
    Mres = np.asarray(result[model], np.float64).ravel()
    # A1: distinct inliers, valid <=> min_nfa < 0; an invalid result reports no inlier
    assert len(set(inl.tolist())) == inl.size and (inl < n).all(), "A1: inliers"
    assert valid == (nfa_g < 0), ("A1: valid <=> min_nfa < 0", valid, nfa_g)
    if not valid:
        assert inl.size == 0, "A1: an invalid result lists inliers"
    if n <= s:   # ACRANSAC returns (0, 0) without a draw
        assert not valid and nfa_g == 0 and em == 0 and not Mres.any(), "A1: n <= sample size"
        return rep
    if nfa_g == math.inf:   # no model was ever scored (precision mode never switched): errorMax stays inf
        assert em == math.inf and not Mres.any(), "A1: unscored"
        return rep
    n1, n2, P = _prep(corr, wh)
    Mm = mpmat(Mres.reshape(3, 3))
    if valid:   # back to the normalised frame the engine scored in, with the exact preconditioners
        N1, N2 = nmat(n1), nmat(n2)
        Mn = N2.T ** -1 * Mm * N1 ** -1 if model == "F" else N2 * Mm * N1 ** -1
    else:       # the reference unnormalises only a meaningful model: an invalid result's model is still normalised
        Mn = Mm
    Mn = [Mn[i, j] for i in range(3) for j in range(3)]
    assert fro(Mn) > 0, "A6: zero model"
    R = _residual_intervals(model, Mn, P, valid, n2)
    lo = sorted(r[0] for r in R)
    hi = sorted(r[1] for r in R)
    if logc is None:
        logc = acrh.AcransacHOracle("port").logc(s, n)
    s, nfa = _nfa_tools(model, n, wh, n2, logc)
    thr = INF if precision == math.inf else M(precision) ** 2 * n2[0] ** 2
    dthr = 7 * U   # maxThreshold = precision^2 s2^2 in double: three products and s2's 2 u, twice
    # order statistics: if every engine residual lies in its interval, the engine's k-th smallest lies in [lo_k, hi_k]
    ks = range(s + 1, n + 1)
    cand = []
    for k in ks:
        if lo[k - 1] > thr * (1 + dthr):
            break                                    # beyond the precision prefix for certain
        vlo, tlo = nfa(lo[k - 1], k)
        vhi, thi = nfa(hi[k - 1], k)
        cand.append((k, vlo - tlo, vhi + thi, hi[k - 1] <= thr * (1 - dthr)))
    assert cand, "A4: no rank within the precision prefix"
    # A4: no rank is certainly lower than what the engine reports (only ranks certainly inside the prefix count)
    for k, vlo, vhi, inside in cand:
        if inside:
            assert M(nfa_g) <= vhi, ("A4: rank", k, "has a lower NFA", float(vhi), nfa_g)
    if valid:
        ks_ = inl.size
        # A1 / A4: the inlier count is a rank whose mp NFA is what the engine reports
        row = next((c for c in cand if c[0] == ks_), None)
        assert row is not None and row[1] <= M(nfa_g) <= row[2], ("A4: min_nfa is not mpNFA(k*)", ks_, nfa_g, row and (float(row[1]), float(row[2])))
        # A5: error_max = sqrt(e_k*) / s2 (sqrt, division and s2's 2 u: 4 u)
        e_lo, e_hi = lo[ks_ - 1], hi[ks_ - 1]
        assert mp.sqrt(e_lo) / n2[0] * (1 - 4 * U) <= M(em) <= mp.sqrt(e_hi) / n2[0] * (1 + 4 * U), ("A5", em, float(mp.sqrt(e_lo) / n2[0]))
        # A2: the list is in ascending residual order up to the intervals; exact ties (identical coordinates) by index
        for i in range(ks_ - 1):
            a, b = inl[i], inl[i + 1]
            assert R[a][0] <= R[b][1], ("A2: order", i, a, b, float(R[a][0]), float(R[b][1]))
        pos = {int(j): t for t, j in enumerate(inl)}
        rows = {}
        for j in inl:
            rows.setdefault(corr[j].tobytes(), []).append(int(j))
        for grp in rows.values():
            assert [pos[j] for j in sorted(grp)] == sorted(pos[j] for j in grp), ("A2: ties not by index", grp)
        # A3: the inlier set is the k* smallest: no outlier is certainly below an inlier
        mask = np.zeros(n, bool)
        mask[inl] = True
        top_in = max(R[j][0] for j in inl)
        out_min = min((R[j][1] for j in range(n) if not mask[j]), default=INF)
        assert top_in <= out_min, ("A3: an outlier is below an inlier", float(top_in), float(out_min))
    else:
        # an invalid result keeps the best rank's NFA and its raw (normalised) squared residual
        hits = [c for c in cand if c[1] <= M(nfa_g) <= c[2]]
        assert hits, ("A4: min_nfa matches no rank", nfa_g)
        assert any(lo[k - 1] * (1 - gamma(1)) <= M(em) <= hi[k - 1] * (1 + gamma(1)) for k, *_ in hits), ("A5: raw errorMax", em)
    # A6: the model is an exact fit of a minimal sample: at least s correspondences at rounding level.  A fitted correspondence has
    # rho <= (nullspace backward error) sqrt(R) max_j |x1h_j| |x2h_j| / (|x1h_i| |x2h_i|) (its row of the minimal system is within
    # that of 0 for both basis vectors, hence for any combination of them), plus the model's and the points' roundings (cm and 2
    # C_POINT u on |N| |x|, <= 3 |xh| per side); the max over all correspondences stands in for the unknown sample.
    rows_n = [mp.sqrt(p[0] ** 2 + p[1] ** 2 + 1) * mp.sqrt(p[2] ** 2 + p[3] ** 2 + 1) for p, _ in P if all(mp.isfinite(v) for v in p)]
    Rn = 2 * s
    eps_ns = (c_householder(Rn if model == "H" else 7) + 9) * U
    cm = C_MODEL[model] * U if valid else 0.0
    rmax = max(rows_n)
    tau = [(eps_ns * mp.sqrt(Rn) * rmax / (mp.sqrt(p[0] ** 2 + p[1] ** 2 + 1) * mp.sqrt(p[2] ** 2 + p[3] ** 2 + 1))
            + 9 * (cm + 2 * C_POINT * U + gamma(6))) if all(mp.isfinite(v) for v in p) else mp.mpf(0) for p, _ in P]
    rl = [i for i in range(n) if R[i][3] <= tau[i]]
    rep.rounding_level = rl
    assert len(rl) >= s, ("A6: fewer than s correspondences at rounding level", len(rl), sorted(float(R[i][3]) for i in range(n))[:s + 1])
    distinct = {}
    for i in rl:
        distinct.setdefault(corr[i].tobytes(), i)
    pts = sorted(distinct.values())
    Mu = [x / fro(Mn) for x in Mn]
    det_rel = abs(mp.det(mp.matrix([[Mn[3 * i + j] for j in range(3)] for i in range(3)]))) / fro(Mn) ** 3
    if len(pts) == s:
        sample = np.array([[float(v) for v in P[i][0]] for i in pts])   # the normalised points (doubles nearest the exact ones)
        if model == "F":
            models, rank, ang = fit7_mp(sample, cm, det_rel)
            if rank == 7:
                rep.sample = "regular"
                # the sample's doubles differ from the engine's by C_POINT u |N| |x| on each side and the model carries cm: the
                # null space bound's eps grows by those amounts (kappa times them on the angle)
                slack = 1 + 2 * C_POINT / (c_householder(7) + 9) + cm / ((c_householder(7) + 9) * U)
                assert any(unit_dist(Mu, G) <= b * slack for G, b in models), ("A6: not the fit of its sample",
                                                                            [float(unit_dist(Mu, G)) for G, b in models], [float(b) for _, b in models])
            else:
                rep.sample = "degenerate"
        else:
            v, ang, basis = fit4_mp(sample)
            if v is not None:
                rep.sample = "regular"
                slack = 1 + 2 * C_POINT / (c_householder(8) + 9) + cm / ((c_householder(8) + 9) * U)
                assert unit_dist(Mu, v) <= ang * slack, ("A6: not the fit of its sample", float(unit_dist(Mu, v)), float(ang))
            else:
                rep.sample = "degenerate"
    elif len(pts) < s:
        rep.sample = "degenerate"
    else:
        rep.sample = "ambiguous"   # more distinct correspondences at rounding level than a sample holds
    if model == "F":
        # rank 2 (for degenerate samples too), within AUDIT_DET_BOUND
        assert det_rel <= AUDIT_DET_BOUND + det_bound(cm), ("A6: rank", float(det_rel))
    return rep


def _logc_f(n):
    return acr_oracle.AcransacOracle("port").logc(n)


def _logc_h(n):
    return acrh.AcransacHOracle("port").logc(4, n)


def audit_f(res, corr, wh, prec):
    return audit(res, corr, wh, prec, "F", _logc_f(len(corr)))


def audit_h(res, corr, wh, prec):
    return audit(res, corr, wh, prec, "H", _logc_h(len(corr)))


# ------------------------------------------------------------------------------------------------------------ 8. audit of the port
@pytest.fixture(scope="module")
def port_f(pf):
    return {name: pf.estimate(*tf.scene(name)[:1], tf.WH, pf.mt_seed(tf.SEED), *tf.scene(name)[1:]) for name, *_ in tf.SCENES}


@pytest.fixture(scope="module")
def port_h(ph):
    return {name: ph.estimate(*th.scene(name)[:1], th.WH, ph.mt_seed(th.SEED), *th.scene(name)[1:]) for name, *_ in th.SCENES}


@pytest.mark.parametrize("name", [s[0] for s in tf.SCENES])
def test_audit_port_f(port_f, name):
    corr, _, prec = tf.scene(name)
    audit_f(port_f[name], corr, tf.WH, prec)


@pytest.mark.parametrize("name", [s[0] for s in th.SCENES])
def test_audit_port_h(port_h, name):
    corr, _, prec = th.scene(name)
    audit_h(port_h[name], corr, th.WH, prec)


def test_audit_rejects_wrong_results(port_f, port_h):
    """The audit is not vacuous: a result with a perturbed model, a dropped inlier, a shifted min_nfa, an unsquare-rooted errorMax or a
    swapped inlier order fails it."""
    corr, _, prec = tf.scene("r50_n100")
    good = port_f["r50_n100"]
    audit_f(good, corr, tf.WH, prec)
    F = np.array(good["F"], copy=True)
    F[0, 1] *= 1 + 1e-6
    bad = [dict(good, F=F), dict(good, inliers=good["inliers"][:-1]), dict(good, min_nfa=good["min_nfa"] - 1e-6),
           dict(good, error_max=good["error_max"] ** 2), dict(good, inliers=good["inliers"][::-1].copy())]
    for b in bad:
        with pytest.raises(AssertionError):
            audit_f(b, corr, tf.WH, prec)
    corr, _, prec = th.scene("plane_r50_n100")
    good = port_h["plane_r50_n100"]
    H = np.array(good["H"], copy=True)
    H[2, 0] *= 1 + 1e-6
    with pytest.raises(AssertionError):
        audit_h(dict(good, H=H), corr, th.WH, prec)


# ------------------------------------------------------------------------------------------------------------ 9. adversarial scenes
def near_planar_scene(n, ratio, seed, spread=1e-3):
    """A two-view scene whose points lie within `spread` of the plane z = 6 (the 7-point systems are close to a 3-D null space)."""
    c = tf.two_view_scene(n, ratio, seed, planar=True, noise=0.0)
    r = np.random.default_rng(seed + 1)
    K = np.array([[1000, 0, 640], [0, 1000, 480], [0, 0, 1.0]])
    X = np.c_[(c[:, :2] - [640, 480]) / 1000 * 6.0, np.full(n, 6.0)]
    X *= (1 + r.uniform(0, spread, n) / 6.0)[:, None]   # along the viewing ray of camera I: image I unchanged, depth 6 .. 6 + spread
    a = 0.2
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    p = (K @ (Ry @ X.T + np.array([-1.0, 0.1, 0.2])[:, None])).T
    out = r.random(n) >= ratio
    x2 = p[:, :2] / p[:, 2:] + r.normal(0, 0.3, (n, 2))
    x2[out] = r.uniform([0, 0], [1200, 900], (int(out.sum()), 2))
    return np.c_[c[:, :2] + r.normal(0, 0.3, (n, 2)), x2]


def _adversarial():
    """(name, model, corr, wh): scenes at the edges of the kernels' domains."""
    out = []
    out.append(("near_planar", "F", near_planar_scene(150, 0.8, 71), tf.WH))
    c = tf.two_view_scene(120, 0.7, 72)
    for wh in ((16, 12, 15, 9), (1, 1, 1, 1), (3, 16, 16, 1)):   # tiny images: the correspondences lie far outside them
        out.append((f"tiny_{wh[0]}x{wh[1]}", "F", c / 80.0, wh))
    out.append(("aspect_8000x50", "F", c * np.array([6.25, 50 / 960, 8000 / 1200, 50 / 900]), (8000, 50, 8000, 50)))
    d = tf.two_view_scene(8, 1.0, 73)
    d[7] = d[2]
    out.append(("n8_duplicate", "F", d, tf.WH))
    out.append(("identical_n50", "F", np.tile(tf.two_view_scene(1, 1.0, 74), (50, 1)), tf.WH))
    h = th.h_scene(150, 0.7, 75)
    for wh in ((16, 12, 15, 9), (1, 1, 1, 1)):
        out.append((f"h_tiny_{wh[0]}x{wh[1]}", "H", h / 80.0, wh))
    out.append(("h_aspect_50x8000", "H", h * np.array([50 / 1280, 8000 / 960, 50 / 1200, 8000 / 900]), (50, 8000, 50, 8000)))
    d = th.h_scene(5, 1.0, 76)
    d[4] = d[1]
    out.append(("h_n5_duplicate", "H", d, th.WH))
    out.append(("h_identical_n50", "H", np.tile(th.h_scene(1, 1.0, 77), (50, 1)), th.WH))
    # residuals that overflow to inf (image-J points at 1e200: |x2 - H x1|^2 > DBL_MAX) next to an inlier plane
    h = th.h_scene(120, 0.8, 78)
    h[::15, 2:] = 1e200
    out.append(("h_overflow", "H", h, th.WH))
    return out


ADVERSARIAL = _adversarial()


@pytest.mark.parametrize("name,model,corr,wh", ADVERSARIAL, ids=[a[0] for a in ADVERSARIAL])
def test_audit_port_adversarial(pf, ph, name, model, corr, wh):
    """The port on the adversarial scenes passes the audit (so the engine's comparison with it below means something)."""
    o = pf if model == "F" else ph
    res = o.estimate(corr, wh, o.mt_seed(tf.SEED), 20000)
    (audit_f if model == "F" else audit_h)(res, corr, wh, math.inf)


# ------------------------------------------------------------------------------------------------------------ 10. GPU: the engine
@pytest.fixture(scope="module")
def ctx():
    import alicevision_b200 as av
    return av.Context(0)


def _engine(ctx, model, corrs, whs, it=50000, prec=math.inf, seed=tf.SEED):
    from alicevision_b200 import matching
    st = matching.mt19937_state(seed)
    f = ctx.acransac_fundamental_pairs if model == "F" else ctx.acransac_homography_pairs
    return f(list(corrs), list(whs), st, it, prec)


@pytest.fixture(scope="module")
def gpu_f(ctx):
    out, groups = {}, {}
    for name, _, _, it, prec, _ in tf.SCENES:
        groups.setdefault((it, prec), []).append(name)
    for (it, prec), names in groups.items():
        out.update(zip(names, _engine(ctx, "F", [tf.scene(nm)[0] for nm in names], [tf.WH] * len(names), it, prec)))
    return out


@pytest.fixture(scope="module")
def gpu_h(ctx):
    out, groups = {}, {}
    for name, _, _, it, prec, _ in th.SCENES:
        groups.setdefault((it, prec), []).append(name)
    for (it, prec), names in groups.items():
        out.update(zip(names, _engine(ctx, "H", [th.scene(nm)[0] for nm in names], [th.WH] * len(names), it, prec)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s[0] for s in tf.SCENES])
def test_gpu_audit_f(gpu_f, name):
    """Every F scene, ILL_CONDITIONED included."""
    corr, _, prec = tf.scene(name)
    audit_f(gpu_f[name], corr, tf.WH, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s[0] for s in th.SCENES])
def test_gpu_audit_h(gpu_h, name):
    """Every H scene, DEGENERATE included."""
    corr, _, prec = th.scene(name)
    audit_h(gpu_h[name], corr, th.WH, prec)


def _list_500(model):
    """The 500-pair lists of test_gpu_500_pairs_default_iterations in test_acransac.py and test_acransac_h.py, pair for pair."""
    r = np.random.default_rng(3 if model == "F" else 4)
    corrs = []
    for k in range(500):
        n = int(r.integers(20, 400)) if k != 250 else 1500
        ratio = 0.7 if k == 250 else 0.0 if k % 3 else float(r.uniform(0.3, 0.9))
        corrs.append(tf.two_view_scene(n, ratio, 10_000 + k) if model == "F" else
                     th.h_scene(n, ratio, 20_000 + k, kind="rotation" if k % 2 else "plane"))
    return corrs


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["F", "H"])
def test_gpu_audit_500_pairs(ctx, model):
    """Every pair of the 500-pair list at maxIteration = 50000, not a sample."""
    corrs = _list_500(model)
    res = _engine(ctx, model, corrs, [tf.WH] * 500)
    assert sum(x["valid"] for x in res) >= 100
    fn = audit_f if model == "F" else audit_h
    for k, (r, c) in enumerate(zip(res, corrs)):
        try:
            fn(r, c, tf.WH, math.inf)
        except AssertionError as e:
            raise AssertionError(f"pair {k}: {e}") from e


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["F", "H"])
def test_gpu_audit_skip_off(ctx, model):
    """Every result of the runs with the certified skip disabled."""
    names = ["r10_n300", "r50_n100", "dup_n120", "planar_n150", "n9", "r70_n2000"] if model == "F" else \
        ["plane_r10_n300", "plane_r50_n100", "dup_n120", "collinear_n150", "n6", "rot_r70_n2000", "general_r80_n300"]
    mod = tf if model == "F" else th
    corrs = [mod.scene(nm)[0] for nm in names]
    ctx.set_acransac_skip(False)
    try:
        res = _engine(ctx, model, corrs, [mod.WH] * len(names))
        assert ctx.acransac_last_stats()["models_skipped"] == 0
    finally:
        ctx.set_acransac_skip(True)
    for nm, r, c in zip(names, res, corrs):
        (audit_f if model == "F" else audit_h)(r, c, mod.WH, math.inf)


# Scenes where the engine and the oracle part after the first meaningful model without a rounding-level NFA improvement to show for
# it.  On the 16 x 12 scene both traces agree up to iteration 4 (minNFA -40.34), then both improve at iteration 6, to -47.4 on the
# device and -66.0 on the host.  The samples after a meaningful model are drawn by position in its inlier list, which starts with the
# 7 fitted correspondences at rounding-level residuals, ordered by the last bits of the device and host acos / cos.  These scenes are
# checked for their outcome and by the audit, like ILL_CONDITIONED in test_acransac.py.
ORDER_FORK = {"tiny_16x12"}


@pytest.mark.gpu
@pytest.mark.parametrize("name,model,corr,wh", ADVERSARIAL, ids=[a[0] for a in ADVERSARIAL])
def test_gpu_adversarial(ctx, pf, ph, name, model, corr, wh):
    """The adversarial scenes through the engine-vs-oracle protocol and through the audit."""
    o, mod = (pf, tf) if model == "F" else (ph, th)
    got = _engine(ctx, model, [corr], [wh], 20000)[0]
    want = o.estimate(corr, wh, o.mt_seed(tf.SEED), 20000)
    if name in ORDER_FORK:
        assert got["valid"] == bool(want["valid"]), name
    else:
        mod._matches_oracle(got, want, name, corr)
    (audit_f if model == "F" else audit_h)(got, corr, wh, math.inf)
