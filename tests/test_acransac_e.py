"""K10 essential-matrix policy (b200m_acransac_essential_pairs, GeometricFilterMatrix_E_AC::geometricEstimation).

CPU: the oracle's "ref" build (the reference's ACRANSAC, sampler and NFA compiled verbatim around the restated E kernel) equals the
port bit for bit, generator end state included, live or from tests/golden/reference_acransac_e.npz; the 5-point solver and its
eigen-solve are audited against an exact (mpmath) reference.
GPU: the engine equals the port bit for bit on a list that mixes small pairs, pure outliers, a precision-mode pair and shared and
per-pair generator states; bad arguments are rejected.
"""
from __future__ import annotations

import zlib

import numpy as np
import pytest

mp = pytest.importorskip("mpmath")

import oracle  # noqa: E402
from oracle import acransac_e  # noqa: E402

SEED = 5489


def _rot(a: float, b: float, c: float) -> np.ndarray:
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def K_of(f: float, w: int, h: int) -> np.ndarray:
    return np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1.0]])


def e_scene(n: int, inlier_ratio: float, seed: int, noise: float = 0.5, translation=(0.6, 0.05, 0.1), rot=(0.02, 0.15, 0.01),
            KI=None, KJ=None, wh=(640, 480), planar: bool = False):
    """Pixels (n x 4) of a calibrated pair: inliers project random 3-D points (or points of one plane) through K_I [I | 0] and
    K_J [R | t] with Gaussian pixel noise; outliers are uniform in the image.  Returns (corr, (K_I, K_J), R, t)."""
    rng = np.random.default_rng(seed)
    KI = K_of(700.0, *wh) if KI is None else KI
    KJ = KI if KJ is None else KJ
    R, t = _rot(*rot), np.asarray(translation, np.float64)
    X = rng.uniform(-1.5, 1.5, (n, 3)) + [0, 0, 6]
    if planar:
        X[:, 2] = 6 + 0.1 * X[:, 0]
    xI = (KI @ X.T).T
    Xc = (R @ X.T).T + t
    xJ = (KJ @ Xc.T).T
    corr = np.concatenate([xI[:, :2] / xI[:, 2:], xJ[:, :2] / xJ[:, 2:]], axis=1) + rng.normal(0, noise, (n, 4))
    n_out = n - int(round(inlier_ratio * n))
    out = rng.permutation(n)[:n_out]
    corr[out] = rng.uniform(0, 1, (n_out, 4)) * [wh[0], wh[1], wh[0], wh[1]]
    return corr, (KI, KJ), R, t


# name, n, inlier ratio, maxIteration, precision (ACRANSAC's argument), scene kwargs
SCENES = [
    ("r90_n200", 200, 0.9, 5000, np.inf, {}),
    ("r50_n300", 300, 0.5, 5000, np.inf, {}),
    ("r20_n400", 400, 0.2, 5000, np.inf, {}),
    ("r0_n150", 150, 0.0, 1000, np.inf, {}),
    ("n6", 6, 1.0, 100, np.inf, {}),
    ("n7", 7, 1.0, 100, np.inf, {}),
    ("n9", 9, 0.8, 200, np.inf, {}),
    ("n5", 5, 1.0, 100, np.inf, {}),
    ("precision16_n300", 300, 0.6, 3000, 16.0, {}),
    ("precision_tiny_n200", 200, 0.6, 1000, 1e-8, {}),
    ("precision4_r60_n400", 400, 0.6, 3000, 4.0, {}),
    ("planar_r80_n300", 300, 0.8, 3000, np.inf, {"planar": True}),
    ("rotation_r80_n300", 300, 0.8, 3000, np.inf, {"translation": (1e-3, 0, 0)}),
    ("twoK_r70_n300", 300, 0.7, 3000, np.inf, {"KJ": np.array([[900.0, 0, 300], [0, 880, 250], [0, 0, 1]]), "wh": (600, 500)}),
    ("max1_n100", 100, 0.8, 1, np.inf, {}),
    ("max11_n100", 100, 0.8, 11, np.inf, {}),
]


def scene(name):
    _, n, r, _, _, kw = next(s for s in SCENES if s[0] == name)
    return e_scene(n, r, seed=zlib.crc32(name.encode()), **kw)


def _params(name):
    return next((it, prec, kw.get("wh", (640, 480))) for nm, _, _, it, prec, kw in SCENES if nm == name)


@pytest.fixture(scope="module")
def port():
    return acransac_e.AcransacEOracle("port")


@pytest.fixture(scope="module")
def port_all(port):
    st = port.mt_seed(SEED)
    out = {}
    for name, *_ in SCENES:
        corr, K, _, _ = scene(name)
        it, prec, wh = _params(name)
        out[name] = port.estimate(corr, K, wh, st, it, prec)
    return out


def reference(name):
    live = acransac_e.available("ref")

    def compute():
        o = acransac_e.AcransacEOracle("ref")
        corr, K, _, _ = scene(name)
        it, prec, wh = _params(name)
        r = o.estimate(corr, K, wh, o.mt_seed(SEED), it, prec)
        return tuple(r[k] for k in acransac_e.FIELDS)
    return dict(zip(acransac_e.FIELDS, acransac_e.reference_output(f"acransac_e_{name}", compute, live)))


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_oracle_ref_equals_port(port_all, name):
    """The port is the compiled reference's loop, sampler and NFA (d = 0.5) bit for bit, generator end state included."""
    want, got = reference(name), port_all[name]
    for k in acransac_e.FIELDS:
        assert oracle._same(got[k], want[k]), (name, k)


def test_scenes_cover_both_outcomes(port_all):
    v = {k: bool(r["valid"]) for k, r in port_all.items()}
    assert v["r90_n200"] and v["r50_n300"] and v["twoK_r70_n300"]
    # pure outliers still give a model: with d = 0.5 and alpha0 from the whole image, NFA(n) < 0 at the largest residual (the
    # reference's behaviour; featureMatching's overlap cut removes such pairs)
    assert v["r0_n150"] and not v["n5"] and not v["precision_tiny_n200"]
    assert int(port_all["n5"]["iterations"]) == 0 and np.array_equal(port_all["n5"]["mt_state_out"], acransac_e.AcransacEOracle("port").mt_seed(SEED))


# ---------------------------------------------------------------------------------------------------------------- exact audit
@pytest.fixture(autouse=True)
def _digits():
    """50 significant digits for every mpmath computation here (other modules set their own precision)."""
    with mp.workdps(50):
        yield


def _epi_rows(c):
    return [[c[i, 2] * c[i, 0], c[i, 2] * c[i, 1], c[i, 2], c[i, 3] * c[i, 0], c[i, 3] * c[i, 1], c[i, 3], c[i, 0], c[i, 1], 1.0]
            for i in range(c.shape[0])]


def audit_model(E, c5, bound: float = 1e-9, epi_bound: float | None = None) -> None:
    """E (any scale) satisfies the five epipolar constraints (to epi_bound, default bound), det E = 0 and 2 E E^T E - tr(E E^T) E = 0
    (to bound), relative to its norm."""
    Em = mp.matrix(E.tolist())
    nrm = mp.sqrt(sum(Em[i, j] ** 2 for i in range(3) for j in range(3)))
    Em = Em / nrm
    for row in _epi_rows(c5):
        r = sum(mp.mpf(row[3 * i + j]) * Em[i, j] for i in range(3) for j in range(3))
        scale = mp.sqrt(sum(mp.mpf(x) ** 2 for x in row))
        assert abs(r) <= (bound if epi_bound is None else epi_bound) * scale, ("epipolar", float(r))
    assert abs(mp.det(Em)) <= bound, ("det", float(mp.det(Em)))
    EEt = Em * Em.T
    tr = EEt[0, 0] + EEt[1, 1] + EEt[2, 2]
    C = 2 * EEt * Em - tr * Em
    assert max(abs(C[i, j]) for i in range(3) for j in range(3)) <= bound, "trace constraint"


def _normalised_sample(rng, R, t, noise=0.0, kind="random"):
    X = rng.uniform(-1, 1, (5, 3)) + [0, 0, 4]
    if kind == "coplanar":
        X[:, 2] = 4 + 1e-7 * rng.normal(size=5)
    elif kind == "duplicate":
        X[4] = X[3] + 1e-9
    x1 = X[:, :2] / X[:, 2:]
    Xc = (R @ X.T).T + t
    x2 = Xc[:, :2] / Xc[:, 2:]
    return np.concatenate([x1, x2], axis=1) + noise * rng.normal(size=(5, 4))


def _cross(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def test_fit5_known_answer(port):
    """On noise-free samples one returned model is [t]x R up to scale and sign, to 1e-9."""
    rng = np.random.default_rng(1)
    for _ in range(40):
        R = _rot(*rng.uniform(-0.3, 0.3, 3))
        t = rng.normal(size=3); t /= np.linalg.norm(t)
        c = _normalised_sample(rng, R, t)
        ms = port.fit5(c)
        assert 1 <= len(ms) <= 10
        E0 = _cross(t) @ R
        E0 /= np.linalg.norm(E0)
        best = min(min(np.linalg.norm(m / np.linalg.norm(m) - E0), np.linalg.norm(m / np.linalg.norm(m) + E0)) for m in ms)
        assert best <= 1e-9, best


@pytest.mark.parametrize("kind", ["random", "coplanar", "rotation", "duplicate"])
def test_fit5_models_satisfy_constraints(port, kind):
    """Every model of seeded samples satisfies the essential constraints, relative to |E|: to 1e-9 on random samples, 1e-6 on nearly
    coplanar or nearly duplicated points, 1e-2 on a nearly pure rotation (|t| = 1e-3: the worst model measured 1e-3; the rows then
    nearly admit every [t]x R, so the constraint matrix is ill-conditioned: test_real_root_count_on_action_matrices measures action
    matrices with entries of 1e7 there).  The five epipolar constraints hold to 1e-9 for every kind."""
    rng = np.random.default_rng({"random": 2, "coplanar": 3, "rotation": 4, "duplicate": 5}[kind])
    n_models = 0
    for _ in range(30):
        R = _rot(*rng.uniform(-0.3, 0.3, 3))
        t = rng.normal(size=3)
        t = t / np.linalg.norm(t) * (1e-3 if kind == "rotation" else 1.0)
        c = _normalised_sample(rng, R, t, noise=1e-3 if kind == "random" else 0.0, kind=kind)
        for m in port.fit5(c):
            audit_model(m, c, {"random": 1e-9, "coplanar": 1e-6, "duplicate": 1e-6, "rotation": 1e-2}[kind], epi_bound=1e-9)
            n_models += 1
    assert n_models > 0


# The real-vs-complex decision: the solver's count of eigenvalues with imag() == 0 against a 50-digit eigen-solve.  A complex pair whose
# |Im| / |lambda| is below MARGIN can be decided either way by rounding (the known divergence from Eigen, DESIGN §4): such matrices are
# counted and listed, not compared.
MARGIN = 1e-8


def _action_like(rng, n_real: int):
    """A 10 x 10 matrix with n_real real eigenvalues and (10 - n_real) / 2 complex pairs, mixed by a random similarity."""
    D = np.zeros((10, 10))
    i = 0
    for _ in range(n_real):
        D[i, i] = rng.normal(); i += 1
    while i < 10:
        a, b = rng.normal(), rng.uniform(0.05, 2.0)
        D[i:i + 2, i:i + 2] = [[a, b], [-b, a]]; i += 2
    S = rng.normal(size=(10, 10))
    return S @ D @ np.linalg.inv(S)


def test_eigen_real_count_against_mp(port):
    rng = np.random.default_rng(7)
    close = []
    for trial in range(60):
        n_real = [0, 2, 4, 6, 8, 10][trial % 6]
        A = _action_like(rng, n_real) if trial % 2 == 0 else rng.normal(size=(10, 10))
        got = port.eigen(A)
        assert got is not None
        re, im = got
        ev = mp.eig(mp.matrix(A.tolist()), left=False, right=False)
        real = [abs(mp.im(e)) <= mp.mpf(10) ** -40 * max(abs(e), 1) for e in ev]   # 50 digits: a real root keeps |Im| ~ 1e-50
        ratios = sorted(float(abs(mp.im(e)) / abs(e)) for e, r in zip(ev, real) if not r)
        want = sum(real)
        if ratios and ratios[0] < MARGIN:
            close.append((trial, ratios[0]))
            continue
        assert int(np.sum(im == 0)) == want, (trial, im, want)
        # the real ones agree with the exact values
        exact = sorted(float(mp.re(e)) for e in ev if abs(mp.im(e)) <= mp.mpf(10) ** -40 * max(abs(e), 1))
        assert np.allclose(sorted(re[im == 0]), exact, rtol=1e-7, atol=1e-9), trial
    assert len(close) <= 3, close   # listed: random draws essentially never land within the margin


def test_fit5_model_count_parity(port):
    """The solver's model count on noisy random samples is at most 10 and has the parity of 10: the non-real roots come in conjugate
    pairs."""
    rng = np.random.default_rng(11)
    for _ in range(50):
        R = _rot(*rng.uniform(-0.5, 0.5, 3)); t = rng.normal(size=3)
        c = _normalised_sample(rng, R, t, noise=1e-2)
        k = len(port.fit5(c))
        assert 0 <= k <= 10 and (10 - k) % 2 == 0, k


# ---------------------------------------------------------------------------------------------------------------- result audit
def _logc(n):
    """The float logc tables of sample size 5 (makelogcombi, pinned bit for bit by the planar tests' oracle)."""
    from oracle import acransac_h
    return acransac_h.AcransacHOracle("port").logc(5, n)


def _mp_inv(K):
    return mp.matrix(np.asarray(K, np.float64).tolist()) ** -1


def audit_e(result: dict, corr, K, wh_j, precision: float, logc=None) -> str:
    """An audit of one ACRANSAC result of the E kernel, from the inputs alone and in 50-digit arithmetic (no code of acransac_math.h):
    K^-1, F = K_J^-T E K_I^-1, every residual, logalpha0 = log10(2 D / A * .5) and the NFA with d = 0.5.  Checks the inlier set (the k
    smallest residuals, ties at rounding level excepted) and its order (ascending residual), errorMax = sqrt(e_k*), minNFA = NFA(k*)
    and that k* is that model's best rank, and that the model is the exact 5-point fit of the 5 inliers it passes through (the sample:
    residuals at rounding level; E satisfies their epipolar rows in K^-1 coordinates, det E = 0 and the trace constraint).  Returns a
    one-word outcome."""
    c = np.asarray(corr, np.float64).reshape(-1, 4)
    n = c.shape[0]
    inl = np.asarray(result["inliers"], np.int64)
    if not bool(result["valid"]):
        assert inl.size == 0
        return "invalid"
    k = inl.size
    assert 5 < k <= n and len(set(inl.tolist())) == k
    E = mp.matrix(np.asarray(result["E"], np.float64).reshape(3, 3).tolist())
    iI, iJ = _mp_inv(K[0]), _mp_inv(K[1])
    F = iJ.T * E * iI
    e = []
    for i in range(n):
        xI = mp.matrix([c[i, 0], c[i, 1], 1]); xJ = mp.matrix([c[i, 2], c[i, 3], 1])
        l = F * xI
        d = l[0] * xJ[0] + l[1] * xJ[1] + l[2]
        e.append(d * d / (l[0] ** 2 + l[1] ** 2))
    tol = lambda v: mp.mpf(1e-7) * v + mp.mpf(1e-24)  # noqa: E731  (double residuals vs exact ones)
    ein = [e[i] for i in inl]
    for a, b in zip(ein, ein[1:]):                 # order: ascending residual
        assert a <= b + tol(b), "inlier order"
    out = sorted(set(range(n)) - set(inl.tolist()))
    if out:
        assert max(ein) <= min(e[i] for i in out) + tol(max(ein)), "inlier set"
    maxthr = mp.inf if precision == np.inf else mp.mpf(precision) ** 2
    assert max(ein) <= maxthr + tol(maxthr if maxthr != mp.inf else 0), "threshold"
    em = mp.sqrt(max(ein))
    assert abs(mp.mpf(float(result["error_max"])) - em) <= mp.mpf(1e-6) * em + mp.mpf(1e-12), ("errorMax", float(em), result["error_max"])
    w, h = wh_j
    la0 = mp.log10(2 * mp.sqrt(mp.mpf(w) ** 2 + mp.mpf(h) ** 2) / (mp.mpf(w) * h) * mp.mpf("0.5"))
    loge0 = mp.log10(10 * (n - 5))
    lcn, lck = logc if logc is not None else _logc(n)
    se = sorted(e)

    def nfa(ek, kk):
        return loge0 + (la0 + mp.mpf("0.5") * mp.log10(mp.sqrt(ek) + mp.mpf(float(np.finfo(np.float32).eps)))) * (kk - 5) + \
            mp.mpf(float(lcn[kk])) + mp.mpf(float(lck[kk]))
    got = nfa(se[k - 1], k)
    assert abs(mp.mpf(float(result["min_nfa"])) - got) <= mp.mpf(1e-6) * max(1, abs(got)), ("minNFA", float(got), result["min_nfa"])
    assert got < 0
    best = min(nfa(se[kk - 1], kk) for kk in range(6, n + 1) if se[kk - 1] <= maxthr)
    assert got <= best + mp.mpf(1e-6) * max(1, abs(best)), ("best rank", float(got), float(best))
    # the sample: the 5 inliers of smallest residual lie on the model to rounding
    scale = max(float(abs(x)) for x in F) * (w + h) ** 2
    sample = inl[:5]
    assert all(e[i] <= mp.mpf(1e-14) * (w * w + h * h) for i in sample), "sample residuals"
    nx = []
    for i in sample:
        u = iI * mp.matrix([c[i, 0], c[i, 1], 1]); v = iJ * mp.matrix([c[i, 2], c[i, 3], 1])
        nx.append([float(u[0] / u[2]), float(u[1] / u[2]), float(v[0] / v[2]), float(v[1] / v[2])])
    audit_model(np.array(E.tolist(), dtype=np.float64), np.array(nx), 1e-7)
    del scale
    return "valid"


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_audit_port(port_all, name):
    corr, K, _, _ = scene(name)
    it, prec, wh = _params(name)
    audit_e(port_all[name], corr, K, wh, prec)


def test_audit_rejects_wrong_results(port_all):
    """The audit is not vacuous: each corruption of a valid result is caught."""
    import copy
    name = "precision4_r60_n400"
    corr, K, _, _ = scene(name)
    it, prec, wh = _params(name)
    r = port_all[name]
    assert audit_e(r, corr, K, wh, prec) == "valid"
    bad = []
    x = copy.deepcopy(r); x["inliers"] = x["inliers"].copy(); x["inliers"][[3, -1]] = x["inliers"][[-1, 3]]; bad.append(x)   # order
    x = copy.deepcopy(r); out = sorted(set(range(len(corr))) - set(r["inliers"].tolist()))
    x["inliers"] = np.append(r["inliers"][:-1], out[0]); bad.append(x)                                                        # set
    x = copy.deepcopy(r); x["error_max"] = float(r["error_max"]) * 1.001; bad.append(x)
    x = copy.deepcopy(r); x["min_nfa"] = float(r["min_nfa"]) + 0.01; bad.append(x)
    x = copy.deepcopy(r); x["E"] = np.asarray(r["E"]).T.copy(); bad.append(x)                                                 # E^T
    x = copy.deepcopy(r); x["E"] = np.asarray(r["E"]) + 1e-5 * np.linalg.norm(r["E"]); bad.append(x)
    for b in bad:
        with pytest.raises(AssertionError):
            audit_e(b, corr, K, wh, prec)
    with pytest.raises(AssertionError):     # a wrong K (transposed, as a K^-T for K^-1 mistake would give) or a wrong image size
        audit_e(r, corr, (K[0].T, K[1].T), wh, prec)
    with pytest.raises(AssertionError):
        audit_e(r, corr, K, (wh[0] * 2, wh[1]), prec)


def _sample_kinds():
    """Seeded normalised 5-samples: random, nearly coplanar, nearly pure rotation, nearly duplicated points (12 each)."""
    rng = np.random.default_rng(21)
    out = []
    for kind in ("random", "coplanar", "rotation", "duplicate"):
        for _ in range(12):
            R = _rot(*rng.uniform(-0.3, 0.3, 3))
            t = rng.normal(size=3)
            t = t / np.linalg.norm(t) * (1e-3 if kind == "rotation" else 1.0)
            out.append((kind, _normalised_sample(rng, R, t, noise=1e-3 if kind == "random" else 0.0, kind=kind)))
    return out


def test_real_root_count_on_action_matrices(port, record_property, capsys):
    """The number of real solutions (eigenvalues with imag() exactly 0, hence models) on the action matrix of every seeded 5-sample
    equals the count of a 50-digit eigen-solve of the same matrix, except where the decision is within rounding: a complex pair within
    |Im| / |lambda| < MARGIN of the real axis, or two eigenvalues closer than their first-order perturbation radii under a backward
    error of 10 eps |A|_F (the nearly pure rotations give action matrices with entries of 1e7 and eigenvalues of 0.3).  Those samples
    are listed (printed, and recorded as the property "near_double_excluded") and counted."""
    excluded, compared = [], 0
    for j, (kind, c) in enumerate(_sample_kinds()):
        A = port.action(c)
        got = port.eigen(A)
        nmod = len(port.fit5(c))
        if got is None:
            assert nmod == 0
            excluded.append((j, kind, "no convergence"))
            continue
        re, im = got
        assert nmod == int(np.sum(im == 0)), (j, kind)
        if not np.isfinite(A).all():
            excluded.append((j, kind, "non-finite action matrix"))
            continue
        ev, L, R = mp.eig(mp.matrix(A.tolist()), left=True, right=True)
        real = [abs(mp.im(e)) <= mp.mpf(10) ** -40 * max(abs(e), 1) for e in ev]
        ratios = [float(abs(mp.im(e)) / abs(e)) for e, r in zip(ev, real) if not r]
        if ratios and min(ratios) < MARGIN:
            excluded.append((j, kind, "near double", min(ratios)))
            continue
        # first-order perturbation radius of each eigenvalue under a backward error of 10 eps |A|_F (its condition number times
        # that): where two radii overlap, rounding alone can turn two real roots into a complex pair or back
        nA = mp.mpf(float(np.linalg.norm(A)))
        rad = []
        for q in range(10):
            lq = L[q, :]; rq = R[:, q]
            kap = mp.norm(lq) * mp.norm(rq) / abs(sum(lq[0, t] * rq[t, 0] for t in range(10)))
            rad.append(10 * kap * mp.mpf(2) ** -52 * nA)   # double epsilon
        close = [(a, b) for a in range(10) for b in range(a + 1, 10) if abs(ev[a] - ev[b]) <= rad[a] + rad[b]]
        if close:
            excluded.append((j, kind, "ill-conditioned", float(max(rad))))
            continue
        compared += 1
        assert int(np.sum(im == 0)) == sum(real), (j, kind, im, sum(real))
    record_property("near_double_excluded", repr(excluded))
    with capsys.disabled():
        print(f"\nreal-root count: {compared} action matrices compared, {len(excluded)} excluded: {excluded}")
    assert compared >= 36 and all(x[1] == "rotation" for x in excluded if x[2] == "ill-conditioned"), excluded


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import alicevision_b200 as av
    return av.Context(0)


def _same(got: dict, want: dict, what: str):
    assert got["valid"] == bool(want["valid"]), what
    assert np.array_equal(got["inliers"], np.asarray(want["inliers"], np.uint32)), what
    assert got["iterations"] == int(want["iterations"]), what
    assert np.array_equal(got["E"].ravel(), np.asarray(want["E"]).ravel()), (what, got["E"], want["E"])
    assert got["error_max"] == float(want["error_max"]), what
    a, c = got["min_nfa"], float(want["min_nfa"])
    assert a == c or abs(a - c) <= 1e-12 * max(abs(a), abs(c)), (what, a, c)   # device vs host log10
    tr = np.asarray(want["trace"])
    assert got["n_trace"] == int(want["n_trace"]) and np.array_equal(got["trace"], tr[:got["trace"].size]), what
    assert np.array_equal(got["mt_state_out"], np.asarray(want["mt_state_out"])), (what, "generator end state")


@pytest.mark.gpu
def test_gpu_equals_port_mixed_list(ctx, port, port_all):
    """Every scene in one call per (maxIteration, precision) group from one shared state, then all scenes in one call with per-pair
    states: the engine is the port bit for bit."""
    from alicevision_b200 import matching
    groups = {}
    for name, _, _, it, prec, _ in SCENES:
        groups.setdefault((it, prec), []).append(name)
    st = matching.mt19937_state(SEED)
    assert np.array_equal(st, port.mt_seed(SEED))
    for (it, prec), names in groups.items():
        sc = [scene(nm) for nm in names]
        res = ctx.acransac_essential_pairs([s[0] for s in sc], [(640, 480) + _params(nm)[2] for nm in names],
                                           [np.concatenate([s[1][0].ravel(), s[1][1].ravel()]) for s in sc], st, it, prec)
        for nm, r, sc_ in zip(names, res, sc):
            _same(r, port_all[nm], nm)
            audit_e(r, sc_[0], sc_[1], _params(nm)[2], prec)
    names = [s[0] for s in SCENES if s[3] == 3000 and s[4] == np.inf]
    states = np.stack([port.mt_seed(100 + k) for k in range(len(names))])
    sc = [scene(nm) for nm in names]
    res = ctx.acransac_essential_pairs([s[0] for s in sc], [(640, 480) + _params(nm)[2] for nm in names],
                                       [np.concatenate([s[1][0].ravel(), s[1][1].ravel()]) for s in sc], states, 3000, np.inf)
    for k, (nm, r) in enumerate(zip(names, res)):
        want = port.estimate(sc[k][0], sc[k][1], _params(nm)[2], states[k], 3000, np.inf)
        _same(r, want, f"{nm} per-pair state")
        audit_e(r, sc[k][0], sc[k][1], _params(nm)[2], np.inf)
    st_ = ctx.acransac_last_stats()
    assert st_["launches"] == 1 and st_["models_evaluated"] >= st_["models_exact"]


@pytest.mark.gpu
def test_gpu_independent_of_skip(ctx, port_all):
    from alicevision_b200 import matching
    names = ["r50_n300", "r20_n400", "r90_n200"]
    sc = [scene(nm) for nm in names]
    args = ([s[0] for s in sc], [(640, 480, 640, 480)] * 3, [np.concatenate([s[1][0].ravel(), s[1][1].ravel()]) for s in sc],
            matching.mt19937_state(SEED), 5000, np.inf)
    ctx.set_acransac_skip(False)
    try:
        res = ctx.acransac_essential_pairs(*args)
    finally:
        ctx.set_acransac_skip(True)
    for nm, r in zip(names, res):
        _same(r, port_all[nm], nm)


@pytest.mark.gpu
def test_gpu_bad_arguments(ctx):
    from alicevision_b200 import matching
    from alicevision_b200.matching import B200MatchError
    corr, K, _, _ = scene("r90_n200")
    Kp = np.concatenate([K[0].ravel(), K[1].ravel()])
    st = matching.mt19937_state(SEED)
    ctx.acransac_essential_pairs([corr], [(640, 480, 640, 480)], [Kp], st, 10)
    for bad in (np.zeros(18), np.where(np.arange(18) == 0, np.nan, Kp), np.where(np.arange(18) == 9, np.inf, Kp)):
        with pytest.raises(B200MatchError):
            ctx.acransac_essential_pairs([corr], [(640, 480, 640, 480)], [bad], st, 10)
    with pytest.raises(B200MatchError):
        ctx.acransac_essential_pairs([corr], [(0, 480, 640, 480)], [Kp], st, 10)
    with pytest.raises(B200MatchError):
        ctx.acransac_essential_pairs([corr], [(640, 480, 640, 480)], [Kp], st, 10, precision=0.0)
