"""K10 fundamental-matrix-with-distortion policy (b200m_acransac_fundamental_distortion_pairs,
GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel>).

CPU: the oracle's "ref" build (the reference's ACRANSAC, sampler and NFA compiled verbatim around the restated F10 kernel) equals
the port bit for bit, generator end state included, live or from tests/golden/reference_acransac_f10.npz; the 10-point solver
reproduces the reference's two known answers and is audited against an exact (mpmath) reference; every result is audited from
its inputs alone.
GPU (tests/test_distortion_filter.py): the engine equals the port.
"""
from __future__ import annotations

import zlib

import numpy as np
import pytest

mp = pytest.importorskip("mpmath")

import oracle  # noqa: E402
from oracle import acransac_f10  # noqa: E402

SEED = 5489
WH = (640, 480, 640, 480)


def _rot(a: float, b: float, c: float) -> np.ndarray:
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def distort(u: np.ndarray, lam: float, wh) -> np.ndarray:
    """Division-model distortion about the image centre, in the preconditioned units s = 1 / sqrt(w h): the distorted d satisfies
    u - c = (d - c) / (1 + lam |s (d - c)|^2) (lam < 0: barrel)."""
    w, h = wh
    s, c = 1.0 / np.sqrt(w * h), np.array([w / 2, h / 2])
    du = (u - c) * s
    d = du.copy()
    for _ in range(200):
        d = du * (1 + lam * np.sum(d * d, axis=1, keepdims=True))
    return d / s + c


def f10_scene(n: int, inlier_ratio: float, seed: int, noise: float = 0.3, translation=(0.5, 0.02, 0.05), rot=(0.0, 0.0, 0.0),
              lam=(-0.2, -0.2), wh=(640, 480), dup: int = 0):
    """Pixels (n x 4) of a planar pair: random 3-D points through K [I | 0] and K [R | t], distorted by the division model (lam_I,
    lam_J), Gaussian noise; outliers uniform in the image; `dup` correspondences repeated (degenerate samples)."""
    rng = np.random.default_rng(seed)
    K = np.array([[600.0, 0, wh[0] / 2], [0, 600.0, wh[1] / 2], [0, 0, 1]])
    X = rng.uniform(-1.5, 1.5, (n, 3)) + [0, 0, 6]
    R, t = _rot(*rot), np.asarray(translation, np.float64)
    xI = (K @ X.T).T
    xJ = (K @ ((R @ X.T).T + t).T).T
    uI, uJ = xI[:, :2] / xI[:, 2:], xJ[:, :2] / xJ[:, 2:]
    corr = np.concatenate([distort(uI, lam[0], wh), distort(uJ, lam[1], wh)], axis=1) + rng.normal(0, noise, (n, 4))
    n_out = n - int(round(inlier_ratio * n))
    out = rng.permutation(n)[:n_out]
    corr[out] = rng.uniform(0, 1, (n_out, 4)) * [wh[0], wh[1], wh[0], wh[1]]
    if dup:
        corr[n - dup:] = corr[0]
    return corr


# name, n, inlier ratio, maxIteration, precision (ACRANSAC's argument), scene kwargs
SCENES = [
    ("translation_r80_n200", 200, 0.8, 2000, np.inf, {"noise": 0.0, "lam": (0.0, 0.0)}),
    ("rotating_r80_n200", 200, 0.8, 2000, np.inf, {"rot": (0.05, 0.2, 0.03), "translation": (0.4, 0.1, 0.1)}),
    ("l0_r70_n250", 250, 0.7, 2000, np.inf, {"lam": (0.0, 0.0)}),
    ("barrel_r70_n250", 250, 0.7, 2000, np.inf, {"lam": (-0.6, -0.4)}),
    ("outliers_n150", 150, 0.0, 500, np.inf, {}),
    ("n10", 10, 1.0, 100, np.inf, {}),
    ("n11", 11, 1.0, 100, np.inf, {}),
    ("n12", 12, 1.0, 100, np.inf, {}),
    ("n13", 13, 1.0, 100, np.inf, {}),
    ("n14", 14, 1.0, 100, np.inf, {}),
    ("n15", 15, 1.0, 100, np.inf, {}),
    ("precision4_r60_n300", 300, 0.6, 2000, 4.0, {}),
    ("precision_tiny_n200", 200, 0.6, 500, 1e-8, {}),
    ("max1_n100", 100, 0.8, 1, np.inf, {}),
    ("max9_n100", 100, 0.8, 9, np.inf, {}),
    ("max10_n100", 100, 0.8, 10, np.inf, {}),
    ("max11_n100", 100, 0.8, 11, np.inf, {}),
    ("dup_r80_n60", 60, 0.8, 500, np.inf, {"dup": 40}),
    ("n2000", 2000, 0.5, 400, np.inf, {}),
]


def scene(name):
    _, n, r, _, _, kw = next(s for s in SCENES if s[0] == name)
    return f10_scene(n, r, seed=zlib.crc32(name.encode()), **kw)


def params(name):
    return next((it, prec) for nm, _, _, it, prec, _ in SCENES if nm == name)


@pytest.fixture(scope="module")
def port():
    acransac_f10.build(ref=False) if not acransac_f10.available("port") else None
    return acransac_f10.AcransacF10Oracle("port")


@pytest.fixture(scope="module")
def port_all(port):
    st = port.mt_seed(SEED)
    return {name: port.estimate(scene(name), WH, st, *params(name)) for name, *_ in SCENES}


def reference(name):
    live = acransac_f10.available("ref")

    def compute():
        o = acransac_f10.AcransacF10Oracle("ref")
        r = o.estimate(scene(name), WH, o.mt_seed(SEED), *params(name))
        return tuple(r[k] for k in acransac_f10.FIELDS)
    return dict(zip(acransac_f10.FIELDS, acransac_f10.reference_output(f"acransac_f10_{name}", compute, live)))


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_oracle_ref_equals_port(port_all, name):
    """The port is the compiled reference's loop, 10-point sampler (shuffle for ranges 11..14, Floyd from 15) and NFA (10 models) bit
    for bit: inliers and their order, F, L, errorMax, minNFA, the `better` trace and the generator's end state."""
    want, got = reference(name), port_all[name]
    for k in acransac_f10.FIELDS:
        assert oracle._same(got[k], want[k]), (name, k)


def test_scenes_cover_both_outcomes(port_all, port):
    v = {k: bool(r["valid"]) for k, r in port_all.items()}
    assert v["translation_r80_n200"] and v["barrel_r70_n250"] and v["l0_r70_n250"] and v["n2000"]
    assert not v["n10"] and int(port_all["n10"]["iterations"]) == 0 and not v["precision_tiny_n200"]
    assert np.array_equal(port_all["n10"]["mt_state_out"], port.mt_seed(SEED))
    assert int(port_all["max1_n100"]["iterations"]) == 1


# ---------------------------------------------------------------------------------------------------------------- the solver
X8 = [1.425203022203948e-01, 1.802107961554276e-02, -2.467473080283717e-01, 1.134013928865132e-01, -2.165429045024671e-01,
      1.016561086554276e-01, -1.779508570620888e-01, -5.443423622532895e-02, -9.503401906866776e-02, -1.912260035464638e-01,
      4.285402960526316e-01, 8.614113255550987e-02, -3.182964124177631e-02, -1.139683291786595e-01, -8.882934570312501e-02,
      9.867373817845394e-02, 3.867745811060855e-01, 1.629066868832237e-02, 4.764409436677632e-01, -8.015930175781250e-02]
U8 = [1.470885587993421e-01, -3.716578433388158e-02, -3.384269955283717e-01, 3.505518863075658e-02, -2.903711258737665e-01,
      2.336130242598684e-02, -2.017722360711349e-01, -1.733409359580592e-01, -1.022310598273026e-01, -1.984814292506168e-01,
      4.136125745271382e-01, 5.560238486842106e-02, -4.780700683593750e-02, -1.279896786338405e-01, -1.000526829769737e-01,
      3.618122301603619e-02, 3.628858064350329e-01, -6.060566149259868e-03, 4.513226639597039e-01, -1.025031481291119e-01]
F8 = [[-5.751087019565978e+02, -4.158188692023641e+02, -3.933617847277337e+01, 5.623077923604983e+02, -1.155037417506222e+03,
       -3.603293875557833e+01, -5.277848487166921e-01, -9.666992599768776e-02, 1],
      [-2.199589063941379e+04, -2.847966717222817e+04, -1.568596434350923e+02, 2.668165615957419e+04, 3.794695160371831e+04,
       3.582097175710577e+02, -1.985243717996453e+03, 3.206256740219327e+03, 1],
      [-2.406164718504593e+02, 1.051858077445098e+03, 1.029257202497226e+02, -9.384606808289793e+02, -1.561769129182295e+00,
       -7.588146214289489e+00, -2.671999077624011e+01, 1.072299253095423e+00, 1],
      [4.773291645793250e+02, -7.340046095681545e+03, -7.622433073293142e+01, 7.353659444399805e+03, -7.228144265103590e+02,
       2.313924014459177e+01, -4.096068639840655e+02, 1.760210427160575e+02, 1],
      [-3.634107580978586e+00, -6.861915294293681e+01, -1.419442789733012e+00, 1.043103524635315e+02, -9.905128840695012e+01,
       -1.288978514515288e+01, -5.004364829690772e+00, 1.759690666207339e+01, 1],
      [3.845891112065496e+02, -3.376624483974341e+02, 1.058628706262809e+00, 4.567090509397883e+02, -1.782032107508239e+01,
       6.603245933354176e-01, -3.057044617411873e+01, -1.171693147510399e+01, 1],
      [9.173705728965071e-01, 6.566802897577452e+02, -9.150842187178472e+01, -6.985651797488533e+02, 6.389672979364663e+01,
       -2.813972637838619e+01, 1.224499375450345e+02, 2.273467046355762e+00, 1],
      [9.260243587671360e+00, 2.901973712182848e+01, -4.525967397412600e+00, 3.873064498047484e+00, -3.308114531934898e+01,
       -1.268705935682481e+01, 3.742963523739931e+00, 1.576531480674961e+01, 1]]
L8 = [[6.664890785418972e+02, 9.360374635703592e-01], [-1.401232955798790e+02, 1.190659194737138e+03],
      [5.478399615715365e+01, 1.277075963855622e+01], [-3.004792949356860e+01, 1.442424098845748e+02],
      [5.619131137084262e+00, 1.528997232119745e+01], [-1.359819306123174e+00, -3.194231629423156e+02],
      [-7.668121663596985e+00, -1.015843563423398e+01], [-8.478427431999348e+00, -4.469547181112368e+00]]
X2 = [-3.229677381013569e-01, 9.796846088610198e-02, -1.859613679584704e-01, -1.331652189555921e-02, 3.993208393297698e-01,
      -4.309213738692434e-02, 4.570184647409539e-01, 6.516200015419409e-02, -2.922935084292763e-02, -3.059326252184416e-01,
      -1.386923378392270e-01, -4.580717387952302e-02, -7.286097476356908e-02, 6.164560418379934e-02, 5.396587171052632e-02,
      9.743896484375000e-02, 4.628304893092105e-01, -1.323552021227385e-01, 4.939758300781250e-01, -4.290067973889802e-02]
U2 = [-4.438024018940173e-01, 3.003572162828947e-05, -2.212387888055099e-01, -1.264103939658717e-01, 3.731781327097040e-01,
      -6.214079204358552e-02, 4.439694053248355e-01, 3.183979235197369e-02, 2.125557026110198e-01, -1.950167364823191e-01,
      -1.560874216180099e-01, -7.848533228824013e-02, -7.585523103412829e-02, -1.291279039884868e-02, -1.167459909539474e-01,
      2.065792686060855e-02, 4.302636076274671e-01, -1.466708052785773e-01, 4.942827405427632e-01, -8.317700837787830e-02]
F2 = [[1.732473500041804e+02, 7.711017146713161e+00, 9.471075243833084e+00, -1.518330376101678e+01, 3.516937871974938e+02,
       1.097973146625093e+01, -1.046922253151639e-01, 6.610316585565101e-03, 1],
      [-1.716387900591730e+04, -3.791505579727971e+04, -4.981406222447205e+00, 6.621894661079650e+03, 4.767612634161247e+04,
       -1.134635374165869e+02, 1.131438262492466e+03, -1.429200024334792e+04, 1]]
L2 = [[-1.904715904949555e+02, 4.147643173367164e-01], [1.258548483732838e+01, -2.918230091342369e+03]]


def _is_approx(a, b, prec):
    """Eigen's isApprox: |a - b| <= prec min(|a|, |b|) in the Frobenius norm."""
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.linalg.norm(a - b) <= prec * min(np.linalg.norm(a), np.linalg.norm(b))


def _sample(X, U):
    return np.concatenate([np.reshape(X, (10, 2)), np.reshape(U, (10, 2))], axis=1)


def test_known_answer_8_solutions(port):
    """fundamental10PSolver_test.cpp's 8-solution case: every expected (F, L) is found, in any order, at the test's isApprox(1e-1),
    and each model solves the sample to 1e-4 relative to |a| |F| |b| in 50 digits (the worst, a model with entries of 3e4, measured
    3.3e-5)."""
    c = _sample(X8, U8)
    ms = port.fit10(c)
    assert len(ms) == 8
    for F, L in zip(F8, L8):
        assert any(_is_approx(F, m[0], 1e-1) and _is_approx(L, m[1], 1e-1) for m in ms)
    for m in ms:
        audit_solution(m, c, 1e-4)


def test_known_answer_2_solutions(port):
    """fundamental10PSolver_test.cpp's 2-solution case, in order, at isApprox(1e-1), each model solving the sample to 1e-5; the
    well-conditioned first model also matches at 1e-6."""
    c = _sample(X2, U2)
    ms = port.fit10(c)
    assert len(ms) == 2
    for (F, L), m in zip(zip(F2, L2), ms):
        assert _is_approx(F, m[0], 1e-1) and _is_approx(L, m[1], 1e-1)
        audit_solution(m, c, 1e-5)
    assert _is_approx(F2[0], ms[0][0], 1e-6) and _is_approx(L2[0], ms[0][1], 1e-6)


@pytest.fixture(autouse=True)
def _digits():
    with mp.workdps(50):
        yield


def _lift(x, y, l):
    return [mp.mpf(x), mp.mpf(y), 1 + mp.mpf(l) * (mp.mpf(x) ** 2 + mp.mpf(y) ** 2)]


def distorted_residual(F, L, c):
    """|[x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T| / (|a| |F| |b|), exact, for each row of c (x_I, y_I, x_J, y_J)."""
    Fm = mp.matrix(np.asarray(F, np.float64).tolist())
    nf = mp.sqrt(sum(Fm[i, j] ** 2 for i in range(3) for j in range(3)))
    out = []
    for x1, y1, x2, y2 in np.asarray(c, np.float64):
        a, b = _lift(x1, y1, L[0]), _lift(x2, y2, L[1])
        r = sum(a[i] * Fm[i, j] * b[j] for i in range(3) for j in range(3))
        out.append(abs(r) / (mp.sqrt(sum(v * v for v in a)) * nf * mp.sqrt(sum(v * v for v in b))))
    return out


def audit_solution(model, c, bound):
    F, L = model
    assert F[2, 2] == 1.0
    assert max(distorted_residual(F, L, c)) <= bound


def _noise_free_sample(rng, lam=(-0.3, 0.2)):
    """10 preconditioned-unit correspondences of a random rigid pair with division-model distortion (l1, l2), and its ground-truth
    solver matrix: [x_I, y_I, 1 + l1 r_I^2] G [x_J, y_J, 1 + l2 r_J^2]^T = 0 with G = ([t]x R)^T, normalised to G(2, 2) = 1."""
    R = _rot(*rng.uniform(-0.2, 0.2, 3))
    t = rng.normal(size=3)
    X = rng.uniform(-1, 1, (10, 3)) + [0, 0, 4]
    uI = X[:, :2] / X[:, 2:]
    Xc = (R @ X.T).T + t
    uJ = Xc[:, :2] / Xc[:, 2:]

    def dist(u, l):   # the distorted d with u = d / (1 + l |d|^2)
        d = u.copy()
        for _ in range(300):
            d = u * (1 + l * np.sum(d * d, axis=1, keepdims=True))
        return d
    c = np.concatenate([dist(uI, lam[0]), dist(uJ, lam[1])], axis=1)
    E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ R
    G = E.T
    return c, G / G[2, 2]


def test_solver_audit(port):
    """Every finite model of seeded noise-free samples has F(2, 2) = 1 and satisfies its 10 distorted constraints relative to
    |a| |F| |b| in 50 digits: to 1e-1 (the worst, a spurious root with l2 near 600 where the float64 Groebner-basis elimination is
    ill-conditioned, measured 1.9e-2) and to 1e-2 when |l1|, |l2| <= 10 (measured 6.8e-4); one of them is the ground truth (F
    relative error plus |L error| at most 1e-6; measured at most 3.9e-7)."""
    rng = np.random.default_rng(7)
    for _ in range(25):
        lam = tuple(rng.uniform(-0.5, 0.5, 2))
        c, G = _noise_free_sample(rng, lam)
        if not np.all(np.isfinite(c)) or np.abs(c).max() > 2:   # the distortion's fixed point diverged: no sample
            continue
        ms = port.fit10(c)
        assert 1 <= len(ms) <= 10
        finite = [m for m in ms if np.all(np.isfinite(m[0])) and np.all(np.isfinite(m[1]))]
        for m in finite:
            audit_solution(m, c, 1e-2 if np.abs(m[1]).max() <= 10 else 1e-1)
        assert min(np.linalg.norm(m[0] - G) / np.linalg.norm(G) + np.linalg.norm(m[1] - lam) for m in finite) <= 1e-6


def test_real_solution_count_against_mp(port, capsys):
    """The number of solutions equals the number of real eigenvalues of the solver's action matrix in a 50-digit eigen-solve, except
    where an eigenvalue's imaginary part is within 1e-6 of 0 relative to its modulus (the 100 eps cut on the solutions and the
    2 eps real/complex assembly rule decide those by rounding); those samples are counted and printed."""
    rng = np.random.default_rng(11)
    excluded = 0
    for _ in range(40):
        c = rng.uniform(-0.5, 0.5, (10, 4))
        ms, At = port.fit10(c, action=True)
        ev = mp.eig(mp.matrix(At.tolist()), left=False, right=False)
        grey = [e for e in ev if 1e-30 * max(1, abs(e)) < abs(mp.im(e)) <= 1e-6 * max(1, abs(e))]
        if grey:
            excluded += 1
            continue
        assert len(ms) == sum(1 for e in ev if mp.im(e) == 0 or abs(mp.im(e)) <= 1e-30 * max(1, abs(e))), c
    with capsys.disabled():
        print(f"\nreal-solution count: {excluded} of 40 samples excluded near the cut")
    assert excluded <= 4


# ---------------------------------------------------------------------------------------------------------------- result audit
def _norm(w, h):
    s = 1.0 / np.sqrt(w * h)
    return np.array([[s, 0, np.float32(-.5 * w) * s], [0, s, -.5 * h * s], [0, 0, 1.0]])


def audit_f10(r, corr, wh, precision=np.inf):
    """Checks a port or engine result from its inputs alone: N1, N2; every residual as the reference scores it (the point-to-line error
    of F x_I on the pixels, in normalised units); the inlier set and order (the k smallest, ties by index); errorMax; minNFA with
    sample size 10 and 10 models; and the model: F renormalised (N2^-T F N1^-1, F(2, 2) = 1) with the returned L satisfies the
    solver's distorted constraint exactly (1e-9 relative, recomputed in 50-digit arithmetic) on at least 10 correspondences, the 10
    equations that fix an F10 solution's 10 unknowns.  No step uses the code under test."""
    if not r["valid"]:
        return
    corr = np.asarray(corr, np.float64)
    n = corr.shape[0]
    N1, N2 = _norm(wh[0], wh[1]), _norm(wh[2], wh[3])
    s2 = N2[0, 0]
    F = np.asarray(r["F"], np.float64)
    xI = np.concatenate([corr[:, :2], np.ones((n, 1))], axis=1)
    xJ = np.concatenate([corr[:, 2:], np.ones((n, 1))], axis=1)
    Fn = np.linalg.inv(N2).T @ F @ np.linalg.inv(N1)          # the preconditioned model the loop scored
    pI, pJ = (N1 @ xI.T).T, (N2 @ xJ.T).T
    l = (Fn @ pI.T).T
    res = np.sum(l * pJ, axis=1) ** 2 / (l[:, 0] ** 2 + l[:, 1] ** 2)
    inl = np.asarray(r["inliers"], np.int64)
    k = inl.size
    assert 10 < k <= n and len(set(inl.tolist())) == k
    tol = 1e-6 * res[inl].max() + 1e-28
    assert np.all(np.diff(res[inl]) >= -tol), "inliers out of residual order"
    assert res[inl].max() <= np.delete(res, inl).min() + tol if k < n else True, "not the k smallest"
    em = np.sqrt(res[inl].max()) / s2
    assert abs(em - r["error_max"]) <= 1e-6 * max(em, 1e-9), ("errorMax", em, r["error_max"])
    # minNFA with sample size 10 and 10 models
    lg = lambda x: float(mp.log10(x))  # noqa: E731
    logc = lambda kk, nn: sum(lg(nn - i + 1) - lg(i) for i in range(1, min(kk, nn - kk) + 1)) if 0 < kk < nn else 0.0  # noqa: E731
    D, A = np.sqrt(wh[2] ** 2 + wh[3] ** 2), wh[2] * wh[3]
    la0 = np.log10(2 * D / A / s2)
    nfa = np.log10(10 * (n - 10)) + (la0 + np.log10(np.sqrt(res[inl].max()) + np.finfo(np.float32).eps)) * (k - 10) + logc(k, n) + logc(10, k)
    assert abs(nfa - r["min_nfa"]) <= 1e-4 * max(1, abs(nfa)), ("minNFA", nfa, r["min_nfa"])
    # the model: its 10 best correspondences under the solver's distorted constraint, and a fit of them
    Lr = np.asarray(r["L"], np.float64)
    a = np.concatenate([pI[:, :2], (1 + Lr[0] * np.sum(pI[:, :2] ** 2, axis=1))[:, None]], axis=1)
    b = np.concatenate([pJ[:, :2], (1 + Lr[1] * np.sum(pJ[:, :2] ** 2, axis=1))[:, None]], axis=1)
    G = Fn / Fn[2, 2]
    d = np.abs(np.einsum("ni,ij,nj->n", a, G, b)) / (np.linalg.norm(a, axis=1) * np.linalg.norm(G) * np.linalg.norm(b, axis=1))
    best = np.argsort(d, kind="stable")[:10]
    c10 = np.concatenate([pI[best, :2], pJ[best, :2]], axis=1)
    with mp.workdps(50):
        exact = max(distorted_residual(G, Lr, c10))
    assert exact <= 1e-9, ("the model's 10 best correspondences do not solve it", float(exact))


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_audit_port(port_all, name):
    audit_f10(port_all[name], scene(name), WH, params(name)[1])


def test_audit_rejects_wrong_results(port_all):
    r = port_all["barrel_r70_n250"]
    corr = scene("barrel_r70_n250")
    audit_f10(r, corr, WH)
    bad = [dict(r, F=r["F"].T.copy()),                                     # the "fixed" convention
           dict(r, L=r["L"][::-1].copy()),                                 # l1 and l2 swapped
           dict(r, F=r["F"] * (1 + 1e-4 * np.arange(9).reshape(3, 3))),    # a perturbed F
           dict(r, inliers=np.concatenate([r["inliers"][1:2], r["inliers"][:1], r["inliers"][2:]]))]
    for b in bad:
        with pytest.raises(AssertionError):
            audit_f10(b, corr, WH)
    with pytest.raises(AssertionError):                                    # the wrong image size
        audit_f10(r, corr, (800, 600, 800, 600))
