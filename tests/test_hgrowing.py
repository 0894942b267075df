"""The homography-growing filter (filterMatchesByHGrowing, featureMatching's `homography_growing`): the oracle's port against an
independent numpy restatement, an mpmath audit of the port's results, the stage rules of robustModelEstimation_HGrowing, and on the GPU
the engine (K12) against the port."""
from __future__ import annotations

import numpy as np
import pytest

from alicevision_b200 import matching
from oracle import hgrowing

DEF = hgrowing.DEFAULT_PARAM


def _port():
    return hgrowing.HGrowingOracle()


# ------------------------------------------------------------------------------------------------ scenes
def _plane_points(rng, H, k, noise, box=2000.0):
    """k matches on the plane H, each with a scale and orientation consistent with H's local affinity at the point."""
    x = rng.uniform(0, box, (k, 2))
    X = np.c_[x, np.ones(k)] @ H.T
    y = X[:, :2] / X[:, 2:] + rng.normal(0, noise, (k, 2))
    sI = rng.uniform(1.5, 8, k)
    oI = rng.uniform(-np.pi, np.pi, k)
    rows = np.zeros((k, 8))
    for i in range(k):
        w = X[i, 2]
        A = (H[:2, :2] * w - np.outer(X[i, :2], H[2, :2])) / w ** 2
        F = A @ (sI[i] * np.array([[np.cos(oI[i]), -np.sin(oI[i])], [np.sin(oI[i]), np.cos(oI[i])]]))
        rows[i] = [x[i, 0], x[i, 1], sI[i], oI[i], y[i, 0], y[i, 1], np.sqrt(abs(np.linalg.det(F))),
                   np.arctan2(F[1, 0] - F[0, 1], F[0, 0] + F[1, 1])]
    return rows


def _random_h(rng, persp=1e-4):
    th, s = rng.uniform(-0.3, 0.3), rng.uniform(0.8, 1.2)
    return np.array([[s * np.cos(th), -s * np.sin(th), rng.uniform(-200, 200)], [s * np.sin(th), s * np.cos(th), rng.uniform(-200, 200)],
                     [rng.uniform(-persp, persp), rng.uniform(-persp, persp), 1.0]])


def scene(n, planes=2, outliers=0.3, seed=0, noise=0.3):
    """n putatives: `planes` planes sharing the inliers, a fraction of outliers, shuffled."""
    rng = np.random.default_rng(seed)
    n_out = int(round(n * outliers))
    n_in = n - n_out
    parts = [np.zeros((0, 8))]
    for p in range(planes):
        parts.append(_plane_points(rng, _random_h(rng), n_in // planes + (1 if p < n_in % planes else 0), noise))
    if n_out:
        parts.append(np.c_[rng.uniform(0, 2000, (n_out, 2)), rng.uniform(1.5, 8, n_out), rng.uniform(-np.pi, np.pi, n_out),
                           rng.uniform(0, 2000, (n_out, 2)), rng.uniform(1.5, 8, n_out), rng.uniform(-np.pi, np.pi, n_out)])
    f = np.concatenate(parts).astype(np.float32)
    return f[rng.permutation(len(f))]


def special_scene(kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "identical":          # the two views are the same image: every grown transformation is the identity
        f = scene(200, 1, 0.0, seed, noise=0.0)
        f[:, 4:8] = f[:, 0:4]
        return f
    if kind == "collinear":          # one plane whose inliers all lie on a line, plus a generic plane
        f = scene(150, 1, 0.2, seed)
        g = _plane_points(rng, _random_h(rng), 80, 0.3)
        g[:, 1] = 0.5 * g[:, 0] + 100
        X = np.c_[g[:, :2], np.ones(len(g))] @ _random_h(np.random.default_rng(seed + 7)).T
        g[:, 4:6] = X[:, :2] / X[:, 2:]
        return np.concatenate([f, g.astype(np.float32)])[rng.permutation(230)]
    if kind == "duplicates":         # every match twice
        f = scene(120, 2, 0.2, seed)
        return np.repeat(f, 2, axis=0)
    if kind == "w0":                 # points mapped to the line at infinity of their plane (w = 0) among generic ones
        H = np.array([[1.0, 0.0, 10.0], [0.0, 1.0, -5.0], [1e-3, 0.0, 1.0]])
        f = _plane_points(rng, H, 150, 0.2, box=900.0)
        bad = f[:10].copy()
        bad[:, 0] = -1000.0          # 1e-3 * -1000 + 1 = 0
        return np.concatenate([f, bad]).astype(np.float32)[rng.permutation(160)]
    raise ValueError(kind)


GENERIC = [(n, pl, s) for n in (0, 5, 19, 20, 21, 200) for pl, s in ((1, 1), (2, 2), (3, 3))] + [(2000, 3, 4)]
SPECIAL = ["identical", "collinear", "duplicates", "w0"]


def all_scenes(big=False):
    out = {f"n{n}_p{pl}_s{s}": scene(n, pl, 0.3, s) for n, pl, s in GENERIC if big or n <= 200}
    out.update({k: special_scene(k) for k in SPECIAL})
    return out


# ------------------------------------------------------------------------------------------------ numpy restatement
def np_error(T, f):
    p = np.c_[f[:, 0:2].astype(np.float64), np.ones(len(f))] @ T.T
    with np.errstate(all="ignore"):
        d = f[:, 4:6].astype(np.float64) - p[:, :2] / p[:, 2:]
        return (d * d).sum(1)


def np_inliers(T, f, tol):
    with np.errstate(invalid="ignore"):
        return set(np.flatnonzero(np_error(T, f) < tol * tol).tolist())


def np_similarity(fi):
    def A(x, y, s, o):
        return np.array([[s * np.cos(o), -s * np.sin(o), x], [s * np.sin(o), s * np.cos(o), y], [0, 0, 1]])
    d = fi.astype(np.float64)
    return A(*d[4:8]) @ np.linalg.inv(A(*d[0:4]))


def np_affinity(f, ids):
    ids = sorted(ids)
    k = len(ids)
    M = np.zeros((2 * k, 6))
    b = np.zeros(2 * k)
    for r, i in enumerate(ids):
        M[r, 0:3] = [f[i, 0], f[i, 1], 1]
        M[r + k, 3:6] = [f[i, 0], f[i, 1], 1]
        b[r], b[r + k] = f[i, 4], f[i, 5]
    a = np.linalg.lstsq(M, b, rcond=6 * np.finfo(float).eps)[0]
    return np.array([a[0:3], a[3:6], [0, 0, 1]])


def np_center(pts):
    pts = pts.astype(np.float32)
    mean = pts.mean(0, dtype=np.float32)
    sd = np.sqrt(((pts - mean) ** 2).sum(0, dtype=np.float32) / np.float32(len(pts) - 1)).astype(np.float32)
    sd = np.maximum(sd, np.float32(0.1))
    return np.array([[1.0 / float(sd[0]), 0, float(-mean[0] / sd[0])], [0, 1.0 / float(sd[1]), float(-mean[1] / sd[1])], [0, 0, 1]])


def np_homography(f, ids):
    ids = sorted(ids)
    CI, CJ = np_center(f[ids][:, 0:2]), np_center(f[ids][:, 4:6])
    k = len(ids)
    A = np.zeros((2 * k, 9))
    for r, i in enumerate(ids):
        pI = CI @ [f[i, 0], f[i, 1], 1.0]
        pJ = CJ @ [f[i, 4], f[i, 5], 1.0]
        A[r, 0:3], A[r, 6:9] = pI, -pJ[0] * pI
        A[r + k, 3:6], A[r + k, 6:9] = pI, -pJ[1] * pI
    h = np.linalg.svd(A)[2][-1]
    H = np.linalg.inv(CJ) @ h.reshape(3, 3) @ CI
    return H / H[2, 2] if abs(H[2, 2]) > np.finfo(float).eps else H


def np_is_identity(T):
    I = np.eye(3)
    return bool(np.all(np.where(I == 1, np.abs(T - 1) <= np.minimum(np.abs(T), 1) * 1e-12, np.abs(T) <= 1e-12)))


def np_grow(f, seed, q):
    planar = set()
    T = np.eye(3)
    for s in range(q["nbRefiningIterations"]):
        if s == 0:
            T, tol = np_similarity(f[seed]), q["similarityTolerance"]
        elif s <= 4:
            T, tol = np_affinity(f, planar), q["affinityTolerance"]
        else:
            T, tol = np_homography(f, planar), q["homographyTolerance"]
        planar = np_inliers(T, f, tol)
        if len(planar) < q["minInliersToRefine"]:
            return False, planar, T
    return not np_is_identity(T), planar, T


def np_robust(T_params, f, tol, jac):
    """RefineHRobustCostFunctor residuals (and Jacobian) of column-major parameters over the rows of f."""
    t = 0.25
    ts2 = 2 * (tol / np.sqrt(-np.log(t * t))) ** 2
    H = T_params.reshape(3, 3).T
    x = np.c_[f[:, 0:2].astype(np.float64), np.ones(len(f))]
    p = x @ H.T
    uw, vw = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    ex, ey = f[:, 4] - uw, f[:, 5] - vw
    e2 = ex * ex + ey * ey
    e = np.where(e2 == 0, e2, np.sqrt(e2))
    E = np.exp(-(e * e) / ts2)
    r = -np.log(E + t) + np.log(1 + t)
    if not jac:
        return r, None
    k = np.where(e2 == 0, 0.0, 2 * E / (ts2 * (E + t)))
    J = np.zeros((len(f), 9))
    for c in range(3):
        xw = x[:, c] / p[:, 2]
        J[:, 3 * c] = -k * ex * xw
        J[:, 3 * c + 1] = -k * ey * xw
        J[:, 3 * c + 2] = k * (ex * uw + ey * vw) * xw
    return r, J


def np_refine(H, f, tol):
    """Ceres' Levenberg-Marquardt at its defaults (max_num_iterations 10), restated in numpy: (usable, H)."""
    x = H.T.reshape(9).copy()
    r, J = np_robust(x, f, tol, True)
    if not (np.all(np.isfinite(r)) and np.all(np.isfinite(J))):
        return False, H
    cost = 0.5 * r @ r
    scale = 1 / (1 + np.sqrt((J * J).sum(0)))
    if np.abs(J.T @ r).max() <= 1e-10:
        return True, H
    radius, factor, reuse, invalid, diag = 1e4, 2.0, False, 0, None
    for _ in range(10):
        Js = J * scale
        if not reuse:
            diag = np.clip((Js * Js).sum(0), 1e-6, 1e32)
        reuse = True
        M = Js.T @ Js + np.diag(diag / radius)
        g = Js.T @ r
        try:
            step = -np.linalg.solve(M, g)
            model = -((Js @ step) @ (r + Js @ step / 2))
            ok = np.all(np.isfinite(step)) and model > 0
        except np.linalg.LinAlgError:
            ok = False
        if not ok:
            invalid += 1
            if invalid >= 5:
                return False, H
            radius /= factor
            factor *= 2
            if radius < 1e-32:
                break
            continue
        invalid = 0
        xn = x + step * scale
        rn, _ = np_robust(xn, f, tol, False)
        cand = 0.5 * rn @ rn if np.all(np.isfinite(rn)) else np.finfo(float).max
        if np.linalg.norm(x - xn) <= (np.linalg.norm(x) + 1e-8) * 1e-8:
            break
        if abs(cost - cand) <= 1e-6 * cost:
            break
        rho = (cost - cand) / model
        if rho > 1e-3:
            x = xn
            r, J = np_robust(x, f, tol, True)
            if not (np.all(np.isfinite(r)) and np.all(np.isfinite(J))):
                return False, H
            cost = 0.5 * r @ r
            radius = min(radius / max(1 / 3, 1 - (2 * rho - 1) ** 3), 1e16)
            factor, reuse = 2.0, False
            if np.abs(J.T @ r).max() <= 1e-10:
                break
        else:
            radius /= factor
            factor *= 2
        if radius < 1e-32:
            break
    Hn = x.reshape(3, 3).T
    return True, Hn / Hn[2, 2] if abs(Hn[2, 2]) > np.finfo(float).eps else Hn


def np_filter(f, q=None):
    """filterMatchesByHGrowing written as the reference's loops, with Python sets and numpy fits."""
    q = dict(DEF, **(q or {}))
    rem = list(range(len(f)))
    Hs, sets, trace = [], [], []
    for _ in range(q["maxNbHomographies"]):
        fr = f[rem]
        used, best, best_H, best_seed = set(), set(), None, -1
        for i in range(len(rem)):
            if i in used:
                continue
            ok, planar, T = np_grow(fr, i, q)
            if not ok:
                continue
            used |= planar
            if len(planar) > len(best):
                best, best_H, best_seed = planar, T, i
        if best_seed < 0:
            trace.append((-1, 0, 0))
            break
        before = len(best)
        ok, H = np_refine(best_H, fr[sorted(best)], q["homographyTolerance"])
        if ok:
            best = np_inliers(H, fr, q["homographyTolerance"])
        else:
            H = best_H
        trace.append((best_seed, before, len(best)))
        if len(best) < q["minNbMatchesPerH"]:
            break
        Hs.append(H)
        sets.append([rem[i] for i in sorted(best)])
        rem = [r for i, r in enumerate(rem) if i not in best]
        if len(rem) < q["minNbMatchesPerH"]:
            break
    return Hs, sets, trace


def _near_tolerance(f, ids, Hs, tol):
    """Whether any of the matches ids lies within 1e-9 relative of the tolerance under any of the homographies."""
    for H in Hs:
        e = np_error(np.asarray(H, np.float64), f[list(ids)])
        if np.any(np.abs(e - tol * tol) <= 1e-9 * tol * tol):
            return True
    return False


def _split(r):
    b = np.concatenate([[0], np.cumsum(r["counts"])]).astype(int)
    return [r["inliers"][b[k]:b[k + 1]].tolist() for k in range(len(r["counts"]))]


# ------------------------------------------------------------------------------------------------ CPU: port vs numpy
@pytest.mark.parametrize("name", list(all_scenes(big=True)))
def test_port_matches_numpy_restatement(name):
    f = all_scenes(big=True)[name]
    r = _port().filter(f)
    Hs, sets, trace = np_filter(f)
    got = _split(r)
    if name == "identical":
        # isIdentity(1e-12) on a pixel-scale homography fitted to identical views is decided by rounding: any homography either side
        # stores is the identity to 1e-9
        for H in list(r["H"]) + Hs:
            np.testing.assert_allclose(H, np.eye(3), atol=1e-9)
        return
    if name.startswith("n"):   # generic scenes: no match lies at a tolerance, so the counts must agree
        assert len(got) == len(sets), (name, r["trace"], trace)
    else:
        assert len(got) == len(sets) or _near_tolerance(f, range(len(f)), list(r["H"]) + Hs, DEF["homographyTolerance"]), (name, r["trace"], trace)
    for k, (a, b) in enumerate(zip(got, sets)):
        diff = set(a) ^ set(b)
        if diff:
            # only matches at the tolerance may differ; the generic scenes have none
            assert not name.startswith("n"), (name, k, sorted(diff))
            assert _near_tolerance(f, diff, [r["H"][k], Hs[k]], DEF["homographyTolerance"]), (name, k, sorted(diff))
            break
        np.testing.assert_allclose(r["H"][k], Hs[k], rtol=1e-6, atol=1e-9)


def test_scenes_have_structure():
    """The generic scenes exercise the loop: several homographies on the multi-plane scenes, none on the tiny ones."""
    p = _port()
    assert len(p.filter(scene(2000, 3, 0.3, 4))["counts"]) == 3
    assert len(p.filter(scene(200, 2, 0.3, 2))["counts"]) >= 1
    for n in (0, 5, 19):
        assert len(p.filter(scene(n, 1, 0.3, 1))["counts"]) == 0
    for H in p.filter(special_scene("identical"))["H"]:
        np.testing.assert_allclose(H, np.eye(3), atol=1e-9)


def test_exp_log_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 200
    p = _port()
    rng = np.random.default_rng(3)
    for x in np.concatenate([-rng.uniform(0, 50, 2000), [0.0, -1e-300, -700.0]]):
        want = float(mpmath.exp(mpmath.mpf(float(x))))
        assert abs(p.lib.hg_exp(float(x)) - want) <= 4 * np.spacing(want)
    for y in np.concatenate([rng.uniform(0.25, 1.25, 2000), [1.0, 0.0625, 1.25, 1e-300, 1e300]]):
        want = float(mpmath.log(mpmath.mpf(float(y))))
        assert abs(p.lib.hg_log(float(y)) - want) <= 4 * np.spacing(abs(want)) + (0 if want else 1e-300)


# ------------------------------------------------------------------------------------------------ CPU: mpmath audit of the port
def _mp_error(H, fr):
    import mpmath
    x, y = mpmath.mpf(float(fr[0])), mpmath.mpf(float(fr[1]))
    Hm = [[mpmath.mpf(float(v)) for v in row] for row in np.asarray(H)]
    w = Hm[2][0] * x + Hm[2][1] * y + Hm[2][2]
    if w == 0:
        return mpmath.inf
    u = (Hm[0][0] * x + Hm[0][1] * y + Hm[0][2]) / w
    v = (Hm[1][0] * x + Hm[1][1] * y + Hm[1][2]) / w
    return (mpmath.mpf(float(fr[4])) - u) ** 2 + (mpmath.mpf(float(fr[5])) - v) ** 2


def _mp_cost(H, f, tol):
    import mpmath
    t = mpmath.mpf(0.25)
    ts2 = 2 * (tol / mpmath.sqrt(-mpmath.log(t * t))) ** 2
    s = mpmath.mpf(0)
    for fr in f:
        e2 = _mp_error(H, fr)
        r = -mpmath.log(mpmath.exp(-e2 / ts2) + t) + mpmath.log(1 + t)
        s += r * r
    return s / 2


@pytest.mark.parametrize("name", ["n200_p1_s1", "n200_p2_s2", "n200_p3_s3", "collinear", "duplicates", "w0"])
def test_port_audit(name):
    """Every round of the port, against that round's remaining list: the chosen seed and best-set size are the reference's skip / union /
    first-maximum walk over the grown seeds; the refine of the best set never raises the robust cost (mpmath) and gives the stored H; the
    stored set is exactly the strict inlier set of the stored H (mpmath), up to matches at the tolerance."""
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 120
    f = all_scenes()[name]
    p = _port()
    r = p.filter(f)
    tol2 = DEF["homographyTolerance"] ** 2
    sets = _split(r)
    rem = list(range(len(f)))
    for rnd, tr in enumerate(r["trace"]):
        fr = f[rem]
        used, best, best_seed, grown = set(), 0, -1, {}
        for seed in range(len(rem)):
            if seed in used:
                continue
            T, cnt = p.grow_steps(fr, seed)
            if len(cnt) < DEF["nbRefiningIterations"] or cnt[-1] < DEF["minInliersToRefine"] or np_is_identity(T[-1]):
                continue
            grown[seed] = T[-1]
            used |= set(np.flatnonzero(np_error(T[-1], fr) < tol2).tolist())
            if cnt[-1] > best:
                best, best_seed = int(cnt[-1]), seed
        assert tuple(tr[:2]) == (best_seed, best), (rnd, tr, best_seed, best)
        if best_seed < 0:
            break
        ids = np.flatnonzero(np_error(grown[best_seed], fr) < tol2)
        ok, Hr = p.refine(fr[ids], grown[best_seed])
        if ok:
            assert _mp_cost(Hr, fr[ids], 5.0) <= _mp_cost(grown[best_seed], fr[ids], 5.0) * (1 + 1e-12), rnd
        if rnd >= len(sets):
            break
        H = Hr if ok else grown[best_seed]
        # the standalone refine folds the set's lanes from a compacted list, so it agrees to rounding, not bit for bit
        np.testing.assert_allclose(H, r["H"][rnd], rtol=1e-9, atol=1e-12)
        H = r["H"][rnd]
        inside = [j for j in rem if _mp_error(H, f[j]) < tol2]
        near = [j for j in rem if abs(float(_mp_error(H, f[j])) - tol2) <= 1e-9 * tol2]
        assert set(inside) ^ set(sets[rnd]) <= set(near), (rnd, sorted(set(inside) ^ set(sets[rnd])))
        assert sets[rnd] == [j for j in rem if j in set(sets[rnd])]          # in remaining-list order
        rem = [j for j in rem if j not in set(sets[rnd])]


# ------------------------------------------------------------------------------------------------ CPU: stage rules
class _PortContext:
    """The engine's hgrowing_pairs answered by the port, so that the stage logic of robustModelEstimation_HGrowing runs without a GPU."""

    def hgrowing_pairs(self, items, param=None):
        p = _port()
        return [p.filter(f, param) for f in items]


def _views(rng, n_views, n_feat, types=("sift",)):
    return {v: {t: np.c_[rng.uniform(0, 2000, (n_feat, 2)), rng.uniform(1.5, 8, n_feat), rng.uniform(-np.pi, np.pi, n_feat)].astype(np.float32)
                for t in types} for v in range(n_views)}


def _matches(i, j, ratio=None):
    m = np.zeros(len(i), matching.MATCH_DTYPE)
    m["i"], m["j"] = i, j
    m["ratio"] = ratio if ratio is not None else 0.5
    return m


def _plane_pair(seed, n=200, planes=2):
    """Two views whose first n features are the putatives of a multi-plane scene, matched i -> i."""
    f = scene(n, planes, 0.3, seed)
    return {0: {"sift": f[:, 0:4].copy()}, 1: {"sift": f[:, 4:8].copy()}}, _matches(np.arange(n), np.arange(n))


def test_stage_rules_cpu():
    rng = np.random.default_rng(5)
    views, m = _plane_pair(2)
    views[2] = {"sift": views[1]["sift"].copy(), "cctag3": np.zeros((4, 4), np.float32)}
    views[3] = {"sift": views[0]["sift"].copy(), "cctag3": np.zeros((4, 4), np.float32)}
    views[4] = {"sift": views[0]["sift"].copy(), "akaze": _views(rng, 1, 50)[0]["sift"]}
    putatives = {
        (0, 1): {"sift": m},
        (2, 3): {"sift": m},                                          # CCTag among the common types: dropped
        (0, 4): {"sift": _matches(np.arange(30), rng.permutation(30))},   # nothing survives: an empty list, still kept
        (1, 4): {"akaze": _matches(np.arange(3), np.arange(3))},      # akaze is not common (view 1 has none): nothing processed
        (0, 3): {"sift": m[:0]},                                      # an empty putative list: processed, empty, kept
    }
    out, hs = matching.robustModelEstimation_HGrowing(putatives, views, ctx=_PortContext())
    want_out, want_hs = hgrowing.stage(putatives, views)
    assert set(out) == set(want_out) == {(0, 1), (0, 4), (0, 3)}
    assert len(out[(0, 4)]["sift"]) == 0 and len(out[(0, 3)]["sift"]) == 0 and hs[(0, 4)]["sift"] == []
    assert len(out[(0, 1)]["sift"]) > 0
    for p in out:
        for t in out[p]:
            assert np.array_equal(out[p][t], want_out[p][t])
            assert len(hs[p][t]) == len(want_hs[p][t])
    # guidedMatching: the kept pairs get an empty map
    g_out, g_hs = matching.robustModelEstimation_HGrowing(putatives, views, guidedMatching=True, ctx=_PortContext())
    assert set(g_out) == set(out) and all(v == {} for v in g_out.values())
    assert len(g_hs[(0, 1)]["sift"]) == len(hs[(0, 1)]["sift"])
    # identical views give nothing
    f = special_scene("identical")
    same = {0: {"sift": f[:, 0:4].copy()}, 1: {"sift": f[:, 4:8].copy()}}
    o, h = matching.robustModelEstimation_HGrowing({(0, 1): {"sift": _matches(np.arange(len(f)), np.arange(len(f)))}}, same, ctx=_PortContext())
    assert (0, 1) in o
    for H, _ in h[(0, 1)]["sift"]:   # nothing, or the identity up to rounding (see test_port_matches_numpy_restatement)
        np.testing.assert_allclose(H, np.eye(3), atol=1e-9)


def test_filter_uses_caller_order_cpu():
    """The putatives are walked in the caller's order: reversing the list changes the seeds, and the outputs are in that order."""
    views, m = _plane_pair(3)
    hm, inl = matching.filterMatchesByHGrowing(views[0]["sift"], views[1]["sift"], m, ctx=_PortContext())
    assert len(hm) >= 1 and sum(len(x[1]) for x in hm) == len(inl)
    hm2, inl2 = matching.filterMatchesByHGrowing(views[0]["sift"], views[1]["sift"], m[::-1].copy(), ctx=_PortContext())
    assert len(hm2) >= 1
    for H, mm in hm2:
        assert np.all(np.diff(mm["i"].astype(np.int64)) < 0)   # each stored set keeps the (reversed) putative order


def _reference_src():
    import oracle
    src = oracle.reference_src()
    if src is None:
        pytest.skip("needs the AliceVision source tree")
    return src


def test_hgrowing_filter_patch_applies(tmp_path):
    """aliceVision_b200_homographyGrowingFilter.patch applies after the existing chain (aliceVision_b200.patch, _geometricFilter,
    _homographyFilter, _sphericalFilter) to copies of the reference files, and routes HOMOGRAPHY_GROWING through the batch with the
    reference's loop as the fallback."""
    import os
    import re
    import shutil
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    patches = [os.path.join(root, "integration", "patches", f"aliceVision_b200{s}.patch")
               for s in ("", "_geometricFilter", "_homographyFilter", "_sphericalFilter", "_homographyGrowingFilter")]
    files = sorted({m for p in patches for m in re.findall(r"^\+\+\+ b/(\S+)", open(p).read(), re.M)})
    for f in files:
        dst = tmp_path / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copy(os.path.join(os.path.dirname(src), f), dst)
    for p in patches:
        r = subprocess.run(["patch", "-p1", "-s", "-i", p], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, (p, r.stdout + r.stderr)
    text = (tmp_path / "src" / "software" / "pipeline" / "main_featureMatching.cpp").read_text()
    assert "GeometricFilterMatrix_HGrowing_Batch_b200 batch;" in text and "robustModelEstimationHGrowingOnB200(" in text
    case = text[text.index("case EGeometricFilterType::HOMOGRAPHY_GROWING:"):]
    assert case.index("robustModelEstimationHGrowingOnB200(") < case.index("GeometricFilterMatrix_HGrowing(geometricErrorMax, maxIteration)")
    assert text.index("sortMatches_byDistanceRatio(matches);") < text.index("robustModelEstimationHGrowingOnB200(geometricMatches")


def test_hgrowing_filter_adaptor_header_compiles():
    import os
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "alicevision_b200", "adaptor", "GeometricFilter_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(root, "oracle", "shim"), "-I", src,
                        "-I", os.path.join(root, "include"), "-I", os.path.join(root, "alicevision_b200", "adaptor"), hdr],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "GeometricFilterMatrix_HGrowing_Batch_b200" in open(hdr).read()


# ------------------------------------------------------------------------------------------------ GPU
def _engine_vs_port(ctx, items, param=None):
    p = _port()
    got = ctx.hgrowing_pairs(items, param)
    parted = 0
    for k, (f, g) in enumerate(zip(items, got)):
        w = p.filter(f, param)
        if not np.array_equal(g["trace"], w["trace"]):
            parted += 1
            continue
        assert np.array_equal(g["counts"], w["counts"]), k
        assert np.array_equal(g["inliers"], w["inliers"]), k
        assert g["H"].tobytes() == w["H"].tobytes(), k
    return got, parted


@pytest.mark.gpu
def test_engine_matches_port_on_every_scene():
    ctx = matching.default_context()
    scenes = all_scenes(big=True)
    _, parted = _engine_vs_port(ctx, list(scenes.values()))
    assert parted == 0
    st = ctx.hgrowing_last_stats()
    assert st["seeds_grown"] > 0 and st["rounds"] >= len(scenes)


@pytest.mark.gpu
def test_engine_large_item_and_mixed_list():
    ctx = matching.default_context()
    _, parted = _engine_vs_port(ctx, [scene(8192, 3, 0.4, 11)])
    assert parted == 0
    rng = np.random.default_rng(12)
    items = [scene(int(n), int(rng.integers(1, 4)), 0.3, 100 + k) for k, n in enumerate(rng.choice([0, 7, 20, 60, 150, 400], 500))]
    _, parted = _engine_vs_port(ctx, items)
    assert parted == 0


@pytest.mark.gpu
def test_window_independence():
    ctx = matching.Context()
    items = list(all_scenes().values()) + [scene(1500, 3, 0.3, 21)]
    try:
        ctx.set_hgrowing_window(1)
        a = ctx.hgrowing_pairs(items)
        sa = ctx.hgrowing_last_stats()
        ctx.set_hgrowing_window(7)
        b = ctx.hgrowing_pairs(items)
        ctx.set_hgrowing_window(256)
        c = ctx.hgrowing_pairs(items)
    finally:
        ctx.close() if hasattr(ctx, "close") else None
    for x, y, z in zip(a, b, c):
        for key in ("counts", "inliers", "trace"):
            assert np.array_equal(x[key], y[key]) and np.array_equal(x[key], z[key])
        assert x["H"].tobytes() == y["H"].tobytes() == z["H"].tobytes()
    p = _port()
    want = [p.filter(f) for f in items]
    assert sa["seeds_grown"] == sum(w["grown"] for w in want)      # window 1 grows exactly the reference's seeds
    assert sa["seeds_skipped"] == sum(w["skipped"] for w in want)


@pytest.mark.gpu
def test_end_to_end_from_matcher():
    """robustModelEstimation_HGrowing on putatives from ImageCollectionMatcherB200 over a two-plane scene, sorted by ratio, against the
    port's stage; every pair stores homographies."""
    from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, synth
    from alicevision_b200.matches_filtering import sortMatches_byDistanceRatio
    descs, feats = synth.planar_views(4, 1500, planes=2, seed=31, visible=0.8)
    pairs = synth.exhaustive_pairs(4)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200)
    got = m.Match({i: (descs[i], np.ascontiguousarray(feats[i][:, :2])) for i in range(4)}, pairs)
    views = {v: {"sift": feats[v]} for v in range(4)}
    putatives = {p: {"sift": sortMatches_byDistanceRatio(mm)} for p, mm in got.items()}
    out, hs = matching.robustModelEstimation_HGrowing(putatives, views)
    want_out, want_hs = hgrowing.stage(putatives, views)
    assert set(out) == set(want_out) == set(putatives) and len(putatives) == 6
    for p in out:
        assert np.array_equal(out[p]["sift"], want_out[p]["sift"])
        assert len(hs[p]["sift"]) == len(want_hs[p]["sift"]) >= 1, p
        for (H, mm), (H2, mm2) in zip(hs[p]["sift"], want_hs[p]["sift"]):
            assert H.tobytes() == H2.tobytes() and np.array_equal(mm, mm2)


@pytest.mark.gpu
def test_hgrowing_filter_cpp_adaptor():
    """The C++ batch adaptor (GeometricFilterMatrix_HGrowing_Batch_b200) against the port in one executable."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "hgrowing_filter_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "hgrowing_filter adaptor ok" in r.stdout


@pytest.mark.gpu
def test_input_validation():
    import ctypes as C
    ctx = matching.default_context()
    lib = ctx.lib
    f = scene(50, 1, 0.2, 1)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    nh = np.zeros(2, np.int32); H = np.zeros((2, 10, 9)); cnt = np.zeros((2, 10), np.int32); inl = np.zeros(100, np.int32)

    def call(offsets, feat, tols=(20.0, 10.0, 5.0), ints=(6, 8, 10, 20)):
        offsets = np.asarray(offsets, np.int64)
        return lib.b200m_hgrowing_pairs(ctx._h, C.c_int(len(offsets) - 1), ptr(offsets), ptr(feat), *[C.c_double(t) for t in tols],
                                        *[C.c_int(i) for i in ints], ptr(nh), ptr(H), ptr(cnt), ptr(inl), None, None)

    feat = np.ascontiguousarray(np.concatenate([f, f]))
    assert call([0, 50, 100], feat) == 0
    ms = ctx.hgrowing_last_stats()
    for bad in ([1, 50, 100], [0, 60, 50], [0, 50, 100 + (1 << 18) * 0 - 200]):
        assert call(bad, feat) != 0
    assert call([0, 50, 100], feat, tols=(np.nan, 10.0, 5.0)) != 0
    assert call([0, 50, 100], feat, tols=(20.0, -1.0, 5.0)) != 0
    assert call([0, 50, 100], feat, ints=(0, 8, 10, 20)) != 0
    assert call([0, 50, 100], feat, ints=(6, 8, 65, 20)) != 0
    assert call([0, 50, 100], feat, ints=(6, 65, 10, 20)) != 0
    assert call([0, 50, 100], feat, ints=(6, 8, 10, -1)) != 0
    big = np.zeros(((1 << 18) + 1, 8), np.float32)
    assert call([0, (1 << 18) + 1], big) != 0
    assert b"262144" in lib.b200m_last_error()
    assert ctx.hgrowing_last_stats() == ms                           # nothing ran
    with pytest.raises(matching.B200MatchError):
        ctx.set_hgrowing_window(0)
