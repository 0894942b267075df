"""K10: a-contrario RANSAC fundamental-matrix estimation (b200m_acransac_fundamental_pairs).

CPU: the engine's host sampler and the oracle's NFA tables against the compiled reference (randSample, makelogcombi), the oracle's
"ref" build (ACRansac.hpp compiled verbatim) against its "port" bit for bit on seeded two-view scenes, and the 7-point known answer.
GPU: the engine against the oracle on the same scenes, and its independence of the skip and of the batching.
"""
from __future__ import annotations

import numpy as np
import pytest

import alicevision_b200 as av
from alicevision_b200 import matching
from oracle import acransac as acr_oracle

WH = (1280, 960, 1200, 900)


def two_view_scene(n: int, inlier_ratio: float, seed: int, planar: bool = False, duplicates: int = 0, noise: float = 0.5) -> np.ndarray:
    """n x 4 correspondences (xI, yI, xJ, yJ) of a random rigid scene seen by two cameras; outliers are uniform in image J."""
    r = np.random.default_rng(seed)
    X = np.c_[r.uniform(-2, 2, (n, 2)), np.full(n, 6.0) if planar else r.uniform(4, 8, n)]
    K = np.array([[1000, 0, 640], [0, 1000, 480], [0, 0, 1.0]])
    a = r.uniform(0.1, 0.3)
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])

    def proj(R, t):
        p = (K @ (R @ X.T + t[:, None])).T
        return p[:, :2] / p[:, 2:]

    x1 = proj(np.eye(3), np.zeros(3)) + r.normal(0, noise, (n, 2))
    x2 = proj(Ry, np.array([-1.0, 0.1, 0.2])) + r.normal(0, noise, (n, 2))
    out = r.random(n) >= inlier_ratio
    x2[out] = r.uniform([0, 0], [WH[2], WH[3]], (int(out.sum()), 2))
    c = np.c_[x1, x2]
    if duplicates:
        c[r.choice(n, duplicates, replace=False)] = c[r.choice(n, duplicates, replace=False)]
    return c


# (name, n, inlier ratio, maxIteration, precision, scene options)
SCENES = [
    ("r10_n300", 300, 0.1, 50000, np.inf, {}),
    ("r50_n100", 100, 0.5, 50000, np.inf, {}),
    ("r90_n500", 500, 0.9, 50000, np.inf, {}),
    ("outliers_n200", 200, 0.0, 5000, np.inf, {}),
    ("n8", 8, 1.0, 50000, np.inf, {}),
    ("n9", 9, 0.9, 50000, np.inf, {}),
    ("n10", 10, 0.9, 50000, np.inf, {}),
    ("n11", 11, 0.9, 50000, np.inf, {}),
    ("n7", 7, 1.0, 50000, np.inf, {}),
    ("dup_n120", 120, 0.6, 50000, np.inf, {"duplicates": 30}),
    ("planar_n150", 150, 0.7, 50000, np.inf, {"planar": True}),
    ("precision4_n300", 300, 0.5, 50000, 4.0, {}),
    ("precision1_outliers", 200, 0.0, 50000, 1.0, {}),
    ("niter1", 100, 0.6, 1, np.inf, {}),
    ("niter9", 100, 0.6, 9, np.inf, {}),
    ("niter10", 100, 0.6, 10, np.inf, {}),
    ("niter11", 100, 0.6, 11, np.inf, {}),
    ("r70_n2000", 2000, 0.7, 50000, np.inf, {}),
    ("r60_n8192", 8192, 0.6, 1500, np.inf, {}),
]
SEED = 5489


def scene(name):
    for k, (nm, n, ratio, it, prec, opt) in enumerate(SCENES):
        if nm == name:
            return two_view_scene(n, ratio, 1000 + k, **opt), it, prec
    raise KeyError(name)


def reference(name):
    corr, it, prec = scene(name)
    live = acr_oracle.available("ref")

    def compute():
        ora = acr_oracle.AcransacOracle("ref")
        r = ora.estimate(corr, WH, ora.mt_seed(SEED), it, prec)
        return tuple(r[k] for k in acr_oracle.FIELDS)
    return dict(zip(acr_oracle.FIELDS, acr_oracle.reference_output(f"acransac_{name}", compute, live)))


@pytest.fixture(scope="module")
def port():
    return acr_oracle.AcransacOracle("port")


# ---------------------------------------------------------------------------------------------------------------- CPU
SEEDS = [0, 1, 42, 5489, 2 ** 32 - 1]


@pytest.mark.parametrize("seed", SEEDS)
def test_mt19937_seed(seed):
    """b200m_mt19937_seed equals std::mt19937(seed) (compiled in the oracle's "ref" build, or its stored words)."""
    got = matching.mt19937_state(seed)
    want = acr_oracle.reference_output(f"mt_seed_{seed}", lambda: acr_oracle.AcransacOracle("ref").mt_seed(seed), acr_oracle.available("ref"))
    assert np.array_equal(got, want)


@pytest.mark.parametrize("rng", [8, 9, 10, 11, 100, 8192])
@pytest.mark.parametrize("seed", [1, 42, 777])
def test_host_sampler_equals_randSample(rng, seed):
    """The engine's sampler (host debug hook) equals randSample<size_t>(g, 0, rng, 7): the samples in their order (the
    unordered_set iteration order on the Floyd path) and the generator state after each of 3000 draws."""
    st = matching.mt19937_state(seed)
    got, got_st = matching.debug_rand_sample(st, rng, 3000)
    if acr_oracle.available("ref"):
        want, want_st = acr_oracle.AcransacOracle("ref").rand_sample(st, rng, 3000, states=True)
        assert np.array_equal(got, want)
        assert np.array_equal(got_st, want_st)
    want = acr_oracle.reference_output(f"rand_sample_{rng}_{seed}",
                                       lambda: acr_oracle.AcransacOracle("ref").rand_sample(st, rng, 3000)[0], acr_oracle.available("ref"))
    assert np.array_equal(got, want)
    assert all(len(set(s)) == 7 and max(s) < rng for s in got.tolist())


@pytest.mark.parametrize("n", [8, 9, 10, 11, 100, 8192])
def test_logc_tables_equal_makelogcombi(port, n):
    """The float logc tables equal the compiled makelogcombi<float> bit for bit (this pins which log10 fills vec_log10)."""
    got = port.logc(n)
    want = acr_oracle.reference_output(f"logc_{n}", lambda: acr_oracle.AcransacOracle("ref").logc(n),
                                       acr_oracle.available("ref"))
    assert np.array_equal(got[0].view(np.uint32), np.asarray(want[0]).view(np.uint32))
    assert np.array_equal(got[1].view(np.uint32), np.asarray(want[1]).view(np.uint32))


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_oracle_ref_equals_port(port, name):
    """The restated loop equals the compiled ACRANSAC bit for bit: inliers and their order, NFA, F, errorMax, iterations, trace."""
    corr, it, prec = scene(name)
    got = port.estimate(corr, WH, port.mt_seed(SEED), it, prec)
    want = reference(name)
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), (name, k)


def test_scenes_cover_both_outcomes():
    """The scene list holds meaningful and meaningless pairs, and pairs that stop early."""
    v = {name: bool(reference(name)["valid"]) for name, *_ in SCENES}
    assert v["r90_n500"] and v["r50_n100"] and v["r70_n2000"]
    assert not v["outliers_n200"] and not v["n7"]
    assert int(reference("precision1_outliers")["iterations"]) == 50000 // 10 * 2 + 2   # early exit once iter > 2 * nIterReserve


def test_seven_point_known_answer(port):
    """multiview/relativePose/fundamentalKernel_test.cpp (Fundamental7PKernel_EasyCase): every model satisfies x2^T F x1 = 0
    on its 7 points and det F = 0."""
    x1 = np.array([[0, 0, 0, 1, 1, 1, 2], [0, 1, 2, 0, 1, 2, 0]], float)
    x2 = np.array([[0, 0, 0, 1, 1, 1, 2], [1, 2, 3, 1, 2, 3, 1]], float)
    Fs = port.fit7(np.c_[x1.T, x2.T])
    assert len(Fs) >= 1
    for F in Fs:
        F = F / np.linalg.norm(F)
        h1 = np.r_[x1, np.ones((1, 7))]; h2 = np.r_[x2, np.ones((1, 7))]
        assert np.abs(np.einsum("ij,ik,kj->j", h2, F, h1)).max() < 1e-8
        assert abs(np.linalg.det(F)) < 1e-8


# ---------------------------------------------------------------------------------------------------------------- GPU
def _tie_level(corr, F) -> np.ndarray:
    """Per correspondence: True where its point-to-line distance in image J under F is at rounding level (< 1e-7 px).  The 7
    points a model was fitted to lie on it up to rounding; their order among themselves follows the last bits of the model,
    which differ between the device and the host libm (acos, cos, pow in the cubic solver)."""
    F = np.asarray(F, np.float64).reshape(3, 3)
    h1 = np.c_[corr[:, :2], np.ones(len(corr))]; h2 = np.c_[corr[:, 2:], np.ones(len(corr))]
    l = h1 @ F.T
    return np.abs(np.sum(l * h2, 1)) / np.hypot(l[:, 0], l[:, 1]) < 1e-7


def _same(got: dict, want: dict, what: str, corr=None):
    assert got["valid"] == bool(want["valid"]), what
    gi, wi = got["inliers"], np.asarray(want["inliers"], np.uint32)
    if corr is not None and gi.size == wi.size and not np.array_equal(gi, wi):
        # the same list, except for an exchange of correspondences that both lie on the model up to rounding
        tie = _tie_level(corr, want["F"])
        diff = gi != wi
        assert np.array_equal(np.sort(gi), np.sort(wi)) and tie[gi[diff]].all() and tie[wi[diff]].all(), what
    else:
        assert np.array_equal(gi, wi), what
    assert got["iterations"] == int(want["iterations"]), what
    tr = np.asarray(want["trace"])
    assert got["n_trace"] == int(want.get("n_trace", tr.size)) and np.array_equal(got["trace"], tr[:got["trace"].size]), what
    if "trace_nfa" in want:
        assert np.array_equal(got["trace_nfa"], np.asarray(want["trace_nfa"])[:got["trace"].size]) or all(
            _rounding_level(a, b) for a, b in zip(got["trace_nfa"], want["trace_nfa"])), what
    for k in ("error_max", "min_nfa"):
        a, b = got[k], float(want[k])
        assert a == b or abs(a - b) <= 1e-9 * max(abs(a), abs(b)), (what, k, a, b)
    Fa, Fb = np.asarray(got["F"]).ravel(), np.asarray(want["F"]).ravel()
    if np.linalg.norm(Fb) == 0:
        assert np.linalg.norm(Fa) == 0, what
    else:
        Fa = Fa / np.linalg.norm(Fa); Fb = Fb / np.linalg.norm(Fb)
        assert min(np.linalg.norm(Fa - Fb), np.linalg.norm(Fa + Fb)) <= 1e-9, what


@pytest.fixture(scope="module")
def ctx():
    return av.Context(0)


@pytest.fixture(scope="module")
def gpu_all(ctx):
    """Every scene in one call per (maxIteration, precision) group."""
    out = {}
    groups = {}
    for name, _, _, it, prec, _ in SCENES:
        groups.setdefault((it, prec), []).append(name)
    for (it, prec), names in groups.items():
        res = ctx.acransac_fundamental_pairs([scene(nm)[0] for nm in names], [WH] * len(names), matching.mt19937_state(SEED), it, prec)
        out.update(zip(names, res))
    return out


def _consistent(got: dict, corr, what: str):
    """A result that holds in itself: distinct inliers, and every inlier within errorMax of its epipolar line under F."""
    inl = got["inliers"]
    assert len(set(inl.tolist())) == inl.size, what
    if got["valid"]:
        assert got["min_nfa"] < 0 and inl.size >= 8, what
        h1 = np.c_[corr[:, :2], np.ones(len(corr))]; h2 = np.c_[corr[:, 2:], np.ones(len(corr))]
        l = h1 @ np.asarray(got["F"]).T
        d = np.abs(np.sum(l * h2, 1)) / np.hypot(l[:, 0], l[:, 1])   # point-to-line distance in image J, pixels
        assert d[inl].max() <= got["error_max"] * (1 + 1e-6), what


def _rounding_level(new: float, prev: float) -> bool:
    return abs(new - prev) <= 1e-9 * max(1.0, abs(prev))


def _matches_oracle(got: dict, want: dict, what: str, corr) -> bool:
    """The engine against the oracle's restated loop (pinned to the compiled reference on the CPU).

    The strict `<` on minNFA accepts an improvement of one rounding unit, and such improvements happen: a 7-subset drawn again
    in another order gives the same model up to rounding, and its NFA may come out lower in the last bits.  Whether it does
    depends on the last bits of acos / cos / pow / log10, which differ between the device and glibc.  So the two `better` traces
    must agree event for event (iteration, and minNFA within 1e-9) up to the first difference; if there is one, the event where
    they part must be such a rounding-level improvement on the side that has it, and from there on the engine's result is checked
    for its outcome and for consistency in itself.  Without a fork every output must be equal.  Returns whether they forked."""
    gt, gn, wt, wn = got["trace"], got["trace_nfa"], np.asarray(want["trace"]), np.asarray(want["trace_nfa"])
    m = min(gt.size, wt.size)
    j = next((i for i in range(m) if gt[i] != wt[i] or not _rounding_level(gn[i], wn[i])), m)
    if j == m and (got["n_trace"] == want["n_trace"] or j == gt.size < got["n_trace"]):
        _same(got, want, what, corr)
        return False
    sides = []
    if j < gt.size and (j >= wt.size or gt[j] <= wt[j]):
        sides.append(("engine", gn))
    if j < wt.size and (j >= gt.size or wt[j] <= gt[j]):
        sides.append(("oracle", wn))
    assert sides, (what, "traces differ in length only", got["n_trace"], want["n_trace"])
    for side, nfa in sides:
        assert j > 0 and _rounding_level(nfa[j], nfa[j - 1]), (what, f"{side} trace parts at event {j} by more than rounding",
                                                                gt[:j + 2], gn[:j + 2], wt[:j + 2], wn[:j + 2])
    assert got["valid"] == bool(want["valid"]), what
    _consistent(got, corr, what)
    return True


@pytest.fixture(scope="module")
def port_all(port):
    """The oracle's restated loop on every scene, with the minNFA of each `better` event."""
    out = {}
    for name, *_ in SCENES:
        corr, it, prec = scene(name)
        out[name] = port.estimate(corr, WH, port.mt_seed(SEED), it, prec)
    return out


# Scenes where the engine and the oracle part at a `better` event by more than rounding: the planar scene (its 7-point systems have
# a 3-D null space, so every fitted model is set by rounding and the libm differences grow into different models from the first
# iterations on) and n9 (9 correspondences, 7 of them fitted exactly by every model).  They are checked for their outcome and for a
# result consistent in itself.
ILL_CONDITIONED = {"n9", "planar_n150"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s[0] for s in SCENES if s[0] not in ILL_CONDITIONED])
def test_gpu_equals_oracle(gpu_all, port_all, name):
    want = port_all[name]
    ref = reference(name)   # the port is the compiled reference's loop bit for bit (test_oracle_ref_equals_port)
    assert all(np.array_equal(np.asarray(want[k]), np.asarray(ref[k])) for k in acr_oracle.FIELDS), name
    _matches_oracle(gpu_all[name], want, name, scene(name)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ILL_CONDITIONED))
def test_gpu_ill_conditioned_scenes(gpu_all, name):
    got, want = gpu_all[name], reference(name)
    assert got["valid"] == bool(want["valid"]) and got["valid"], name
    _consistent(got, scene(name)[0], name)


@pytest.mark.gpu
def test_gpu_independent_of_skip_and_batching(ctx, gpu_all):
    """The same outputs with the certified skip disabled, and with the list given pair by pair."""
    names = ["r10_n300", "r50_n100", "dup_n120", "planar_n150", "n9", "r70_n2000"]
    st = matching.mt19937_state(SEED)
    ctx.set_acransac_skip(False)
    try:
        noskip = ctx.acransac_fundamental_pairs([scene(nm)[0] for nm in names], [WH] * len(names), st, 50000)
        stats = ctx.acransac_last_stats()
        assert stats["models_skipped"] == 0 and stats["models_exact"] == stats["models_evaluated"] > 0
    finally:
        ctx.set_acransac_skip(True)
    for nm, r in zip(names, noskip):
        _same(r, gpu_all[nm], nm + " (no skip)")
        assert np.array_equal(r["F"], gpu_all[nm]["F"]) and r["min_nfa"] == gpu_all[nm]["min_nfa"]
    for nm in names:
        one = ctx.acransac_fundamental_pairs([scene(nm)[0]], [WH], st, 50000)[0]
        assert np.array_equal(one["F"], gpu_all[nm]["F"]) and np.array_equal(one["inliers"], gpu_all[nm]["inliers"])
        assert one["iterations"] == gpu_all[nm]["iterations"] and one["min_nfa"] == gpu_all[nm]["min_nfa"]


@pytest.mark.gpu
def test_gpu_500_pairs_default_iterations(ctx, port):
    """A 500-pair list at maxIteration = 50000: overlapping and non-overlapping pairs and one above the shared-memory sort
    capacity; a sample of pairs matches the oracle."""
    r = np.random.default_rng(3)
    corrs = []
    for k in range(500):
        n = int(r.integers(20, 400)) if k != 250 else 1500
        ratio = 0.7 if k == 250 else 0.0 if k % 3 else float(r.uniform(0.3, 0.9))
        corrs.append(two_view_scene(n, ratio, 10_000 + k))
    st = matching.mt19937_state(SEED)
    res = ctx.acransac_fundamental_pairs(corrs, [WH] * 500, st, 50000)
    stats = ctx.acransac_last_stats()
    assert stats["models_skipped"] > 0
    assert sum(x["valid"] for x in res) >= 100 and res[250]["valid"]   # the pair sorted in global memory has a model
    for k in (0, 1, 3, 250, 499):
        want = port.estimate(corrs[k], WH, st, 50000)
        _matches_oracle(res[k], want, f"pair {k}", corrs[k])


@pytest.mark.gpu
def test_geometricEstimation_F_AC(ctx, port):
    corr, it, prec = scene("r50_n100")
    got = matching.geometricEstimation_F_AC(corr[:, :2], corr[:, 2:], WH[:2], WH[2:], SEED, it, prec, ctx=ctx)
    _matches_oracle(got, port.estimate(corr, WH, port.mt_seed(SEED), it, prec), "geometricEstimation_F_AC", corr)
