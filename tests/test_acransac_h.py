"""K10 for the homography: a-contrario RANSAC homography estimation (b200m_acransac_homography_pairs, the homography_matrix filter).

CPU: the engine's host sampler for sample size 4 and the oracle's NFA tables against the compiled reference (randSample,
makelogcombi), the oracle's "ref" build (ACRansac.hpp compiled verbatim) against its "port" bit for bit on seeded two-view scenes,
generator end states included, and the 4-point known answer.
GPU: the engine against the oracle on the same scenes; its independence of the skip, of the batching and of shared vs per-pair
generator states; the generator chain of the reference's single-threaded filter; a 500-pair list; argument checks.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import alicevision_b200 as av
from alicevision_b200 import matching
from oracle import acransac_h as acrh

WH = (1280, 960, 1200, 900)
K = np.array([[1000, 0, 640], [0, 1000, 480], [0, 0, 1.0]])


def _rot(a: float, b: float, c: float) -> np.ndarray:
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    Rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def h_scene(n: int, inlier_ratio: float, seed: int, kind: str = "plane", duplicates: int = 0, noise: float = 0.5) -> np.ndarray:
    """n x 4 correspondences (xI, yI, xJ, yJ) of a seeded two-view scene; outliers are uniform in image J.
    kind: "plane"      a tilted plane seen from two poses (one homography);
          "rotation"   a general 3-D scene under a pure rotation (one homography);
          "general"    a deep non-planar scene with translation (no homography explains it exactly);
          "two_planes" two planes of different orientation under translation (two homographies);
          "collinear"  every inlier on one 3-D line, seen from two poses (degenerate 4-point samples)."""
    r = np.random.default_rng(seed)
    u = r.uniform(-2, 2, (n, 2))
    R, t = _rot(r.uniform(-0.1, 0.1), r.uniform(0.1, 0.3), r.uniform(-0.1, 0.1)), np.array([-1.0, 0.1, 0.2])
    if kind == "plane":
        X = np.c_[u, 6.0 + 0.4 * u[:, 0] + 0.2 * u[:, 1]]
    elif kind == "rotation":
        X = np.c_[u, r.uniform(4, 8, n)]
        t = np.zeros(3)
    elif kind == "general":
        X = np.c_[u * 1.5, r.uniform(3, 10, n)]
        t = np.array([-1.5, 0.2, 0.3])
    elif kind == "two_planes":
        first = np.arange(n) < n // 2
        X = np.c_[u, np.where(first, 5.0 + 0.3 * u[:, 1], 8.0 - 0.6 * u[:, 0])]
    elif kind == "collinear":
        s = r.uniform(-2, 2, n)
        X = np.c_[s, 0.3 * s + 0.1, 6.0 + 0.2 * s]
    else:
        raise ValueError(kind)

    def proj(Rm, tv):
        p = (K @ (Rm @ X.T + tv[:, None])).T
        return p[:, :2] / p[:, 2:]

    x1 = proj(np.eye(3), np.zeros(3)) + r.normal(0, noise, (n, 2))
    x2 = proj(R, t) + r.normal(0, noise, (n, 2))
    out = r.random(n) >= inlier_ratio
    x2[out] = r.uniform([0, 0], [WH[2], WH[3]], (int(out.sum()), 2))
    c = np.c_[x1, x2]
    if duplicates:
        c[r.choice(n, duplicates, replace=False)] = c[r.choice(n, duplicates, replace=False)]
    return c


# (name, n, inlier ratio, maxIteration, precision, scene kind and options)
SCENES = [
    ("plane_r10_n300", 300, 0.1, 50000, np.inf, {}),
    ("plane_r50_n100", 100, 0.5, 50000, np.inf, {}),
    ("rot_r90_n500", 500, 0.9, 50000, np.inf, {"kind": "rotation"}),
    ("general_r80_n300", 300, 0.8, 50000, np.inf, {"kind": "general"}),
    ("two_planes_n400", 400, 0.8, 50000, np.inf, {"kind": "two_planes"}),
    ("outliers_n200", 200, 0.0, 5000, np.inf, {}),
    ("n3", 3, 1.0, 50000, np.inf, {}),
    ("n4", 4, 1.0, 50000, np.inf, {}),
    ("n5", 5, 1.0, 50000, np.inf, {}),
    ("n6", 6, 0.9, 50000, np.inf, {}),
    ("n7", 7, 0.9, 50000, np.inf, {}),
    ("dup_n120", 120, 0.6, 50000, np.inf, {"duplicates": 30}),
    ("collinear_n150", 150, 0.7, 50000, np.inf, {"kind": "collinear"}),
    ("precision4_n300", 300, 0.5, 50000, 4.0, {}),
    ("precision1_outliers", 200, 0.0, 50000, 1.0, {}),
    ("niter1", 100, 0.6, 1, np.inf, {}),
    ("niter9", 100, 0.6, 9, np.inf, {}),
    ("niter10", 100, 0.6, 10, np.inf, {}),
    ("niter11", 100, 0.6, 11, np.inf, {}),
    ("rot_r70_n2000", 2000, 0.7, 50000, np.inf, {"kind": "rotation"}),
    ("plane_r60_n8192", 8192, 0.6, 1500, np.inf, {}),
]
SEED = 5489
# degenerate samples (duplicated or collinear points) have a null space of dimension 2 or more, so their models are set by rounding
DEGENERATE = {"dup_n120", "collinear_n150"}


def scene(name):
    for k, (nm, n, ratio, it, prec, opt) in enumerate(SCENES):
        if nm == name:
            return h_scene(n, ratio, 2000 + k, **opt), it, prec
    raise KeyError(name)


def reference(name):
    corr, it, prec = scene(name)

    def compute():
        ora = acrh.AcransacHOracle("ref")
        r = ora.estimate(corr, WH, ora.mt_seed(SEED), it, prec)
        return tuple(r[k] for k in acrh.FIELDS)
    return dict(zip(acrh.FIELDS, acrh.reference_output(f"acransac_h_{name}", compute, acrh.available("ref"))))


@pytest.fixture(scope="module")
def port():
    return acrh.AcransacHOracle("port")


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("seed", [1, 42])
@pytest.mark.parametrize("rng", list(range(5, 41)) + [100, 8192, 1 << 20])
def test_host_sampler_k4_equals_randSample(rng, seed):
    """The engine's sampler (host debug hook) equals randSample<size_t>(g, 0, rng, 4): the samples in their order (std::shuffle
    for range 5, the unordered_set iteration order on the Floyd path otherwise) and the generator state after each draw."""
    st = matching.mt19937_state(seed)
    got, got_st = matching.debug_rand_sample(st, rng, 1000, sample_size=4)
    if acrh.available("ref"):
        want, want_st = acrh.AcransacHOracle("ref").rand_sample(st, 4, rng, 1000, states=True)
        assert np.array_equal(got, want)
        assert np.array_equal(got_st, want_st)
    want = acrh.reference_output(f"rand_sample4_{rng}_{seed}", lambda: acrh.AcransacHOracle("ref").rand_sample(st, 4, rng, 1000)[0][:100],
                                 acrh.available("ref"))
    assert np.array_equal(got[:100], want)
    assert all(len(set(s)) == 4 and max(s) < rng for s in got.tolist())


@pytest.mark.parametrize("rng", [8, 10, 11, 100])
def test_host_sampler_k7_unchanged(rng):
    """sample_size=7 is the default, and the 7-sample of the generalised sampler is the one the fundamental-matrix path draws."""
    st = matching.mt19937_state(7)
    a, sa = matching.debug_rand_sample(st, rng, 500)
    b, sb = matching.debug_rand_sample(st, rng, 500, sample_size=7)
    assert a.shape == (500, 7) and np.array_equal(a, b) and np.array_equal(sa, sb)
    if acrh.available("ref"):
        want, want_st = acrh.AcransacHOracle("ref").rand_sample(st, 7, rng, 500, states=True)
        assert np.array_equal(a, want) and np.array_equal(sa, want_st)


def test_host_sampler_bad_arguments():
    st = matching.mt19937_state(1)
    for k, rng in ((4, 4), (7, 7), (5, 10), (3, 10)):
        with pytest.raises(av.B200MatchError):
            matching.debug_rand_sample(st, rng, 1, sample_size=k)


@pytest.mark.parametrize("n", [5, 6, 7, 8, 100, 8192])
def test_logc_tables_equal_makelogcombi_4(port, n):
    """The float logc tables for sample size 4 equal the compiled makelogcombi<float>(4, n) bit for bit."""
    got = port.logc(4, n)
    want = acrh.reference_output(f"logc4_{n}", lambda: acrh.AcransacHOracle("ref").logc(4, n), acrh.available("ref"))
    assert np.array_equal(got[0].view(np.uint32), np.asarray(want[0]).view(np.uint32))
    assert np.array_equal(got[1].view(np.uint32), np.asarray(want[1]).view(np.uint32))


@pytest.mark.parametrize("name", [s[0] for s in SCENES])
def test_oracle_ref_equals_port(port, name):
    """The restated loop equals the compiled ACRANSAC bit for bit: inliers and their order, NFA, H, errorMax, iterations, trace and
    the generator's state after the estimation."""
    corr, it, prec = scene(name)
    got = port.estimate(corr, WH, port.mt_seed(SEED), it, prec)
    want = reference(name)
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), (name, k)


def test_scenes_cover_both_outcomes():
    """The scene list holds meaningful and meaningless pairs, pairs too small to draw, and pairs that stop early."""
    v = {name: bool(reference(name)["valid"]) for name, *_ in SCENES}
    assert v["plane_r50_n100"] and v["rot_r90_n500"] and v["rot_r70_n2000"] and v["plane_r60_n8192"] and v["two_planes_n400"]
    assert not v["outliers_n200"] and not v["n3"] and not v["n4"]
    for nm in ("n3", "n4"):
        ref = reference(nm)
        assert int(ref["iterations"]) == 0 and np.array_equal(ref["mt_state_out"], acrh.AcransacHOracle("port").mt_seed(SEED))
    assert int(reference("precision1_outliers")["iterations"]) == 50000 // 10 * 2 + 2   # early exit once iter > 2 * nIterReserve
    # the two-plane scene keeps one plane: at most the larger half of its correspondences
    assert reference("two_planes_n400")["inliers"].size <= 0.6 * 400


def test_four_point_known_answer(port):
    """Homography4PSolver on 4 exact correspondences recovers H up to scale, and the 4 points have zero transfer error."""
    H = np.array([[1.1, 0.05, 0.3], [-0.04, 0.95, -0.2], [0.02, -0.03, 1.0]])
    x1 = np.array([[0.0, 0.0], [1.0, 0.1], [0.9, 1.2], [-0.1, 0.8]])
    p = np.c_[x1, np.ones(4)] @ H.T
    x2 = p[:, :2] / p[:, 2:]
    corr = np.c_[x1, x2]
    G = port.fit4(corr)
    G = G / G[2, 2]
    assert np.abs(G - H).max() < 1e-12
    assert port.errors(port.fit4(corr), corr).max() < 1e-24


# ---------------------------------------------------------------------------------------------------------------- GPU
def _transfer(H, corr) -> np.ndarray:
    """Per correspondence: the distance in image J between xJ and H xI, pixels."""
    p = np.c_[corr[:, :2], np.ones(len(corr))] @ np.asarray(H, np.float64).reshape(3, 3).T
    return np.hypot(corr[:, 2] - p[:, 0] / p[:, 2], corr[:, 3] - p[:, 1] / p[:, 2])


def _rounding_level(new: float, prev: float) -> bool:
    return abs(new - prev) <= 1e-9 * max(1.0, abs(prev))


def _same(got: dict, want: dict, what: str, corr=None):
    assert got["valid"] == bool(want["valid"]), what
    gi, wi = got["inliers"], np.asarray(want["inliers"], np.uint32)
    if corr is not None and gi.size == wi.size and not np.array_equal(gi, wi):
        # the same list, except for an exchange of correspondences the model maps at rounding level (the 4 it was fitted to)
        tie = _transfer(want["H"], corr) < 1e-7
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
    Ha, Hb = np.asarray(got["H"]).ravel(), np.asarray(want["H"]).ravel()
    if np.linalg.norm(Hb) == 0:
        assert np.linalg.norm(Ha) == 0, what
    else:
        Ha = Ha / np.linalg.norm(Ha); Hb = Hb / np.linalg.norm(Hb)
        assert min(np.linalg.norm(Ha - Hb), np.linalg.norm(Ha + Hb)) <= 1e-9, what
    assert np.array_equal(got["mt_state_out"], np.asarray(want["mt_state_out"])), (what, "generator end state")


def _consistent(got: dict, corr, what: str):
    """A result that holds in itself: distinct inliers, and every inlier within errorMax of H xI in image J.  errorMax comes from
    normalised coordinates and the check maps pixels through the unnormalised H, so the two agree to rounding in pixel units
    (1e-6 px absolute; a degenerate sample's inliers can all lie at rounding level, errorMax ~1e-10 px)."""
    inl = got["inliers"]
    assert len(set(inl.tolist())) == inl.size, what
    if got["valid"]:
        assert got["min_nfa"] < 0 and inl.size >= 5, what
        assert _transfer(got["H"], corr)[inl].max() <= got["error_max"] * (1 + 1e-6) + 1e-6, what


def _matches_oracle(got: dict, want: dict, what: str, corr) -> bool:
    """The engine against the oracle's restated loop (pinned to the compiled reference on the CPU), under the protocol of the
    fundamental-matrix tests: the two `better` traces agree event for event (iteration, and minNFA within 1e-9) up to the first
    difference, every output (H and the generator end state included) is equal when there is none, and a difference must be a
    rounding-level improvement on the side that has it (a 4-subset drawn again in another order gives the same model up to the
    last bits of the device and host log10), after which the engine's result is checked for its outcome and for consistency.
    Returns whether they forked."""
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
def ctx():
    return av.Context(0)


@pytest.fixture(scope="module")
def gpu_all(ctx):
    """Every scene in one call per (maxIteration, precision) group, one generator state for all."""
    out = {}
    groups = {}
    for name, _, _, it, prec, _ in SCENES:
        groups.setdefault((it, prec), []).append(name)
    for (it, prec), names in groups.items():
        res = ctx.acransac_homography_pairs([scene(nm)[0] for nm in names], [WH] * len(names), matching.mt19937_state(SEED), it, prec)
        out.update(zip(names, res))
    return out


@pytest.fixture(scope="module")
def port_all(port):
    """The oracle's restated loop on every scene, with the minNFA of each `better` event."""
    out = {}
    for name, *_ in SCENES:
        corr, it, prec = scene(name)
        out[name] = port.estimate(corr, WH, port.mt_seed(SEED), it, prec)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s[0] for s in SCENES if s[0] not in DEGENERATE])
def test_gpu_equals_oracle(gpu_all, port_all, name):
    want = port_all[name]
    ref = reference(name)   # the port is the compiled reference's loop bit for bit (test_oracle_ref_equals_port)
    assert all(np.array_equal(np.asarray(want[k]), np.asarray(ref[k])) for k in acrh.FIELDS), name
    _matches_oracle(gpu_all[name], want, name, scene(name)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DEGENERATE))
def test_gpu_degenerate_scenes(gpu_all, name):
    got, want = gpu_all[name], reference(name)
    assert got["valid"] == bool(want["valid"]), name
    _consistent(got, scene(name)[0], name)


@pytest.mark.gpu
def test_gpu_small_pairs_do_not_draw(gpu_all):
    st = matching.mt19937_state(SEED)
    for nm in ("n3", "n4"):
        g = gpu_all[nm]
        assert not g["valid"] and g["iterations"] == 0 and g["inliers"].size == 0 and g["n_trace"] == 0, nm
        assert np.array_equal(g["mt_state_out"], st), nm
        assert g["error_max"] == 0 and g["min_nfa"] == 0 and not g["H"].any(), nm


@pytest.mark.gpu
def test_gpu_independent_of_skip_batching_and_state_layout(ctx, gpu_all):
    """The same outputs with the certified skip disabled, with the list given pair by pair, and with the shared start state given
    once per pair; distinct per-pair states give each pair what it gives alone."""
    names = ["plane_r10_n300", "plane_r50_n100", "dup_n120", "collinear_n150", "n6", "rot_r70_n2000", "general_r80_n300"]
    corrs = [scene(nm)[0] for nm in names]
    st = matching.mt19937_state(SEED)
    ctx.set_acransac_skip(False)
    try:
        noskip = ctx.acransac_homography_pairs(corrs, [WH] * len(names), st, 50000)
        stats = ctx.acransac_last_stats()
        assert stats["models_skipped"] == 0 and stats["models_exact"] == stats["models_evaluated"] > 0
    finally:
        ctx.set_acransac_skip(True)
    per_pair = ctx.acransac_homography_pairs(corrs, [WH] * len(names), np.tile(st, (len(names), 1)), 50000)
    for nm, a, b in zip(names, noskip, per_pair):
        for r, how in ((a, "no skip"), (b, "per-pair states")):
            _same(r, gpu_all[nm], f"{nm} ({how})")
            assert np.array_equal(r["H"], gpu_all[nm]["H"]) and r["min_nfa"] == gpu_all[nm]["min_nfa"]
    for nm, c in zip(names, corrs):
        one = ctx.acransac_homography_pairs([c], [WH], st, 50000)[0]
        assert np.array_equal(one["H"], gpu_all[nm]["H"]) and np.array_equal(one["inliers"], gpu_all[nm]["inliers"])
        assert one["iterations"] == gpu_all[nm]["iterations"] and one["min_nfa"] == gpu_all[nm]["min_nfa"]
        assert np.array_equal(one["mt_state_out"], gpu_all[nm]["mt_state_out"])
    states = np.stack([matching.mt19937_state(100 + k) for k in range(len(names))])
    many = ctx.acransac_homography_pairs(corrs, [WH] * len(names), states, 50000)
    for k, (nm, c) in enumerate(zip(names, corrs)):
        one = ctx.acransac_homography_pairs([c], [WH], states[k], 50000)[0]
        assert np.array_equal(one["H"], many[k]["H"]) and np.array_equal(one["inliers"], many[k]["inliers"]), nm
        assert np.array_equal(one["mt_state_out"], many[k]["mt_state_out"]), nm


@pytest.mark.gpu
def test_gpu_generator_chain(ctx, port):
    """The reference's single-threaded filter passes one std::mt19937 by reference from pair to pair.  Chaining the engine's calls
    through mt_state_out gives the oracle's chain: one generator handed through 6 pairs."""
    kinds = ["plane", "rotation", "plane", "general", "rotation", "plane"]
    ratios = [0.7, 0.8, 0.0, 0.6, 0.5, 0.9]
    st_g = st_o = port.mt_seed(SEED)
    for k, (kind, ratio) in enumerate(zip(kinds, ratios)):
        corr = h_scene(150 + 40 * k, ratio, 3000 + k, kind=kind)
        want = port.estimate(corr, WH, st_o, 20000)
        got = ctx.acransac_homography_pairs([corr], [WH], st_g, 20000)[0]
        forked = _matches_oracle(got, want, f"chain pair {k}", corr)
        assert got["iterations"] > 0 and not np.array_equal(got["mt_state_out"], st_g)
        st_g = got["mt_state_out"]
        st_o = got["mt_state_out"] if forked else want["mt_state_out"]   # after a fork, the oracle continues from the engine's state


@pytest.mark.gpu
def test_gpu_500_pairs_default_iterations(ctx, port):
    """A 500-pair list at maxIteration = 50000: planar, rotation and outlier pairs and one above the shared-memory sort capacity;
    a sample of pairs matches the oracle, generator end states included."""
    r = np.random.default_rng(4)
    corrs = []
    for k in range(500):
        n = int(r.integers(20, 400)) if k != 250 else 1500
        ratio = 0.7 if k == 250 else 0.0 if k % 3 else float(r.uniform(0.3, 0.9))
        corrs.append(h_scene(n, ratio, 20_000 + k, kind="rotation" if k % 2 else "plane"))
    st = matching.mt19937_state(SEED)
    res = ctx.acransac_homography_pairs(corrs, [WH] * 500, st, 50000)
    stats = ctx.acransac_last_stats()
    assert stats["models_skipped"] > 0 and stats["launches"] == 1
    assert sum(x["valid"] for x in res) >= 100 and res[250]["valid"]   # the pair sorted in global memory has a model
    for k in (0, 1, 3, 250, 499):
        want = port.estimate(corrs[k], WH, st, 50000)
        _matches_oracle(res[k], want, f"pair {k}", corrs[k])


@pytest.mark.gpu
def test_geometricEstimation_H_AC(ctx, port):
    corr, it, prec = scene("plane_r50_n100")
    got = matching.geometricEstimation_H_AC(corr[:, :2], corr[:, 2:], WH[:2], WH[2:], SEED, it, prec, ctx=ctx)
    _matches_oracle(got, port.estimate(corr, WH, port.mt_seed(SEED), it, prec), "geometricEstimation_H_AC", corr)


@pytest.mark.gpu
def test_gpu_bad_arguments(ctx):
    lib = ctx.lib
    corr = scene("plane_r50_n100")[0]
    offsets = np.array([0, len(corr)], np.int64)
    c = np.ascontiguousarray(corr, np.float64)
    st = matching.mt19937_state(1)
    out = {k: np.zeros(s, t) for k, s, t in (("valid", 1, np.uint8), ("ninl", 1, np.int32), ("inl", len(corr), np.uint32), ("H", 9, np.float64),
                                             ("em", 1, np.float64), ("nfa", 1, np.float64), ("it", 1, np.int32), ("sto", 625, np.uint32))}
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None  # noqa: E731

    def call(n=1, offs=offsets, wh=np.array(WH, np.int32), per_pair=0, it=1000, prec=np.inf, state=st):
        return lib.b200m_acransac_homography_pairs(ctx._h, C.c_int(n), p(offs), p(c), p(np.ascontiguousarray(wh, np.int32)), p(state),
                                                   C.c_int(per_pair), C.c_int64(it), C.c_double(prec), p(out["valid"]), p(out["ninl"]),
                                                   p(out["inl"]), p(out["H"]), p(out["em"]), p(out["nfa"]), p(out["it"]), p(out["sto"]))
    assert call() == 0
    for bad in ({"n": -1}, {"per_pair": 2}, {"per_pair": -1}, {"it": -1}, {"it": 1 << 31}, {"prec": 0.0}, {"prec": -1.0},
                {"prec": np.nan}, {"state": None}, {"offs": np.array([1, len(corr) + 1], np.int64)},
                {"offs": np.array([0, -1], np.int64)}, {"wh": np.array([1280, 0, 1200, 900])},
                {"wh": np.array([70000, 70000, 1200, 900])}):
        assert call(**bad) != 0, bad
    assert call(n=0) == 0
