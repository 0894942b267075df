"""The host logic the three a-contrario filter stages share (robustModelEstimation_F_AC, _H_AC and _E_AC), against a recording
stand-in for the engine context: which engine calls each stage makes and with which pairs and start states (chain=False / True), the
per-pair `info`, the strong-support threshold of each stage at its boundary, the kept lists, and the guided step (its items, models,
squared thresholds and ratio, the position-only call of H, views uploaded once and always removed)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from alicevision_b200 import matching

MD = matching.MATCH_DTYPE
S0 = np.arange(625, dtype=np.uint32) * 3       # the caller's generator state; the stand-in's calls advance a state by one


def _matches(n: int, offset: int = 0) -> np.ndarray:
    m = np.zeros(n, MD)
    m["i"] = np.arange(n) + offset
    m["j"] = np.arange(n) + offset
    m["ratio"] = 0.5
    m["dist"] = np.arange(n) + offset + 0.25
    return m


class _Regions:
    def __init__(self, n: int, shift: float = 0.0):
        self.positions = np.stack([np.arange(n, dtype=np.float32) + shift, np.arange(n, dtype=np.float32) * 0.5], 1)

    def RegionCount(self) -> int:
        return len(self.positions)


class _Lib:
    def __init__(self):
        self.removed = []

    def b200m_remove_view(self, h, vid):
        assert h == "ctx-handle"
        self.removed.append(vid.value)


class _FakeCtx:
    """Stands in for Context: every K10 and guided call is recorded; each K10 pair gets the scripted result of its correspondence count
    n, script[n] = (valid, inliers, error_max), and the model n * ones + eye (3 x 3).  "mt_state_out" (the pair's start state + 1) is
    returned by the calls whose real method returns it: all but the planar fundamental one."""

    def __init__(self, script: dict, guided_raises: bool = False):
        self.script, self.guided_raises = script, guided_raises
        self.calls, self.guided = [], []
        self.lib, self._h = _Lib(), "ctx-handle"

    def _k10(self, kind, key, corr_list, st, maxIteration, precision, wh=None, K=None):
        st = np.asarray(st, np.uint32)
        self.calls.append({"kind": kind, "n": [len(c) for c in corr_list], "corr": [np.asarray(c) for c in corr_list], "wh": wh, "K": K,
                           "state": st.copy(), "maxIteration": maxIteration, "precision": precision})
        out = []
        for q, c in enumerate(corr_list):
            valid, inl, em = self.script[len(c)]
            r = {"valid": valid, "inliers": np.asarray(inl, np.uint32), key: len(c) * np.ones((3, 3)) + np.eye(3), "error_max": em,
                 "min_nfa": -1.0, "iterations": 1}
            if kind != "F":
                r["mt_state_out"] = (st if st.ndim == 1 else st[q]) + np.uint32(1)
            out.append(r)
        return out

    def acransac_fundamental_pairs(self, corr_list, wh, mt_state, maxIteration=50000, precision=np.inf):
        return self._k10("F", "F", corr_list, mt_state, maxIteration, precision, wh=wh)

    def acransac_fundamental_spherical_pairs(self, corr_list, mt_state_or_states, maxIteration=50000, precision=np.inf):
        return self._k10("S", "F", corr_list, mt_state_or_states, maxIteration, precision)

    def acransac_homography_pairs(self, corr_list, wh, mt_state_or_states, maxIteration=50000, precision=np.inf):
        return self._k10("H", "H", corr_list, mt_state_or_states, maxIteration, precision, wh=wh)

    def acransac_essential_pairs(self, corr_list, wh, K, mt_state_or_states, maxIteration=50000, precision=np.inf):
        return self._k10("E", "E", corr_list, mt_state_or_states, maxIteration, precision, wh=wh, K=K)

    def _lists(self, call, pairs, M, errorTh, **kw):
        self.guided.append(dict(call=call, pairs=[tuple(int(v) for v in p) for p in pairs], M=[np.asarray(m) for m in M],
                                errorTh=list(errorTh), **kw))
        if self.guided_raises:
            raise RuntimeError("guided call failed")
        return [_matches(q, offset=100 * q) for q in range(len(pairs))]     # item 0 gets an empty list

    def guided_match_pairs(self, pairs, M, errorTh, distRatio, model=matching.MODEL_FUNDAMENTAL):
        return self._lists("ratio", pairs, M, errorTh, distRatio=distRatio, model=model)

    def guided_match_positions_pairs(self, pairs, M, errorTh, model=matching.MODEL_HOMOGRAPHY, decorate=True):
        return self._lists("positions", pairs, M, errorTh, model=model, decorate=decorate)


@pytest.fixture
def uploads(monkeypatch):
    """Records matching._upload_pair: (view id, regions, guided positions) per upload."""
    rec = []

    def upload(ctx, ids, regions, geometry, up):
        for vid, r, xy in zip(ids, regions, geometry):
            rec.append((vid, r, xy))
            up.append(vid)
    monkeypatch.setattr(matching, "_upload_pair", upload)
    return rec


# The scene.  Pairs in putative-list order, with their correspondence counts:
#   P1 (0, 1)  30 cctag3                 planar     valid, 10 inliers given descending, errorMax 2
#   P2 (5, 6)  22 cctag3                 spherical  valid, 12 inliers, errorMax +inf
#   P3 (1, 2)  13 sift + 5 cctag3 = 18   planar     valid, 3 sift + 5 cctag3 inliers: support 5.42, only above 4 and 5
#   P4 (0, 4)  no common type
#   P5 (6, 5)  17 cctag3                 spherical  not valid (errorMax 3 all the same)
#   P6 (2, 0)  12 cctag3                 planar     valid, 12 inliers, errorMax 0.5
P1, P2, P3, P4, P5, P6 = (0, 1), (5, 6), (1, 2), (0, 4), (6, 5), (2, 0)
SCRIPT = {30: (True, np.arange(9, -1, -1), 2.0), 22: (True, np.arange(12), np.inf), 18: (True, [17, 16, 15, 14, 13, 2, 1, 0], 1.5),
          17: (False, np.arange(17), 3.0), 12: (True, np.arange(12), 0.5)}
K0 = np.array([[700.0, 0, 320], [0, 700, 240], [0, 0, 1]])
KS = {0: K0, 1: K0 * [[1.1], [1.1], [1]], 2: K0 + [[0, 0.5, 10], [0, 0, -5], [0, 0, 0]], 4: K0, 6: None}   # view 5: no entry


def _scene():
    regions = {0: {"cctag3": _Regions(40)}, 1: {"sift": _Regions(40, 1), "cctag3": _Regions(40, 2)},
               2: {"sift": _Regions(40, 3), "cctag3": _Regions(40, 4)}, 4: {"dspsift": _Regions(40)}, 5: {"cctag3": _Regions(40, 5)},
               6: {"cctag3": _Regions(40, 6)}}
    putatives = {P1: {"cctag3": _matches(30)}, P2: {"cctag3": _matches(22)}, P3: {"sift": _matches(13, 1), "cctag3": _matches(5, 2)},
                 P4: {}, P5: {"cctag3": _matches(17)}, P6: {"cctag3": _matches(12, 3)}}
    sizes = {v: (640 + v, 480 - v) for v in regions}
    bearings = {v: {"cctag3": np.tile([[0.0, 0.6, 0.8]], (40, 1)) * (1 + v)} for v in (5, 6)}
    guided_geometry = {1: {"sift": np.full((40, 2), 7.0)}}
    return regions, putatives, sizes, bearings, guided_geometry


def _run(stage, ctx, scene=None, **kw):
    regions, putatives, sizes, bearings, guided_geometry = scene or _scene()
    kw.setdefault("guided_geometry", guided_geometry)
    if stage == "F":
        return matching.robustModelEstimation_F_AC(putatives, regions, sizes, kw.pop("seed", S0), bearings=bearings, ctx=ctx, **kw)
    if stage == "H":
        return matching.robustModelEstimation_H_AC(putatives, regions, sizes, kw.pop("seed", S0), ctx=ctx, **kw)
    return matching.robustModelEstimation_E_AC(putatives, regions, sizes, KS, kw.pop("seed", S0), ctx=ctx, **kw)


def _calls(ctx):
    """(kind, correspondence counts, first word of the start state(s)) per K10 call."""
    return [(c["kind"], c["n"], c["state"].reshape(-1, 625)[:, 0].tolist()) for c in ctx.calls]


# --- the engine calls ------------------------------------------------------------------------------------------------------------

ONE_CALL = {
    "F": [("F", [30, 18, 12], [0]), ("S", [22, 17], [0])],
    "H": [("H", [30, 22, 18, 17, 12], [0])],
    "E": [("E", [30, 18, 12], [0])],
}
CHAINED = {     # every spherical F, H or E pair alone, handing its mt_state_out on (planar runs: test_planar_runs_share_one_call)
    "F": [("F", [30], [0]), ("S", [22], [0]), ("F", [18], [1]), ("S", [17], [1]), ("F", [12], [2])],
    "H": [("H", [n], [k]) for k, n in enumerate([30, 22, 18, 17, 12])],
    "E": [("E", [n], [k]) for k, n in enumerate([30, 18, 12])],
}


@pytest.mark.parametrize("stage", "FHE")
@pytest.mark.parametrize("chain", [False, True])
def test_engine_calls(stage, chain):
    ctx = _FakeCtx(SCRIPT)
    _run(stage, ctx, chain=chain, maxIteration=1234, precision=3.0)
    assert _calls(ctx) == (CHAINED if chain else ONE_CALL)[stage]
    for c in ctx.calls:
        assert c["maxIteration"] == 1234
        assert c["precision"] == (9.0 if stage == "E" else 3.0)          # the E filter passes Square(precision) to ACRANSAC
        if not chain:
            assert np.array_equal(c["state"], S0)
    if chain:                                                          # the state handed on is the previous call's mt_state_out
        assert all(np.array_equal(c["state"], S0 + np.uint32(w)) for c, (_, _, (w,)) in zip(ctx.calls, CHAINED[stage]))


@pytest.mark.parametrize("chain", [False, True])
def test_planar_runs_share_one_call(chain):
    """Adjacent planar F pairs go in one call, with chain=True from the state the last spherical pair left; a pair without a common
    type between them draws nothing and does not split the run."""
    regions = {v: {"cctag3": _Regions(40, v)} for v in (0, 1, 2, 3, 5, 6)}
    regions[4] = {"dspsift": _Regions(40)}
    order = [((0, 1), 11), ((1, 2), 12), ((5, 6), 13), ((2, 3), 14), ((0, 4), 0), ((3, 0), 15), ((0, 2), 16), ((6, 5), 17), ((1, 3), 18)]
    putatives = {p: ({"cctag3": _matches(n)} if n else {}) for p, n in order}
    bearings = {v: {"cctag3": np.tile([[0.0, 0.6, 0.8]], (40, 1))} for v in (5, 6)}
    scene = (regions, putatives, {v: (640, 480) for v in regions}, bearings, None)
    ctx = _FakeCtx({n: (True, np.arange(8), 1.0) for _, n in order if n})
    _, info = _run("F", ctx, scene, chain=chain)
    want = ([("F", [11, 12], [0]), ("S", [13], [0]), ("F", [14, 15, 16], [1]), ("S", [17], [1]), ("F", [18], [2])] if chain else
            [("F", [11, 12, 14, 15, 16, 18], [0]), ("S", [13, 17], [0])])
    assert _calls(ctx) == want
    assert [p for p, d in info.items() if d["strong_support"]] == [p for p, n in order if n]


def test_engine_call_inputs():
    """Correspondences, image sizes, bearings and K reach the calls as the pairs' putatives select them."""
    regions, putatives, sizes, bearings, _ = scene = _scene()
    for stage in "FHE":
        ctx = _FakeCtx(SCRIPT)
        _run(stage, ctx, scene)
        by_n = {n: (c, k) for c in ctx.calls for k, n in enumerate(c["n"])}
        for p in (P1, P2, P3, P5, P6):
            n = sum(len(m) for m in putatives[p].values())
            if n not in by_n:
                continue
            c, k = by_n[n]
            types = [t for t in matching.DESCRIBER_TYPES if t in putatives[p]]
            if c["kind"] == "S":
                want = np.concatenate([np.c_[bearings[p[0]][t][putatives[p][t]["i"]], bearings[p[1]][t][putatives[p][t]["j"]]] for t in types])
            else:
                want = np.concatenate([np.c_[regions[p[0]][t].positions[putatives[p][t]["i"]], regions[p[1]][t].positions[putatives[p][t]["j"]]]
                                       for t in types])
                assert tuple(c["wh"][k]) == tuple(sizes[p[0]]) + tuple(sizes[p[1]])
            assert np.array_equal(c["corr"][k], want)
            if stage == "E":
                assert np.array_equal(c["K"][k], np.concatenate([np.ravel(KS[p[0]]), np.ravel(KS[p[1]])]))


def test_seed_is_the_generator_state():
    """An integer seed starts every stage from std::mt19937(seed)."""
    for stage in "FHE":
        ctx = _FakeCtx(SCRIPT)
        _run(stage, ctx, seed=5489)
        assert ctx.calls and all(np.array_equal(c["state"], matching.mt19937_state(5489)) for c in ctx.calls)


def test_no_estimated_pair_makes_no_call():
    regions, putatives, sizes, bearings, gg = _scene()
    scene = (regions, {P4: {}}, sizes, bearings, gg)
    for stage in "FHE":
        for chain in (False, True):
            ctx = _FakeCtx(SCRIPT)
            out, info = _run(stage, ctx, scene, chain=chain, guidedMatching=True)
            assert ctx.calls == [] and out == {} and list(info) == [P4]


@pytest.mark.parametrize("geom", ["F", "H", "E"])
def test_geometric_estimation_single_pair(geom):
    """geometricEstimation_*_AC: one pair, its n x 4 correspondences (xI, yI, xJ, yJ), its sizes, the seed's state and the engine's
    result for it."""
    ctx = _FakeCtx({5: (True, [0, 1, 2], 1.0)})
    xI, xJ = np.arange(10.0).reshape(5, 2), np.arange(10.0, 20.0).reshape(5, 2)
    if geom == "E":
        r = matching.geometricEstimation_E_AC(xI, xJ, (640, 480), (600, 400), K0, 2 * K0, 42, 77, 2.5, ctx=ctx)
        assert np.array_equal(ctx.calls[0]["K"][0], np.r_[K0.ravel(), 2 * K0.ravel()])
    else:
        fn = matching.geometricEstimation_F_AC if geom == "F" else matching.geometricEstimation_H_AC
        r = fn(xI, xJ, (640, 480), (600, 400), 42, 77, 2.5, ctx=ctx)
    (c,) = ctx.calls
    assert c["kind"] == geom and c["n"] == [5] and c["maxIteration"] == 77 and c["precision"] == 2.5
    assert np.array_equal(c["corr"][0], np.c_[xI, xJ]) and [tuple(w) for w in c["wh"]] == [(640, 480, 600, 400)]
    assert np.array_equal(c["state"], matching.mt19937_state(42))
    assert r["valid"] and np.array_equal(r["inliers"], [0, 1, 2])
    ctx = _FakeCtx({5: (True, [0], 1.0)})
    st = S0 + np.uint32(7)
    if geom == "E":
        matching.geometricEstimation_E_AC(xI, xJ, (640, 480), (600, 400), K0, K0, st, ctx=ctx)
    else:
        fn(xI, xJ, (640, 480), (600, 400), st, ctx=ctx)
    assert np.array_equal(ctx.calls[0]["state"], st) and ctx.calls[0]["maxIteration"] == 50000 and np.isinf(ctx.calls[0]["precision"])


# --- info, support and the kept lists ----------------------------------------------------------------------------------------------

def _model(n):
    return n * np.ones((3, 3)) + np.eye(3)


@pytest.mark.parametrize("stage", "FHE")
@pytest.mark.parametrize("chain", [False, True])
def test_info(stage, chain):
    ctx = _FakeCtx(SCRIPT)
    _, info = _run(stage, ctx, chain=chain)
    _, putatives, *_ = _scene()
    assert list(info) == list(putatives)
    strong = {"F": {P1, P2, P6}, "H": {P1, P2, P3, P6}, "E": {P1, P3, P6}}[stage]
    estimated = {"F": {P1, P2, P3, P5, P6}, "H": {P1, P2, P3, P5, P6}, "E": {P1, P3, P6}}[stage]
    counts = {P1: 30, P2: 22, P3: 18, P5: 17, P6: 12}
    out_state = {n: c["state"] + np.uint32(1) for c in ctx.calls for n in c["n"]}     # every call here has one shared start state
    for p, d in info.items():
        keys = {"valid", "strong_support", stage, "error_max"} | ({"spherical"} if stage == "F" else set())
        if p in estimated and (stage != "F" or p in (P2, P5)):
            keys.add("mt_state_out")
        assert set(d) == keys, p
        if stage == "F":
            assert d["spherical"] == (p in (P2, P5))
        if p in estimated:
            valid, _, em = SCRIPT[counts[p]]
            assert d["valid"] == valid and np.array_equal(d[stage], _model(counts[p])) and d["error_max"] == em
        else:
            assert not d["valid"] and np.array_equal(d[stage], np.zeros((3, 3))) and np.isinf(d["error_max"])
        assert d["strong_support"] == (p in strong), p
        if "mt_state_out" in d:
            assert np.array_equal(d["mt_state_out"], out_state[counts[p]])


@pytest.mark.parametrize("stage", "FHE")
def test_kept_lists_without_guided_matching(stage):
    ctx = _FakeCtx(SCRIPT)
    out, _ = _run(stage, ctx)
    _, putatives, *_ = _scene()
    want = {"F": {P1, P2, P6}, "H": {P1, P2, P3, P6}, "E": {P1, P3, P6}}[stage]
    assert set(out) == want and ctx.guided == []
    assert set(out[P1]) == {"cctag3"} and np.array_equal(out[P1]["cctag3"], putatives[P1]["cctag3"][:10])
    if P3 in want:     # inliers given descending, split per type, ratio and distance kept
        assert list(out[P3]) == ["sift", "cctag3"]
        assert np.array_equal(out[P3]["sift"], putatives[P3]["sift"][:3]) and np.array_equal(out[P3]["cctag3"], putatives[P3]["cctag3"])
    assert np.array_equal(out[P6]["cctag3"], putatives[P6]["cctag3"])


@pytest.mark.parametrize("stage,minimum", [("F", 7), ("H", 4), ("E", 5)])
def test_strong_support_threshold(stage, minimum):
    """A pair needs a support score above the solver's minimum sample count: 7 (F), 4 (H), 5 (E); cctag3 counts 1 per match."""
    regions = {v: {"cctag3": _Regions(40)} for v in range(3)}
    putatives = {(0, 1): {"cctag3": _matches(20)}, (1, 2): {"cctag3": _matches(21)}}
    scene = (regions, putatives, {v: (640, 480) for v in regions}, {}, None)
    ctx = _FakeCtx({20: (True, np.arange(minimum), 1.0), 21: (True, np.arange(minimum + 1), 1.0)})
    out, info = _run(stage, ctx, scene)
    assert [info[p]["strong_support"] for p in putatives] == [False, True]
    assert list(out) == [(1, 2)] and len(out[(1, 2)]["cctag3"]) == minimum + 1


# --- the guided step ---------------------------------------------------------------------------------------------------------------

GUIDED_ITEMS = {"F": [(P1, "cctag3"), (P6, "cctag3")],
                "H": [(P1, "cctag3"), (P3, "sift"), (P3, "cctag3"), (P6, "cctag3")],
                "E": [(P1, "cctag3"), (P3, "sift"), (P3, "cctag3"), (P6, "cctag3")]}
COUNTS = {P1: 30, P2: 22, P3: 18, P5: 17, P6: 12}


@pytest.mark.parametrize("stage,ratio,call", [("F", 0.6, "ratio"), ("F", -0.5, "ratio"), ("H", 0.7, "ratio"), ("H", -1.0, "positions"),
                                              ("E", 0.6, "ratio"), ("E", -0.5, "ratio")])
def test_guided_step(stage, ratio, call, uploads):
    regions, putatives, sizes, bearings, gg = scene = _scene()
    ctx = _FakeCtx(SCRIPT)
    out, info = _run(stage, ctx, scene, guidedMatching=True, distanceRatio=ratio)
    items = GUIDED_ITEMS[stage]
    (g,) = ctx.guided
    assert g["call"] == call
    assert g["model"] == (matching.MODEL_HOMOGRAPHY if stage == "H" else matching.MODEL_FUNDAMENTAL)
    if call == "ratio":
        assert g["distRatio"] == ratio * ratio
    else:
        assert g["decorate"] is True
    # each (view, type) of the items is uploaded once, with its regions and guided positions
    ids = {}
    for vid, r, xy in uploads:
        (v, t), = [(v, t) for v in regions for t in regions[v] if regions[v][t] is r]
        assert (v, t) not in ids
        ids[(v, t)] = vid
        assert xy is (gg.get(v, {}).get(t))
    assert set(ids) == {(v, t) for p, t in items for v in p}
    assert g["pairs"] == [(ids[(p[0], t)], ids[(p[1], t)]) for p, t in items]
    for (p, _), M, th in zip(items, g["M"], g["errorTh"]):
        em = SCRIPT[COUNTS[p]][2]
        assert th == em * em
        want = matching.fundamentalFromEssential(_model(COUNTS[p]), KS[p[0]], KS[p[1]]) if stage == "E" else _model(COUNTS[p])
        assert np.array_equal(M, want)
    # the guided lists replace the inliers (empty ones included); a kept pair with an infinite errorMax gets none
    want = {p: {} for p in {"F": (P1, P2, P6), "H": (P1, P2, P3, P6), "E": (P1, P3, P6)}[stage]}
    for q, (p, t) in enumerate(items):
        want[p][t] = _matches(q, offset=100 * q)
    assert set(out) == set(want)
    for p in want:
        assert list(out[p]) == list(want[p]) and all(np.array_equal(out[p][t], want[p][t]) for t in want[p])
    assert len(out[P1]["cctag3"]) == 0
    if P2 in out:
        assert out[P2] == {} and info[P2]["strong_support"]
    assert sorted(ctx.lib.removed) == sorted(ids.values())


@pytest.mark.parametrize("stage", "FHE")
def test_guided_views_removed_when_the_call_fails(stage, uploads):
    ctx = _FakeCtx(SCRIPT, guided_raises=True)
    with pytest.raises(RuntimeError, match="guided call failed"):
        _run(stage, ctx, guidedMatching=True)
    assert uploads and sorted(ctx.lib.removed) == sorted(vid for vid, _, _ in uploads)


@pytest.mark.parametrize("stage", "FHE")
def test_guided_step_without_finite_error_max(stage, uploads):
    """Kept pairs whose errorMax is infinite get an empty map and no guided call is made."""
    regions = {v: {"cctag3": _Regions(40)} for v in range(2)}
    scene = (regions, {(0, 1): {"cctag3": _matches(20)}}, {v: (640, 480) for v in regions}, {}, None)
    ctx = _FakeCtx({20: (True, np.arange(10), np.inf)})
    out, _ = _run(stage, ctx, scene, guidedMatching=True)
    assert out == {(0, 1): {}} and ctx.guided == [] and uploads == []
