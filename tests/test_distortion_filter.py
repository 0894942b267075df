"""The fundamental_with_distortion filter on the GPU (b200m_acransac_fundamental_distortion_pairs, K10's F10Policy): the engine
equals the port oracle bit for bit (minNFA to 1e-12 relative for the device log10) on a mixed list, results do not depend on the
certified skip, and bad arguments are rejected and leave nothing behind.  On the CPU: the Python stage applies the minimum sample
count of each call group (10 for F10, 7 for the spherical call) in one mixed list."""
from __future__ import annotations

import numpy as np
import pytest

from test_acransac_f10 import SCENES, SEED, WH, audit_f10, params, port, port_all, scene  # noqa: F401

from alicevision_b200 import matching


def _same(got, want, what):
    assert got["valid"] == bool(want["valid"]), what
    assert np.array_equal(got["inliers"], np.asarray(want["inliers"])), what
    assert np.array_equal(got["F"].ravel(), np.asarray(want["F"]).ravel()), (what, got["F"], want["F"])
    assert np.array_equal(got["L"], np.asarray(want["L"])), (what, got["L"], want["L"])
    assert got["error_max"] == float(want["error_max"]), what
    a, c = got["min_nfa"], float(want["min_nfa"])
    assert a == c or abs(a - c) <= 1e-12 * max(abs(a), abs(c)), (what, a, c)   # device vs host log10
    tr = np.asarray(want["trace"])
    assert got["n_trace"] == int(want["n_trace"]) and np.array_equal(got["trace"], tr[:got["trace"].size]), what


@pytest.fixture(scope="module")
def ctx():
    c = matching.Context(0)
    yield c
    c.close()


@pytest.mark.gpu
def test_gpu_equals_port_mixed_list(ctx, port_all):
    """Every scene, in one call per (maxIteration, precision) group from one shared state: the engine is the port bit for bit, and
    every result passes the audit."""
    groups = {}
    for name, _, _, it, prec, _ in SCENES:
        groups.setdefault((it, prec), []).append(name)
    st = matching.mt19937_state(SEED)
    for (it, prec), names in groups.items():
        res = ctx.acransac_fundamental_distortion_pairs([scene(nm) for nm in names], [WH] * len(names), st, it, prec)
        for nm, r in zip(names, res):
            _same(r, port_all[nm], nm)
            audit_f10(r, scene(nm), WH, prec)
            if not r["valid"] and r["n_trace"] == 0:
                assert np.array_equal(r["L"], np.zeros(2))
    st_ = ctx.acransac_last_stats()
    assert st_["launches"] == 1 and st_["models_evaluated"] >= st_["models_exact"]


@pytest.mark.gpu
def test_gpu_independent_of_skip(ctx, port_all):
    names = ["rotating_r80_n200", "barrel_r70_n250", "l0_r70_n250"]
    ctx.set_acransac_skip(False)
    try:
        res = ctx.acransac_fundamental_distortion_pairs([scene(nm) for nm in names], [WH] * 3, matching.mt19937_state(SEED), 2000)
    finally:
        ctx.set_acransac_skip(True)
    for nm, r in zip(names, res):
        _same(r, port_all[nm], nm)


@pytest.mark.gpu
def test_gpu_bad_arguments(ctx):
    from alicevision_b200.matching import B200MatchError
    corr = scene("l0_r70_n250")
    st = matching.mt19937_state(SEED)
    first = ctx.acransac_fundamental_distortion_pairs([corr], [WH], st, 10)[0]
    for bad_wh, prec in (((0, 480, 640, 480), np.inf), ((640, 480, 640, -1), np.inf), ((70000, 70000, 640, 480), np.inf), (WH, 0.0)):
        with pytest.raises(B200MatchError):
            ctx.acransac_fundamental_distortion_pairs([corr], [bad_wh], st, 10, prec)
    again = ctx.acransac_fundamental_distortion_pairs([corr], [WH], st, 10)[0]   # the rejected calls left nothing behind
    _same(again, first, "after rejected calls")


def test_stage_minimum_samples_per_group():
    """_acransac_stage with a per-group minimum sample count: 60 sift inliers (score 8.4) give strong support in the spherical group
    (> 7) and not in the F10 group (> 10); 75 (score 10.5) in both; with one count for every group (the F, H and E callers) both
    pairs of 60 are kept at 7."""
    pairs = [(0, 1), (0, 2), (1, 2), (2, 3)]
    counts = {(0, 1): 60, (0, 2): 60, (1, 2): 75, (2, 3): 75}
    putatives = {p: {"sift": np.zeros(100, matching.MATCH_DTYPE)} for p in pairs}
    common = {p: ["sift"] for p in pairs}

    def run(ks, st):
        return [{"valid": True, "inliers": np.arange(counts[pairs[k]]), "F": np.eye(3), "error_max": 1.0, "L": np.zeros(2)} for k in ks]
    calls = [(run, False), (run, True)]
    groups = [0, 1, 0, 1]   # (0, 1) and (1, 2) through F10, (0, 2) and (2, 3) spherical
    out, info = matching._acransac_stage(None, putatives, {}, None, common, pairs, groups, calls, "F", [10, 7], 1, False, False, 0.6, None)
    assert sorted(out) == [(0, 2), (1, 2), (2, 3)]
    assert not info[(0, 1)]["strong_support"] and info[(0, 2)]["strong_support"]
    out7, _ = matching._acransac_stage(None, putatives, {}, None, common, pairs, groups, calls, "F", 7, 1, False, False, 0.6, None)
    assert sorted(out7) == pairs


# ---------------------------------------------------------------------------------------------- the stage end to end, on the GPU
def _ring(ctx):
    from test_geometric_filter import _putatives, _ring_scene
    regions, sizes = _ring_scene(n_views=6, seed=8)
    pairs = [(i, j) for i in range(6) for j in range(i + 1, 6)]
    return regions, sizes, pairs, _putatives(regions, pairs, ctx)


def _bearings(regions, views):
    """Unit vectors of every feature of `views` through the ring's pinhole K (their pairs become spherical pairs)."""
    out = {}
    for v in views:
        out[v] = {}
        for t, r in regions[v].items():
            x = (r.positions.astype(np.float64) - [960.0, 540.0]) / 1500.0
            b = np.concatenate([x, np.ones((x.shape[0], 1))], 1)
            out[v][t] = b / np.linalg.norm(b, axis=1, keepdims=True)
    return out


def _corr(regions, put, p, types):
    return np.concatenate([np.zeros((0, 4))] + [np.concatenate([regions[p[0]][t].positions[put[p][t]["i"]], regions[p[1]][t].positions[put[p][t]["j"]]], 1)
                                                for t in types if t in put[p]]).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("guided", [False, True])
def test_gpu_robust_model_estimation_with_distortion(guided):
    """robustModelEstimation_F_AC(estimateDistortion=True) on a ring with one spherical pair: every planar pair's F and L are the F10
    call's from the caller's state, the spherical pair's F the spherical call's; a pair is kept iff its copied inliers pass
    hasStrongSupport(.., 10) (planar) or (.., 7) (spherical); with guided matching every kept pair's lists are the guided-matching
    loop's (oracle) on the F10 model matrix read as x_J^T F x_I and errorMax^2, every common type included."""
    from test_geometric_filter import _same_ij
    from oracle import guided_fast as gfo
    O = gfo.best()
    ctx = matching.Context(0)
    try:
        regions, sizes, pairs, put = _ring(ctx)
        bear = _bearings(regions, (0, 1))
        seed, max_it = 42, 300
        out, info = matching.robustModelEstimation_F_AC(put, regions, sizes, seed, max_it, guidedMatching=guided, ctx=ctx, bearings=bear,
                                                        estimateDistortion=True)
        st = matching.mt19937_state(seed)
        kept = {10: 0, 7: 0}
        guided_total = 0
        for p in pairs:
            types = [t for t in matching.DESCRIBER_TYPES if t in regions[p[0]] and t in regions[p[1]]]
            spherical = p == (0, 1)
            assert info[p]["spherical"] == spherical and info[p]["L"].shape == (2,)
            if spherical:
                b = np.concatenate([np.concatenate([bear[p[0]][t][put[p][t]["i"]], bear[p[1]][t][put[p][t]["j"]]], 1) for t in types if t in put[p]])
                want = ctx.acransac_fundamental_spherical_pairs([b], st, max_it)[0]
                assert np.array_equal(info[p]["L"], np.zeros(2))
            else:
                want = ctx.acransac_fundamental_distortion_pairs([_corr(regions, put, p, types)], [sizes[p[0]] + sizes[p[1]]], st, max_it)[0]
                assert np.array_equal(info[p]["L"], want["L"]), p
            assert want["valid"] == info[p]["valid"] and np.array_equal(want["F"], info[p]["F"]) and want["error_max"] == info[p]["error_max"], p
            ms = 7 if spherical else 10
            strong = bool(want["valid"]) and matching.hasStrongSupport(matching.copyInlierMatches(want["inliers"], put[p], types), ms)
            assert (p in out) == strong, p
            kept[ms] += strong
            if strong and guided:
                assert sorted(out[p]) == sorted(types)
                for t in types:
                    r0, r1 = regions[p[0]][t], regions[p[1]][t]
                    w = O.guided_match(r0.descriptors, r0.positions.astype(np.float64), r1.descriptors, r1.positions.astype(np.float64),
                                       info[p]["F"], info[p]["error_max"] ** 2, 0.36, binary=r0.binary)
                    assert _same_ij(out[p][t], w), (p, t)
                    guided_total += len(w)
            elif strong:
                assert all(np.array_equal(out[p][t], v[t]) for v in [matching.copyInlierMatches(want["inliers"], put[p], types)] for t in v)
        assert kept[10] >= 5 and (guided_total > 0 or not guided), (kept, guided_total)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_without_distortion_unchanged():
    """estimateDistortion=False is the fundamental_matrix stage as before: the same results as a call without the argument, every F the
    7-point call's, support at 7, and no "L" in info."""
    ctx = matching.Context(0)
    try:
        regions, sizes, pairs, put = _ring(ctx)
        a = matching.robustModelEstimation_F_AC(put, regions, sizes, 42, 300, guidedMatching=True, ctx=ctx)
        b = matching.robustModelEstimation_F_AC(put, regions, sizes, 42, 300, guidedMatching=True, ctx=ctx, estimateDistortion=False)
        assert a[0].keys() == b[0].keys() and all(a[0][p].keys() == b[0][p].keys() for p in a[0])
        assert all(np.array_equal(a[0][p][t], b[0][p][t]) for p in a[0] for t in a[0][p])
        st = matching.mt19937_state(42)
        for p in pairs:
            assert "L" not in b[1][p] and a[1][p].keys() == b[1][p].keys()
            types = [t for t in matching.DESCRIBER_TYPES if t in regions[p[0]] and t in regions[p[1]]]
            want = ctx.acransac_fundamental_pairs([_corr(regions, put, p, types)], [sizes[p[0]] + sizes[p[1]]], st, 300)[0]
            assert np.array_equal(want["F"], b[1][p]["F"]) and want["valid"] == b[1][p]["valid"]
            assert np.array_equal(a[1][p]["F"], b[1][p]["F"]) and a[1][p]["error_max"] == b[1][p]["error_max"]
            strong = bool(want["valid"]) and matching.hasStrongSupport(matching.copyInlierMatches(want["inliers"], put[p], types), 7)
            assert b[1][p]["strong_support"] == strong
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------- C++ adaptor and integration patch
PATCH_CHAIN = ("", "_knownPoses", "_geometricFilter", "_homographyFilter", "_sphericalFilter", "_homographyGrowingFilter", "_essentialFilter",
               "_distortionFilter")


def _reference_src():
    import oracle
    src = oracle.reference_src()
    if src is None:
        pytest.skip("no AliceVision source tree (ALICEVISION_SRC)")
    return src


def test_distortion_filter_patch_applies(tmp_path):
    """aliceVision_b200_distortionFilter.patch applies after the seven existing patches, in order; it sends the
    FUNDAMENTAL_WITH_DISTORTION case to robustModelEstimationOnB200(.., estimateDistortion = true) for *_B200 matchers with ACRANSAC,
    with the reference's call as the fallback, and changes nothing else but that function's distortion argument."""
    import os
    import re
    import shutil
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    patches = [os.path.join(root, "integration", "patches", f"aliceVision_b200{s}.patch") for s in PATCH_CHAIN]
    files = sorted({m for p in patches for m in re.findall(r"^\+\+\+ b/(\S+)", open(p).read(), re.M)})
    for f in files:
        dst = tmp_path / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        if os.path.exists(os.path.join(os.path.dirname(src), f)):
            shutil.copy(os.path.join(os.path.dirname(src), f), dst)
    for p in patches:
        r = subprocess.run(["patch", "-p1", "-s", "-i", p], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, (p, r.stdout + r.stderr)
    text = (tmp_path / "src" / "software" / "pipeline" / "main_featureMatching.cpp").read_text()
    case = text[text.index("case EGeometricFilterType::FUNDAMENTAL_WITH_DISTORTION:"):text.index("case EGeometricFilterType::ESSENTIAL_MATRIX:")]
    assert "ERobustEstimator::ACRANSAC" in case and "randomNumberGenerator, guidedMatching, true))" in case
    assert case.index("robustModelEstimationOnB200(") < case.index("GeometricFilterMatrix_F_AC(geometricErrorMax, maxIteration, geometricEstimator, true)")
    assert "GeometricFilterMatrix_F_AC_Batch_b200 batch(matching::b200detail::sharedContext(), estimateDistortion);" in text
    ours = open(patches[-1]).read()
    assert set(re.findall(r"^\+\+\+ b/(\S+)", ours, re.M)) == {"src/software/pipeline/main_featureMatching.cpp"}
    removed = [ln[1:].strip() for ln in ours.splitlines() if ln.startswith("-") and not ln.startswith("---")]
    assert removed and all(ln in ("/// Returns false (geometricMatches untouched) when the engine is unavailable or fails.",
                                  "const std::mt19937& randomNumberGenerator, bool guidedMatching)",
                                  "GeometricFilterMatrix_F_AC_Batch_b200 batch;")
                           or ln.startswith("matchingImageCollection::robustModelEstimation(") or ln in (
                               "&sfmData,", "regionPerView,", "GeometricFilterMatrix_F_AC(geometricErrorMax, maxIteration, geometricEstimator, true),",
                               "mapPutativesMatches,", "randomNumberGenerator,", "guidedMatching);") for ln in removed), removed


def test_distortion_filter_adaptor_header_compiles():
    import os
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "alicevision_b200", "adaptor", "GeometricFilter_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(root, "oracle", "shim"), "-I", src,
                        "-I", os.path.join(root, "include"), "-I", os.path.join(root, "alicevision_b200", "adaptor"), hdr],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.gpu
def test_gpu_distortion_filter_cpp_adaptor():
    """GeometricFilterMatrix_F_AC_Batch_b200 with estimateDistortion against the "ref" oracles in one executable
    (tests/cpp/distortion_filter_test.cpp)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "distortion_filter_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "distortion_filter adaptor ok" in r.stdout
