"""The `essential_matrix` filter stage: robustModelEstimation_E_AC (pair selection, the geometricErrorMax^4 threshold, support,
guided matching with F from E, the generator chain) and removePoorlyOverlappingImagePairs.

CPU tests run the stage's host logic against a recording stand-in for the engine context; GPU tests run it end to end on engine
putatives of a calibrated ring of views and compare every estimate with the oracle port and every guided list with the guided-matching
oracle fed the same F.
"""
from __future__ import annotations

import numpy as np
import pytest

from alicevision_b200 import matching, synth
from oracle import acransac_e as acre
from oracle import guided_fast as gfo

MD = matching.MATCH_DTYPE


def _matches(n: int, offset: int = 0) -> np.ndarray:
    m = np.zeros(n, MD)
    m["i"] = np.arange(n) + offset
    m["j"] = np.arange(n) + offset
    return m


class _Regions:
    def __init__(self, n: int):
        self.positions = np.stack([np.arange(n, dtype=np.float32), np.arange(n, dtype=np.float32) * 0.5], 1)

    def RegionCount(self) -> int:
        return len(self.positions)


class _RecordingCtx:
    """Stands in for Context.acransac_essential_pairs: records each call and returns one invalid estimate per pair."""
    def __init__(self):
        self.calls = []

    def acransac_essential_pairs(self, corr_list, wh, K, st, maxIteration, precision):
        self.calls.append({"corr": corr_list, "wh": wh, "K": K, "precision": precision, "maxIteration": maxIteration})
        return [{"valid": False, "inliers": np.zeros(0, np.uint32), "E": np.zeros((3, 3)), "error_max": np.inf, "min_nfa": np.inf,
                 "iterations": 0, "mt_state_out": np.asarray(st).reshape(-1, 625)[0]} for _ in corr_list]


K0 = np.array([[700.0, 0, 320], [0, 700, 240], [0, 0, 1]])


def _stage_inputs():
    regions = {0: {"sift": _Regions(40)}, 1: {"sift": _Regions(40)}, 2: {"sift": _Regions(40)}, 3: {"akaze_mldb": _Regions(40)},
               4: {"sift": _Regions(40)}, 5: {"sift": _Regions(40)}}
    putatives = {(0, 1): {"sift": _matches(30)}, (0, 2): {"sift": _matches(20)}, (1, 3): {}, (0, 4): {"sift": _matches(10)},
                 (1, 5): {"sift": _matches(12)}}
    sizes = {v: (640, 480) for v in regions}
    # view 2 has no intrinsic entry, view 4 a non-pinhole camera (None)
    intrinsics = {0: K0, 1: K0 * [[1.1], [1.1], [1]], 3: K0, 4: None, 5: K0}
    return regions, putatives, sizes, intrinsics


def test_stage_pair_selection():
    """A pair is estimated only with a common describer type and a pinhole K on both views; the others get the default estimate and
    make no draw."""
    regions, putatives, sizes, intrinsics = _stage_inputs()
    ctx = _RecordingCtx()
    out, info = matching.robustModelEstimation_E_AC(putatives, regions, sizes, intrinsics, 5489, ctx=ctx)
    assert out == {} and set(info) == set(putatives)
    (call,) = ctx.calls
    assert [c.shape[0] for c in call["corr"]] == [30, 12]          # (0, 1) and (1, 5)
    assert np.array_equal(call["K"][0], np.concatenate([K0.ravel(), (K0 * [[1.1], [1.1], [1]]).ravel()]))
    assert call["wh"] == [(640, 480, 640, 480)] * 2
    for p in ((0, 2), (1, 3), (0, 4)):
        assert not info[p]["valid"] and np.isinf(info[p]["error_max"]) and "mt_state_out" not in info[p]


@pytest.mark.parametrize("prec,want", [(np.inf, np.inf), (2.0, 4.0), (0.5, 0.25), (3.0, 9.0)])
def test_stage_threshold_is_squared_twice(prec, want):
    """The filter passes Square(geometricErrorMax) to ACRANSAC, which squares it again: the residual threshold is precision^4; the
    default (+inf) stays +inf."""
    regions, putatives, sizes, intrinsics = _stage_inputs()
    ctx = _RecordingCtx()
    matching.robustModelEstimation_E_AC(putatives, regions, sizes, intrinsics, 5489, precision=prec, ctx=ctx)
    assert ctx.calls[0]["precision"] == want


def test_stage_chain_runs_one_pair_per_call():
    regions, putatives, sizes, intrinsics = _stage_inputs()
    ctx = _RecordingCtx()
    matching.robustModelEstimation_E_AC(putatives, regions, sizes, intrinsics, 5489, chain=True, ctx=ctx)
    assert [len(c["corr"]) for c in ctx.calls] == [1, 1]


def test_fundamental_from_essential_order():
    E = np.array([[0.0, -1, 0.2], [1, 0, -0.3], [-0.1, 0.4, 0]])
    KJ = K0 * [[1.1], [1.1], [1]]
    F = matching.fundamentalFromEssential(E, K0, KJ)
    assert np.allclose(F, np.linalg.inv(KJ).T @ E @ np.linalg.inv(K0), rtol=1e-14, atol=1e-18)


def _geo(counts: dict) -> dict:
    return {p: {"sift": _matches(g)} for p, g in counts.items()}


@pytest.mark.parametrize("g,n,kept", [
    (50, 166, True),     # 50 / 166 = 0.3012 >= 0.3
    (50, 167, False),    # 0.2994 < 0.3
    (49, 100, False),    # fewer than 50 geometric matches
    (50, 50, True),
    (60, 200, True),     # 60 / 200 = 0.3f exactly: not below
    (3, 10, False),      # 0.3f exactly but fewer than 50
])
def test_remove_poorly_overlapping_image_pairs(g, n, kept):
    geo = _geo({(0, 1): g})
    put = {(0, 1): {"sift": _matches(n - n // 2), "akaze_mldb": _matches(n // 2)}}   # the putative count spans the types
    out = matching.removePoorlyOverlappingImagePairs(geo, put)
    assert ((0, 1) in out) == kept


def test_remove_poorly_overlapping_float_ratio():
    """The ratio is a float division compared with the float 0.3f: 3 / 10 in float equals 0.3f, so a pair at that ratio is kept."""
    assert np.float32(3) / np.float32(10) == np.float32(0.3)
    out = matching.removePoorlyOverlappingImagePairs(_geo({(0, 1): 3}), {(0, 1): {"sift": _matches(10)}}, minimumGeometricCount=0)
    assert (0, 1) in out
    out = matching.removePoorlyOverlappingImagePairs(_geo({(0, 1): 299}), {(0, 1): {"sift": _matches(1000)}}, minimumGeometricCount=0)
    assert (0, 1) not in out


def _reference_src():
    import oracle
    src = oracle.reference_src()
    if src is None:
        pytest.skip("needs the AliceVision source tree")
    return src


PATCH_CHAIN = ("", "_knownPoses", "_geometricFilter", "_homographyFilter", "_sphericalFilter", "_homographyGrowingFilter", "_essentialFilter")


def test_essential_filter_patch_applies(tmp_path):
    """aliceVision_b200_essentialFilter.patch applies after the six existing patches, in order, to copies of the reference files; it
    sends only the ESSENTIAL_MATRIX case's robustModelEstimation call to the batch, with the reference's call as the fallback, and
    leaves the reference's removePoorlyOverlappingImagePairs where it is."""
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
    assert "GeometricFilterMatrix_E_AC_Batch_b200 batch;" in text
    case = text[text.index("case EGeometricFilterType::ESSENTIAL_MATRIX:"):text.index("case EGeometricFilterType::HOMOGRAPHY_MATRIX:")]
    assert case.index("robustModelEstimationEOnB200(") < case.index("GeometricFilterMatrix_E_AC(geometricErrorMax, maxIteration)")
    assert case.index("GeometricFilterMatrix_E_AC(geometricErrorMax, maxIteration)") < case.index(
        "removePoorlyOverlappingImagePairs(geometricMatches, mapPutativesMatches, 0.3f, 50);")
    ours = open(patches[-1]).read()
    assert set(re.findall(r"^\+\+\+ b/(\S+)", ours, re.M)) == {"src/software/pipeline/main_featureMatching.cpp"}
    assert not [ln for ln in ours.splitlines() if ln.startswith("-") and not ln.startswith("---") and "E_AC" not in ln
                and "robustModelEstimation(" not in ln and ln.strip("-").strip() not in
                ("&sfmData,", "regionPerView,", "mapPutativesMatches,", "randomNumberGenerator,", "guidedMatching);")]


def test_essential_filter_adaptor_header_compiles():
    import os
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "alicevision_b200", "adaptor", "GeometricFilter_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(root, "oracle", "shim"), "-I", src,
                        "-I", os.path.join(root, "include"), "-I", os.path.join(root, "alicevision_b200", "adaptor"), hdr],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "GeometricFilterMatrix_E_AC_Batch_b200" in open(hdr).read()


def test_adaptor_fundamental_from_essential_matches_python():
    """The adaptor's F (the one its guided step uses) is matching.fundamentalFromEssential's, bit for bit, through a tiny C++ program."""
    import os
    import subprocess
    import tempfile
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    prog = r"""
#include <GeometricFilter_b200.hpp>
#include <cstdio>
int main() {
    const double E[9] = {0.0, -1, 0.2, 1, 0, -0.3, -0.1, 0.4, 0};
    const double KI[9] = {700, 0, 320, 0, 700, 240, 0, 0, 1}, KJ[9] = {770, 0.5, 300, 0, 760, 250, 0, 0, 1};
    double F[9];
    aliceVision::matchingImageCollection::GeometricFilterMatrix_E_AC_Batch_b200::fundamentalFromEssential(E, KI, KJ, F);
    for (double f : F) std::printf("%.17g\n", f);
}
"""
    with tempfile.TemporaryDirectory() as d:
        cpp, exe = os.path.join(d, "f.cpp"), os.path.join(d, "f")
        open(cpp, "w").write(prog)
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(root, "oracle", "shim"), "-I", src, "-I",
                            os.path.join(root, "include"), "-I", os.path.join(root, "alicevision_b200", "adaptor"), cpp, "-o", exe],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        got = np.array([float(x) for x in subprocess.run([exe], capture_output=True, text=True).stdout.split()])
    E = np.array([[0.0, -1, 0.2], [1, 0, -0.3], [-0.1, 0.4, 0]])
    want = matching.fundamentalFromEssential(E, np.array([[700, 0, 320], [0, 700, 240], [0, 0, 1.0]]),
                                             np.array([[770, 0.5, 300], [0, 760, 250], [0, 0, 1.0]]))
    assert np.array_equal(got, want.ravel())


# ---------------------------------------------------------------------------------------------- GPU: the filter stage
def _calibrated_ring(n_views=5, n_points=900, fresh=300, seed=4):
    """A camera moving along a short arc and looking at a cloud of points: SIFT uchar descriptors of the visible points with per-view
    noise plus fresh features; one shared pinhole K."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, (n_points, 3)) + [0, 0, 8]
    sift = synth.sift_images(1, n_points, np.uint8, seed=seed, pool_factor=1.0)[0][0]
    K = np.array([[1500.0, 0, 960], [0, 1500.0, 540], [0, 0, 1]])
    regions, sizes, intr = {}, {}, {}
    for v in range(n_views):
        a = (v - n_views / 2) * 0.04
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        c = np.array([v * 0.3, 0.02 * v, 0])
        x = ((X - c) @ R.T) @ K.T
        xy = x[:, :2] / x[:, 2:] + rng.normal(0, 0.4, (n_points, 2))
        vis = np.flatnonzero((x[:, 2] > 0) & (xy[:, 0] > 0) & (xy[:, 0] < 1920) & (xy[:, 1] > 0) & (xy[:, 1] < 1080))
        d = np.clip(sift[vis].astype(np.int32) + rng.integers(-6, 7, (vis.size, 128)), 0, 255).astype(np.uint8)
        fd = synth.sift_images(1, fresh, np.uint8, seed=seed * 100 + v, pool_factor=1.0)[0][0]
        fxy = np.stack([rng.uniform(0, 1920, fresh), rng.uniform(0, 1080, fresh)], 1)
        perm = rng.permutation(vis.size + fresh)
        regions[v] = {"sift": matching.Regions(np.concatenate([d, fd])[perm], np.concatenate([xy[vis], fxy]).astype(np.float32)[perm])}
        sizes[v] = (1920, 1080)
        intr[v] = K
    return regions, sizes, intr


@pytest.fixture(scope="module")
def ring():
    regions, sizes, intr = _calibrated_ring()
    pairs = [(i, j) for i in range(5) for j in range(i + 1, 5)]
    ctx = matching.Context(0)
    views = {v: (r["sift"].descriptors, r["sift"].positions) for v, r in regions.items()}
    m = matching.ImageCollectionMatcherB200(0.8, False, matching.EMatcherType.BRUTE_FORCE_L2_B200, ctx).Match(views, pairs)
    put = {p: ({"sift": np.asarray(m[p]).copy()} if p in m and len(m[p]) else {}) for p in pairs}
    yield regions, sizes, intr, pairs, put, ctx
    ctx.close()


def _corr(regions, put, p):
    m = put[p].get("sift")
    if m is None:
        return np.zeros((0, 4))
    return np.concatenate([regions[p[0]]["sift"].positions[m["i"]], regions[p[1]]["sift"].positions[m["j"]]], 1).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("guided", [False, True])
def test_gpu_robust_model_estimation_E_AC(ring, guided):
    """Every estimate equals the oracle port's; kept lists are the strong-support inliers; guided lists equal the guided-matching oracle
    fed the same F = K_J^-T E K_I^-1, errorTh = error_max^2 and distRatio^2."""
    regions, sizes, intr, pairs, put, ctx = ring
    port = acre.AcransacEOracle("port")
    st = matching.mt19937_state(5489)
    out, info = matching.robustModelEstimation_E_AC(put, regions, sizes, intr, st, maxIteration=4000, guidedMatching=guided,
                                                    distanceRatio=0.6, ctx=ctx)
    n_valid = 0
    for p in pairs:
        c = _corr(regions, put, p)
        if not put[p]:
            assert not info[p]["valid"]
            continue
        want = port.estimate(c, (intr[p[0]], intr[p[1]]), sizes[p[1]], st, 4000)
        assert info[p]["valid"] == bool(want["valid"]), p
        assert np.array_equal(info[p]["E"], want["E"]) and info[p]["error_max"] == float(want["error_max"]), p
        n_valid += info[p]["valid"]
        if not info[p]["valid"]:
            continue
        inl = matching.copyInlierMatches(want["inliers"], put[p], ["sift"])
        assert (p in out) == matching.hasStrongSupport(inl, 5), p
        if p not in out:
            continue
        if not guided:
            assert np.array_equal(out[p]["sift"], inl["sift"]), p
        else:
            F = matching.fundamentalFromEssential(info[p]["E"], intr[p[0]], intr[p[1]])
            r0, r1 = regions[p[0]]["sift"], regions[p[1]]["sift"]
            w = gfo.best().guided_match(r0.descriptors, r0.positions.astype(np.float64), r1.descriptors, r1.positions.astype(np.float64), F,
                                        info[p]["error_max"] ** 2, 0.36, model=matching.MODEL_FUNDAMENTAL)
            g = out[p]["sift"]
            assert np.array_equal(g["i"], w["i"]) and np.array_equal(g["j"], w["j"]), p
    assert n_valid >= 4 and len(out) >= 4
    kept = matching.removePoorlyOverlappingImagePairs(out, put)
    assert set(kept) <= set(out)


@pytest.mark.gpu
def test_gpu_chain_replays_the_reference(ring):
    """chain=True: each pair starts where the previous estimated pair left the generator, as the reference's single-threaded filter."""
    regions, sizes, intr, pairs, put, ctx = ring
    port = acre.AcransacEOracle("port")
    st = matching.mt19937_state(77)
    _, info = matching.robustModelEstimation_E_AC(put, regions, sizes, intr, st, maxIteration=3000, chain=True, ctx=ctx)
    for p in pairs:
        if not put[p]:
            continue
        want = port.estimate(_corr(regions, put, p), (intr[p[0]], intr[p[1]]), sizes[p[1]], st, 3000)
        assert info[p]["valid"] == bool(want["valid"]) and np.array_equal(info[p]["E"], want["E"]), p
        assert np.array_equal(info[p]["mt_state_out"], want["mt_state_out"]), p
        st = want["mt_state_out"]


@pytest.mark.gpu
def test_essential_filter_cpp_adaptor():
    """The C++ batch adaptor (GeometricFilterMatrix_E_AC_Batch_b200) against the "ref" oracles in one executable."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "essential_filter_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "essential_filter adaptor ok" in r.stdout
