"""GPU parity tests (run with -m gpu on an H100).  Every comparison goes through the C ABI
(alicevision_b200.matching binds include/b200match.h with ctypes) and checks the CUDA path against the
oracle: match index pairs bit-exact, distances exact on integer-valued data and exact by construction on
real-valued data (the exact path follows the reference's summation order; tolerance 1e-4 relative is the
north-star bound, asserted as equality here and relaxed only if equality fails)."""
import os

import numpy as np
import pytest

import oracle
from alicevision_b200 import (ArrayMatcherB200, EMatcherType, ImageCollectionMatcherB200, matching, synth)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "reference_small.npz")


def assert_same(got, want, rtol=0.0):
    assert sorted(got) == sorted(want), (sorted(got)[:5], sorted(want)[:5])
    for k in want:
        g, w = got[k], want[k]
        assert len(g) == len(w), (k, len(g), len(w))
        assert np.array_equal(g["i"], w["i"]) and np.array_equal(g["j"], w["j"]), f"index pairs differ for {k}"
        if rtol == 0.0:
            assert np.array_equal(g["dist"], w["dist"]) and np.array_equal(g["ratio"], w["ratio"]), f"distances differ for {k}"
        else:
            assert np.allclose(g["dist"], w["dist"], rtol=rtol, atol=0) and np.allclose(g["ratio"], w["ratio"], rtol=rtol, atol=0)


def run(ds, xys, pairs, hamming=False, cross=False, ratio=0.8, force_exact=False, variant=4):
    t = EMatcherType.BRUTE_FORCE_HAMMING_B200 if hamming else EMatcherType.BRUTE_FORCE_L2_B200
    m = ImageCollectionMatcherB200(ratio, cross, t)
    m.clear()
    m.ctx.set_force_exact(force_exact)
    m.ctx.set_tc_variant(variant)
    try:
        return m.Match({i: (ds[i], xys[i]) for i in range(len(ds))}, pairs), m
    finally:
        m.ctx.set_force_exact(False)
        m.ctx.set_tc_variant(4)


# ---------------------------------------------------------------------------------------------- Surface 1
def test_arraymatcher_known_answers():
    """matching/matching_test.cpp:22-89,128-140 ported onto ArrayMatcherB200."""
    m = ArrayMatcherB200()
    assert m.Build(np.array([[0], [1], [2], [3], [4]], np.float32))
    ok, i, d = m.SearchNeighbour(np.array([2], np.float32))
    assert ok and i == 2 and abs(d) < 1e-8
    assert m.Build(np.array([[0], [1], [2], [5], [6]], np.float32))
    ok, idx, dist = m.SearchNeighbours(np.array([[2]], np.float32), 1, 5)
    assert ok and idx.tolist() == [[2, 1, 0, 3, 4]] and dist.tolist() == [[0, 1, 4, 9, 16]]
    assert m.Build(np.arange(12, dtype=np.float32).reshape(3, 4))
    ok, i, d = m.SearchNeighbour(np.array([4, 5, 6, 7], np.float32))
    assert ok and i == 1 and abs(d) < 1e-8
    e = ArrayMatcherB200()
    assert not e.Build(np.zeros((0, 4), np.float32))
    assert not e.SearchNeighbour(np.zeros(4, np.float32))[0]
    assert m.Build(np.ones((1, 4), np.float32)) and not m.SearchNeighbours(np.zeros((1, 4), np.float32), 1, 2)[0]   # NN > rows


@pytest.mark.parametrize("kind", ["u8", "f32", "real", "bin"])
def test_arraymatcher_top2_vs_oracle(ora, kind):
    if kind == "bin":
        ds, _ = synth.mldb_images(2, 1500, seed=21)
        m = ArrayMatcherB200(binary=True)
        metric = "hamming"
    else:
        ds, _ = synth.sift_images(2, 1500, np.uint8, seed=21, pool_factor=1.0)
        ds = {"u8": ds, "f32": [d.astype(np.float32) for d in ds], "real": synth.real_valued(ds)}[kind]
        m = ArrayMatcherB200(matching.L2_VECTORIZED)
        metric = "l2_vectorized"
    assert m.Build(ds[0])
    ok, idx, dist = m.SearchNeighbours(ds[1], NN=2)
    okr, ridx, rdist = ora.knn(ds[0], ds[1], 2, metric=metric)
    assert ok and okr and np.array_equal(dist, rdist)
    strict = rdist[:, 0] < rdist[:, 1]
    assert np.array_equal(idx[strict, 0], ridx[strict, 0])          # ties are unspecified in the reference (matching_test.cpp:46)
    # general NN through the generic kernel
    ok, idx5, dist5 = m.SearchNeighbours(ds[1][:64], NN=5)
    okr, ridx5, rdist5 = ora.knn(ds[0], ds[1][:64], 5, metric=metric)
    assert ok and np.array_equal(dist5, rdist5)


# ---------------------------------------------------------------------------------------------- Surface 2
def test_golden_fixtures_gpu():
    g = np.load(GOLD)
    pairs = g["pairs"]
    cases = [("u8", list(g["sift_u8"]), list(g["xy"]), False), ("f32", [d.astype(np.float32) for d in g["sift_u8"]], list(g["xy"]), False),
             ("real", list(g["sift_real"]), list(g["xy"]), False), ("bin", list(g["mldb"]), list(g["mldb_xy"]), True),
             ("adv", list(g["sift_u8"]), list(g["adv_xy"]), False)]
    for name, ds, xy, ham in cases:
        for cross in ((False, True) if name in ("u8", "f32", "real") else (False,)):
            got, m = run(ds, xy, pairs, ham, cross)
            gp, go, gm = g[f"{name}_cross{int(cross)}_pairs"], g[f"{name}_cross{int(cross)}_off"], g[f"{name}_cross{int(cross)}_matches"]
            want = {(int(p[0]), int(p[1])): gm[go[k]:go[k + 1]].view(oracle.MATCH_DTYPE) for k, p in enumerate(gp)}
            assert_same(got, want)
            if name in ("u8", "f32", "adv"):
                assert m.ctx.last_tc_pairs() > 0 and m.ctx.exactness_errors() == 0


@pytest.mark.parametrize("variant", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("cross", [False, True])
def test_collection_tensorcore_vs_oracle(ora, dtype, cross, variant):
    """Config-2 shape, down-scaled: ragged feature counts (not multiples of 128 / 256), TC path."""
    descs, xys = synth.sift_images(5, 1400, dtype, seed=31, pool_factor=1.0)
    cut = [1400, 1111, 257, 640, 129]
    descs = [d[:c] for d, c in zip(descs, cut)]; xys = [x[:c] for x, c in zip(xys, cut)]
    pairs = synth.exhaustive_pairs(5)
    got, m = run(descs, xys, pairs, cross=cross, variant=variant)
    assert m.ctx.last_tc_pairs() == len(pairs) * (2 if cross else 1) and m.ctx.exactness_errors() == 0
    assert_same(got, ora.collection_match(descs, xys, pairs, 0.8, cross))
    # the exact CUDA-core path must agree too
    got2, m2 = run(descs, xys, pairs, cross=cross, force_exact=True)
    assert m2.ctx.last_tc_pairs() == 0
    assert_same(got2, got)


def test_collection_real_valued_exact_path(ora):
    """Real-valued fp32 on the exact CUDA-core kernel (force_exact), and on the default path (tensor-core filter since round 2)."""
    descs, xys = synth.sift_images(3, 900, np.uint8, seed=41, pool_factor=1.0)
    real = synth.real_valued(descs)
    pairs = synth.exhaustive_pairs(3)
    want = ora.collection_match(real, xys, pairs, 0.8)
    got, m = run(real, xys, pairs, force_exact=True)
    assert m.ctx.last_tc_pairs() == 0 and m.ctx.last_real_tc_pairs() == 0
    assert_same(got, want)
    got, m = run(real, xys, pairs)
    assert m.ctx.last_tc_pairs() == 0 and m.ctx.last_real_tc_pairs() == len(pairs) and m.ctx.exactness_errors() == 0
    assert_same(got, want)


def test_collection_extreme_values_fall_back_to_exact(ora):
    """uchar descriptors with ||v||^2 >= 2^22 are outside the tensor-core exactness domain."""
    rng = np.random.default_rng(5)
    d = [rng.integers(150, 256, (300, 128)).astype(np.uint8) for _ in range(2)]
    d[1][:100] = np.clip(d[0][:100].astype(np.int16) + rng.integers(-3, 4, (100, 128)), 0, 255).astype(np.uint8)
    xys = [synth.positions(300, rng) for _ in range(2)]
    got, m = run(d, xys, [(0, 1)])
    assert m.ctx.last_tc_pairs() == 0
    assert_same(got, ora.collection_match(d, xys, [(0, 1)], 0.8))


def test_collection_hamming_vs_oracle(ora):
    bd, bxy = synth.mldb_images(4, 1300, seed=51)
    bd = [bd[0], bd[1][:700], bd[2][:257], bd[3]]; bxy = [bxy[0], bxy[1][:700], bxy[2][:257], bxy[3]]
    pairs = synth.exhaustive_pairs(4)
    for cross in (False, True):
        got, _ = run(bd, bxy, pairs, hamming=True, cross=cross)
        assert_same(got, ora.collection_match(bd, bxy, pairs, 0.8, cross, True))


def test_edge_cases(ora):
    """Empty views, single-row database (NN=2 > rows), duplicated pair entries, unsorted pair list, tiny views."""
    descs, xys = synth.sift_images(4, 300, np.uint8, seed=61, pool_factor=1.0)
    descs = [descs[0], np.zeros((0, 128), np.uint8), descs[2][:1], descs[3][:5]]
    xys = [xys[0], np.zeros((0, 2), np.float32), xys[2][:1], xys[3][:5]]
    pairs = [(2, 3), (0, 1), (0, 3), (0, 2), (1, 2), (0, 3), (2, 0), (3, 0)]
    got, _ = run(descs, xys, pairs)
    assert_same(got, ora.collection_match(descs, xys, pairs, 0.8))
    m = ImageCollectionMatcherB200()
    with pytest.raises(matching.B200MatchError):
        m.match_uploaded([(0, 99)])                      # unknown view: the reference throws std::out_of_range
    out = {(7, 8): "kept"}
    m.Match({0: (descs[0], xys[0]), 3: (descs[3], xys[3])}, [(0, 3)], out)   # appends, does not clear
    assert out[(7, 8)] == "kept"


def test_adversarial_positions(ora):
    """Duplicated / colliding feature positions: the coordinate de-duplication is order-dependent (App. B)."""
    descs, xys = synth.sift_images(3, 800, np.uint8, seed=71, pool_factor=1.0, generic_positions=False)
    pairs = synth.exhaustive_pairs(3)
    got, _ = run(descs, xys, pairs)
    assert_same(got, ora.collection_match(descs, xys, pairs, 0.8))


def test_ratio_values(ora):
    descs, xys = synth.sift_images(2, 600, np.uint8, seed=81, pool_factor=1.0)
    for r in (0.6, 0.95, 1.0):
        got, _ = run(descs, xys, [(0, 1)], ratio=r)
        assert_same(got, ora.collection_match(descs, xys, [(0, 1)], r))


@pytest.mark.parametrize("variant", [1, 2, 3, 4])
def test_full_size_properties(variant):
    """BASELINE config sizes (8192 features): size-independent properties instead of the (slow) oracle.
    1. self-match: every feature's nearest neighbour in its own image is itself (d = 0) -> after the ratio test
       (0 < r^2*d2 whenever d2 > 0) and de-duplication the match list is the identity on features with d2 > 0.
    2. tensor-core result == exact CUDA-core result, bit for bit.
    3. planted correspondences are recovered."""
    m = 8192
    descs, xys = synth.sift_images(3, m, np.uint8, seed=91, pool_factor=1.0)
    got, mm = run(descs, xys, [(0, 0), (0, 1), (1, 2)], variant=variant)
    assert mm.ctx.exactness_errors() == 0 and mm.ctx.last_tc_pairs() == 3
    s = got[(0, 0)]
    assert np.array_equal(s["i"], s["j"]) and np.all(s["dist"] == 0) and len(s) > 0.9 * m
    got_exact, _ = run(descs, xys, [(0, 0), (0, 1), (1, 2)], force_exact=True)
    assert_same(got_exact, got)
    assert len(got[(0, 1)]) > 0.05 * m


def test_raw_stage_is_superset_of_full(ora):
    descs, xys = synth.sift_images(2, 700, np.uint8, seed=95, pool_factor=1.0)
    m = ImageCollectionMatcherB200()
    m.clear()
    m.upload({0: (descs[0], xys[0]), 1: (descs[1], xys[1])})
    _, off, raw = m.match_uploaded([(0, 1)], matching.STAGE_RAW)
    _, off2, full = m.match_uploaded([(0, 1)], matching.STAGE_FULL)
    rawset = {(int(a), int(b)) for a, b in zip(raw["i"], raw["j"])}
    assert all((int(a), int(b)) in rawset for a, b in zip(full["i"], full["j"]))
    _, off3, none = m.match_uploaded([(0, 1)], matching.STAGE_DEVICE)
    assert len(none) == 0 and m.ctx.last_records() == len(raw)


def test_cpp_adaptors_against_reference_classes():
    """oracle/_ref/adaptor_test: the header-only C++ adaptors (deriving from the reference's ArrayMatcher /
    IImageCollectionMatcher) vs the reference classes themselves, compiled together by oracle.build() from an AliceVision source tree."""
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(__file__)), "oracle", "_ref", "adaptor_test")
    if not os.path.exists(exe):
        pytest.skip("adaptor_test not built (oracle.build() needs the AliceVision source tree)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ADAPTOR TEST PASSED" in r.stdout, r.stdout + r.stderr


def test_reupload_replaces_view_and_bulk_upload_edge_cases(ora):
    """b200m_upload_views: replacing an uploaded view (no clear), empty views inside a bulk call, views without positions."""
    descs, xys = synth.sift_images(3, 520, np.uint8, seed=101, pool_factor=1.0)
    m = ImageCollectionMatcherB200()
    m.clear()
    m.upload({0: (descs[0], xys[0]), 1: (descs[1], xys[1]), 2: (np.zeros((0, 128), np.uint8), np.zeros((0, 2), np.float32))})
    first = m.Match({}, [(0, 1), (0, 2)])
    assert_same(first, ora.collection_match([descs[0], descs[1], descs[2][:0]], [xys[0], xys[1], xys[2][:0]], [(0, 1), (0, 2)], 0.8))
    m.upload({1: (descs[2], xys[2])})                       # replace view 1 in place
    second = m.Match({}, [(0, 1)])
    assert_same(second, ora.collection_match([descs[0], descs[2]], [xys[0], xys[2]], [(0, 1)], 0.8))
    m.upload({5: (descs[1], None)})                         # no positions: fine for RAW, an error for FULL
    _, off, raw = m.match_uploaded([(0, 5)], matching.STAGE_RAW)
    assert len(raw) > 0
    with pytest.raises(matching.B200MatchError):
        m.match_uploaded([(0, 5)], matching.STAGE_FULL)


# ---------------------------------------------------------------------------------------------- Surface 1b
@pytest.mark.parametrize("kind", ["u8", "f32", "real", "bin"])
def test_regions_matcher_vs_oracle(ora, kind):
    """IRegionsMatcher / RegionsDatabaseMatcher / DistanceRatioMatch mirrors (matching/RegionsMatcher.hpp:49-78,183-220,
    RegionsMatcher.cpp:19-52): one database, several queries, against RegionsMatcher::Match of the oracle."""
    from alicevision_b200 import DistanceRatioMatch, Regions, RegionsDatabaseMatcherB200, createRegionsMatcher
    hamming = kind == "bin"
    if hamming:
        descs, xys = synth.mldb_images(3, 777, seed=31)
    else:
        descs, xys = synth.sift_images(3, 777, np.uint8 if kind == "u8" else np.float32, seed=31, pool_factor=1.0)
        if kind == "real":
            descs = synth.real_valued(descs)
    t = EMatcherType.BRUTE_FORCE_HAMMING_B200 if hamming else EMatcherType.BRUTE_FORCE_L2_B200
    regs = [Regions(d, x, binary=hamming) for d, x in zip(descs, xys)]
    db = RegionsDatabaseMatcherB200(t, regs[0])
    assert db.getDatabaseRegions() is regs[0]
    for q in (1, 2, 1):                       # the database stays resident across queries
        ok, got = db.Match(0.8, regs[q])
        ok_want, want = ora.regions_match(descs[0], xys[0], descs[q], xys[q], 0.8, hamming)
        assert ok == ok_want and len(want) > 0
        assert_same({0: got}, {0: want})
    got = DistanceRatioMatch(0.6, t, regs[1], regs[2])
    assert_same({0: got}, {0: ora.regions_match(descs[1], xys[1], descs[2], xys[2], 0.6, hamming)[1]})
    # factory validity rules (RegionsMatcher.cpp:61-64) and the empty cases (RegionsMatcher.cpp:32-38, RegionsMatcher.hpp:109-110)
    wrong = EMatcherType.BRUTE_FORCE_L2_B200 if hamming else EMatcherType.BRUTE_FORCE_HAMMING_B200
    assert createRegionsMatcher(regs[0], wrong) is None
    assert createRegionsMatcher(regs[0], EMatcherType.ANN_L2) is None
    ok, got = RegionsDatabaseMatcherB200(wrong, regs[0]).Match(0.8, regs[1])
    assert not ok and len(got) == 0
    empty = Regions(descs[0][:0], xys[0][:0], binary=hamming)
    ok, got = db.Match(0.8, empty)
    assert not ok and len(got) == 0
    ok, got = RegionsDatabaseMatcherB200(t, empty).Match(0.8, regs[1])
    assert not ok and len(got) == 0
    one = Regions(descs[0][:1], xys[0][:1], binary=hamming)       # NN = 2 > rows: SearchNeighbours false (bruteForce.hpp:105)
    ok, got = RegionsDatabaseMatcherB200(t, one).Match(0.8, regs[1])
    assert not ok and len(got) == 0


@pytest.mark.parametrize("cross", [False, True])
def test_async_upload_overlaps_and_keeps_pairset_order(ora, cross):
    """b200m_upload_views_async + b200m_match_pairs: the pair list is processed in order of view arrival (several short
    batches while copies are in flight) but reported in PairSet order with the reference's results; a second call on the
    now-resident views (natural order, one batch) returns the same lists."""
    n = 13
    descs, xys = synth.sift_images(n, 640, np.uint8, seed=77, pool_factor=1.0)
    descs[5] = descs[5][:0]; xys[5] = xys[5][:0]                       # an empty view in the middle of the upload
    pairs = synth.exhaustive_pairs(n)[::-1]                            # given in reverse: PairSet semantics sort them
    m = ImageCollectionMatcherB200(0.8, cross)
    m.clear()
    views = {i: (descs[i], xys[i]) for i in range(n)}
    m.upload({i: v for i, v in views.items() if i % 2 == 1}); m.upload({i: v for i, v in views.items() if i % 2 == 0})   # two jobs
    pid, off, mat = m.match_uploaded(pairs)
    assert [tuple(p) for p in pid.tolist()] == sorted(map(tuple, pairs.tolist()))
    got = {(int(a), int(b)): mat[off[k]:off[k + 1]] for k, (a, b) in enumerate(pid) if off[k + 1] > off[k]}
    want = ora.collection_match(descs, xys, pairs, 0.8, cross=cross)
    assert_same(got, want)
    pid2, off2, mat2 = m.match_uploaded(pairs)
    assert np.array_equal(pid, pid2) and np.array_equal(off, off2) and np.array_equal(mat, mat2)
    m.clear()


# ---------------------------------------------------------------------------------------------- single-process multi-device
@pytest.mark.parametrize("cross", [False, True])
def test_multi_device_single_process(ora, cross):
    """b200m_multi_match: the pair list sharded over several engine contexts inside one process, merged in PairSet order.
    Uses every visible GPU, and at least two contexts (both on device 0 when the box has one GPU)."""
    import torch
    ndev = max(1, torch.cuda.device_count())
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    n = 9
    descs, xys = synth.sift_images(n, 700, np.uint8, seed=55, pool_factor=1.0)
    descs[3] = descs[3][:0]; xys[3] = xys[3][:0]
    pairs = np.concatenate([synth.exhaustive_pairs(n), [[7, 2], [8, 0]]])        # includes I > J pairs, kept as given (PairSet semantics)
    m = ImageCollectionMatcherB200(0.8, cross, EMatcherType.BRUTE_FORCE_L2_B200, devices=devices)
    got = m.Match({i: (descs[i], xys[i]) for i in range(n)}, pairs)
    want = ora.collection_match(descs, xys, pairs, 0.8, cross=cross)
    assert_same(got, want)
    assert list(got) == sorted(got)                    # merged in PairSet order
    assert m.multi.exactness_errors() == 0
    got2 = m.Match({i: (descs[i], xys[i]) for i in range(n)}, pairs)      # contexts are reused by the next call
    assert_same(got2, want)
    m.multi.close()
    # more contexts than database images: some shards are empty
    m3 = ImageCollectionMatcherB200(0.8, cross, EMatcherType.BRUTE_FORCE_L2_B200, devices=(devices + [devices[0]])[:3] if len(devices) >= 3 else [0, 0, 0])
    few = [(0, 1), (0, 2), (0, 4)]
    assert_same(m3.Match({i: (descs[i], xys[i]) for i in range(n)}, few), ora.collection_match(descs, xys, few, 0.8, cross=cross))
    assert m3.Match({i: (descs[i], xys[i]) for i in range(n)}, np.zeros((0, 2), np.uint32)) == {}
    m3.multi.close()


# ---------------------------------------------------------------------------------------------- more full-size properties
def test_full_size_cross_matching_is_symmetric():
    """BASELINE config size (8192): with cross matching the kept correspondences of (I, J) are the transposed kept
    correspondences of (J, I) (a match survives iff it is a ratio-test match in both directions,
    ImageCollectionMatcher_generic.cpp:83-111) - as long as no coordinate de-duplication removes one side, which the
    generic synthetic positions guarantee only for the left image, so the property is checked on the (i, j) SETS of
    the raw mutual matches: cross(I,J) subset of fwd(I,J), and {(i,j)} == {(j,i) of cross(J,I)} for features matched once."""
    m = 8192
    descs, xys = synth.sift_images(2, m, np.uint8, seed=92, pool_factor=1.0)
    fwd, _ = run(descs, xys, [(0, 1), (1, 0)], cross=False)
    crs, mm = run(descs, xys, [(0, 1), (1, 0)], cross=True)
    assert mm.ctx.exactness_errors() == 0
    f01 = set(zip(fwd[(0, 1)]["i"].tolist(), fwd[(0, 1)]["j"].tolist())); f10 = set(zip(fwd[(1, 0)]["i"].tolist(), fwd[(1, 0)]["j"].tolist()))
    c01 = set(zip(crs[(0, 1)]["i"].tolist(), crs[(0, 1)]["j"].tolist())); c10 = set(zip(crs[(1, 0)]["i"].tolist(), crs[(1, 0)]["j"].tolist()))
    assert c01 <= f01 and c10 <= f10 and len(c01) > 0.03 * m
    assert c01 == {(i, j) for (i, j) in f01 if (j, i) in f10}
    assert c10 == {(i, j) for (i, j) in f10 if (j, i) in f01}
    assert c01 == {(j, i) for (i, j) in c10}


def test_full_size_hamming_properties():
    """BASELINE configs[3] size (16384 MLDB features): self-match identity, planted correspondences, and a numpy popcount
    check of the two smallest distances for a sample of queries."""
    m = 16384
    descs, xys = synth.mldb_images(2, m, seed=93)
    got, _ = run(descs, xys, [(0, 0), (0, 1)], hamming=True)
    s = got[(0, 0)]
    assert np.array_equal(s["i"], s["j"]) and np.all(s["dist"] == 0) and len(s) > 0.9 * m and np.all(s["ratio"] == 0)
    g = got[(0, 1)]
    assert len(g) > 0.05 * m
    rng = np.random.default_rng(3)
    pick = rng.choice(len(g), 48, replace=False)
    lut = np.array([bin(v).count("1") for v in range(256)], np.uint16)
    for k in pick:
        i, j = int(g["i"][k]), int(g["j"][k])
        d = lut[np.bitwise_xor(descs[0], descs[1][j][None, :])].sum(axis=1)
        o = np.argsort(d, kind="stable")
        assert o[0] == i and d[o[0]] == g["dist"][k] and np.float32(d[o[0]]) < np.float32(0.8) * np.float32(d[o[1]])
    # queries the kernel rejected really fail the ratio test
    rejected = np.setdiff1d(np.arange(m), g["j"])[:24]
    for j in rejected:
        d = np.sort(lut[np.bitwise_xor(descs[0], descs[1][j][None, :])].sum(axis=1))
        assert not (np.float32(d[0]) < np.float32(0.8) * np.float32(d[1]))


def test_largest_sweep_size_32k():
    """BASELINE configs[4] upper end (32768 features/image): tensor-core result == exact CUDA-core result bit for bit."""
    m = 32768
    descs, xys = synth.sift_images(2, m, np.uint8, seed=94, pool_factor=1.0)
    got, mm = run(descs, xys, [(0, 1)])
    assert mm.ctx.exactness_errors() == 0 and mm.ctx.last_tc_pairs() == 1 and len(got[(0, 1)]) > 0.03 * m
    got_exact, _ = run(descs, xys, [(0, 1)], force_exact=True)
    assert_same(got_exact, got)


def test_shared_context_from_several_host_threads(ora):
    """One engine context used by several host threads at once (IRegionsMatcher adaptors built inside an OpenMP region share
    b200detail::sharedContext()): calls serialise on the context's lock and every thread gets the reference's result."""
    import threading
    from alicevision_b200 import Regions, RegionsMatcherB200
    descs, xys = synth.sift_images(5, 600, np.uint8, seed=61, pool_factor=1.0)
    regs = [Regions(d, x) for d, x in zip(descs, xys)]
    want = {(a, b): ora.regions_match(descs[a], xys[a], descs[b], xys[b], 0.8, False)[1] for a in range(5) for b in range(5) if a != b}
    errors = []

    def worker(a):
        try:
            db = RegionsMatcherB200(regs[a])
            for rep in range(2):
                for b in range(5):
                    if b != a:
                        ok, got = db.Match(0.8, regs[b])
                        assert_same({0: got}, {0: want[(a, b)]})
            db.close()
        except Exception as e:      # noqa: BLE001
            errors.append((a, repr(e)))

    th = [threading.Thread(target=worker, args=(a,)) for a in range(5)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


# ---------------------------------------------------------------------------------------------- ties / degenerate descriptors on the tensor-core path
def test_tensorcore_path_with_massive_ties(ora):
    """Tiny alphabets make most distances equal (whole 16-row chunks tie, best == second best for most queries): the chunk-minimum
    logic of the tensor-core kernel and its exactness pass must still give the reference's lists (a tie never passes d1 < r^2 d2,
    so the surviving index is unique, SURVEY Appendix A.4)."""
    rng = np.random.default_rng(5)
    n, m = 3, 1300
    descs = [rng.integers(0, 2, (m, 128)).astype(np.uint8) for _ in range(n)]
    for k in range(1, n):                                   # plant exact and near copies so that something passes the ratio test
        src = rng.permutation(m)[: m // 3]
        descs[k][: m // 3] = descs[0][src]
        descs[k][: m // 6, :3] ^= 1
    _, xys = synth.sift_images(n, m, np.uint8, seed=6, pool_factor=1.0)
    for ratio in (0.8, 0.99):
        got, mm = run(descs, xys, synth.exhaustive_pairs(n), ratio=ratio)
        assert mm.ctx.last_tc_pairs() == 3 and mm.ctx.exactness_errors() == 0
        assert_same(got, ora.collection_match(descs, xys, synth.exhaustive_pairs(n), ratio))
    got, _ = run(descs, xys, [(0, 0)])                       # duplicates inside one image: d1 == d2 == 0 never passes
    assert_same(got, ora.collection_match(descs, xys, [(0, 0)], 0.8))


def test_cctag_like_one_hot_descriptors(ora):
    """CCTAG_Regions are Scalar<uchar,128> with a single 255 at the marker id (feature/cctag/ImageDescriber_CCTAG.cpp:117-122) and go
    down the L2 uchar path: every distance is 0 or 2*255^2, so the kernel sees nothing but ties apart from the matching marker."""
    rng = np.random.default_rng(9)
    def markers(ids):
        d = np.zeros((len(ids), 128), np.uint8)
        d[np.arange(len(ids)), ids] = 255
        return d
    ids0 = rng.permutation(128)[:40]; ids1 = np.concatenate([rng.permutation(ids0)[:25], np.setdiff1d(np.arange(128), ids0)[:10]])
    ids2 = np.concatenate([ids0[:10], ids0[:10]])             # the same marker twice: d1 == d2 == 0 for it
    descs = [markers(ids0), markers(ids1), markers(ids2)]
    xys = [synth.positions(len(d), rng) for d in descs]
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0), (1, 2)]
    for cross in (False, True):
        got, mm = run(descs, xys, pairs, cross=cross)
        assert mm.ctx.exactness_errors() == 0
        want = ora.collection_match(descs, xys, pairs, 0.8, cross=cross)
        assert_same(got, want)
    assert len(got[(0, 1)]) == 25 if (0, 1) in got else True


# ---------------------------------------------------------------------------------------------- other descriptor lengths
@pytest.mark.parametrize("kind", ["akaze_float64", "liop_u8_144", "float_130"])
def test_other_descriptor_lengths_on_the_collection_surface(kind):
    """AKAZE_Float_Regions (float x 64) and AKAZE_Liop_Regions (uchar x 144) (feature/regionsFactory.hpp:25-27) go through
    createRegionsMatcher's BRUTE_FORCE_L2 cases like SIFT (RegionsMatcher.cpp:74-79,103-108): generic exact kernel, compared with the
    restated oracle (the compiled-reference oracle only instantiates the 128 / 64-byte Regions types).  A float length that is not a
    multiple of 4 makes L2_Vectorized<float> return 0 for every pair (feature/metric.hpp:118-122) -> no match survives."""
    P = oracle.Oracle("port")
    rng = np.random.default_rng(12)
    n, m = 3, 900
    dim = {"akaze_float64": 64, "liop_u8_144": 144, "float_130": 130}[kind]
    base = rng.gamma(2.0, 20.0, (m, dim))
    descs = []
    for k in range(n):
        d = base[rng.permutation(m)] + rng.normal(0, 2.5, (m, dim))
        d[m // 2:] = rng.gamma(2.0, 20.0, (m - m // 2, dim))
        descs.append(np.clip(d, 0, 255).astype(np.uint8) if kind == "liop_u8_144" else d.astype(np.float32))
    xys = [synth.positions(m, rng) for _ in range(n)]
    pairs = synth.exhaustive_pairs(n)
    for cross in (False, True):
        got, mm = run(descs, xys, pairs, cross=cross)
        want = P.collection_match(descs, xys, pairs, 0.8, cross=cross)
        assert mm.ctx.last_tc_pairs() == 0
        assert_same(got, want)
        if kind == "float_130":
            assert len(got) == 0
        else:
            assert len(got) == 3 and all(len(v) > 100 for v in got.values())
    from alicevision_b200 import Regions, RegionsDatabaseMatcherB200
    db = RegionsDatabaseMatcherB200(EMatcherType.BRUTE_FORCE_L2_B200, Regions(descs[0], xys[0]))
    ok, got1 = db.Match(0.8, Regions(descs[1], xys[1]))
    ok_w, want1 = P.regions_match(descs[0], xys[0], descs[1], xys[1], 0.8, False)
    assert ok == ok_w
    assert_same({0: got1}, {0: want1})


# ---------------------------------------------------------------------------------------------- round 2: staging / finishing variants
def _fresh_matcher(env: dict, hamming=False, cross=False):
    """An ImageCollectionMatcherB200 on its OWN engine context created under `env` (the context reads its switches at creation)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        ctx = matching.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    t = EMatcherType.BRUTE_FORCE_HAMMING_B200 if hamming else EMatcherType.BRUTE_FORCE_L2_B200
    return ImageCollectionMatcherB200(0.8, cross, t, ctx)


@pytest.mark.parametrize("kind", ["f32", "u8", "bin", "adv"])
def test_device_finishing_equals_host_finishing(ora, kind):
    """The finishing stage on the device (finish.cuh: general-position views) and the literal host stage give the reference's lists;
    views with colliding coordinates are left to the host by the device stage (flag from pos_rank_kernel)."""
    hamming = kind == "bin"
    if hamming:
        descs, xys = synth.mldb_images(4, 1100, seed=131)
    else:
        descs, xys = synth.sift_images(4, 1100, np.float32 if kind == "f32" else np.uint8, seed=131, pool_factor=1.0, generic_positions=kind != "adv")
    if kind == "f32":                 # one view in general position, one not, inside the same batch
        xys[2] = synth.positions(1100, np.random.default_rng(3), generic=False)
    cut = [1100, 901, 1100, 257]
    descs = [d[:c] for d, c in zip(descs, cut)]; xys = [x[:c] for x, c in zip(xys, cut)]
    pairs = [(0, 1), (1, 0), (2, 3), (3, 2), (0, 2), (2, 0), (1, 1)]
    views = {i: (descs[i], xys[i]) for i in range(4)}
    for cross in (False, True):
        want = ora.collection_match(descs, xys, pairs, 0.8, cross, hamming)
        for env in ({"B200M_DEVICE_FINISH": "1"}, {"B200M_DEVICE_FINISH": "0"}):
            m = _fresh_matcher(env, hamming, cross)
            assert_same(dict(m.Match(views, pairs)), want)
            m.ctx.close()


def test_u8_staging_of_integer_valued_fp32(ora):
    """Integer-valued fp32 descriptors are staged and stored as uchar (hostconv.hpp); with the staging switched off, and for a view
    whose first rows look integer but a later value is not (the probe passes, the checked conversion of a later chunk fails and the
    view is re-uploaded as fp32), the results are the reference's."""
    descs, xys = synth.sift_images(4, 1300, np.float32, seed=141, pool_factor=1.0)
    descs[2] = descs[2].copy(); descs[2][777, 5] += 0.25            # surprise far behind the probe
    descs[3] = synth.real_valued([descs[3]])[0]                      # real-valued from the first row
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0), (0, 3), (3, 1), (2, 3)]
    views = {i: (descs[i], xys[i]) for i in range(4)}
    want = ora.collection_match(descs, xys, pairs, 0.8)
    for env in ({"B200M_U8_STAGING": "1"}, {"B200M_U8_STAGING": "0"}, {"B200M_U8_STAGING": "1", "B200M_UP_CHUNK_MB": "1"}):
        m = _fresh_matcher(env)
        got = dict(m.Match(views, pairs))
        assert_same(got, want)
        assert m.ctx.last_tc_pairs() == 2 and m.ctx.exactness_errors() == 0     # (0,1), (1,0): both views integer-valued
        m.ctx.close()
    # guided matching between an integer-valued (stored as uchar) and a real-valued fp32 view: temporary fp32 expansion
    from alicevision_b200 import Regions, matching as mt
    F = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)
    got = mt.guidedMatching(F, Regions(descs[0], xys[0]), Regions(descs[3], xys[3]), 400.0, 0.81)
    want_g = ora.guided_match(descs[0], xys[0], descs[3], xys[3], F, 400.0, 0.81)
    assert np.array_equal(got["i"], want_g["i"]) and np.array_equal(got["j"], want_g["j"]) and len(got) > 0


def test_upload_rejects_duplicate_ids_and_survives():
    descs, xys = synth.sift_images(2, 300, np.uint8, seed=151, pool_factor=1.0)
    m = ImageCollectionMatcherB200()
    m.clear()
    import ctypes as C
    lib = m.ctx.lib
    ids = np.array([4, 4], np.uint32); counts = np.array([300, 300], np.int32)
    dptr = (C.c_void_p * 2)(descs[0].ctypes.data, descs[1].ctypes.data)
    rc = lib.b200m_upload_views_async(m.ctx._h, C.c_int(2), ids.ctypes.data_as(C.c_void_p), dptr, counts.ctypes.data_as(C.c_void_p), C.c_int(128), C.c_int(1), None)
    assert rc == 1 and b"twice" in lib.b200m_last_error()
    m.upload({0: (descs[0], xys[0]), 1: (descs[1], xys[1])})      # the context is still usable
    assert len(m.Match({}, [(0, 1)])) == 1


# ---------------------------------------------------------------------------------------------- round 2: real-valued fp32 on the tensor cores
def _real_images(n, m, seed, scale=1.0, sigma=0.37):
    descs, xys = synth.sift_images(n, m, np.float32, seed=seed, pool_factor=1.0)
    real = [np.ascontiguousarray((d * np.float32(scale)).astype(np.float32)) for d in synth.real_valued(descs, sigma=sigma)]
    return real, xys


@pytest.mark.parametrize("case", ["small", "ragged", "unit_norm", "mixed", "duplicates"])
def test_real_valued_tensorcore_filter_vs_oracle(ora, case):
    """Real-valued fp32 descriptors on the tensor-core FILTER kernel (MODE_REAL): fp16-rounded GEMM, rigorous error bound, exact
    re-scoring in the reference's SSE order (feature/metric.hpp:94-123), exact_rows fallback for the undecided queries - bit-identical
    to the oracle.  small / ragged: stand-alone re-scoring (short images); unit_norm: descriptors scaled by 1/512 (every bound is
    relative); mixed: integer-valued (stored as uchar) against real-valued views; duplicates: identical rows inside an image."""
    if case == "unit_norm":
        descs, xys = _real_images(3, 1500, 301, scale=1.0 / 512.0)
    else:
        descs, xys = _real_images(4 if case != "small" else 3, 1500 if case != "small" else 700, 302)
    if case == "ragged":
        cut = [1500, 1111, 257, 129]
        descs = [d[:c] for d, c in zip(descs, cut)]; xys = [x[:c] for x, c in zip(xys, cut)]
    if case == "mixed":
        descs[1] = np.ascontiguousarray(np.floor(descs[1]))          # integer-valued fp32 view: staged / stored as uchar
        descs[3] = np.ascontiguousarray(np.floor(descs[3]))
    if case == "duplicates":
        descs[0] = descs[0].copy(); descs[0][100:140] = descs[0][:40]    # d1 == d2 for their matches: never pass the ratio test
        descs[2] = descs[2].copy(); descs[2][:60] = descs[0][200:260]    # exact copies across images: d1 == 0
    n = len(descs)
    pairs = [(a, b) for a in range(n) for b in range(n) if a != b] + [(0, 0)]
    for cross in ((False, True) if case in ("small", "mixed") else (False,)):
        got, m = run(descs, xys, pairs, cross=cross)
        want = ora.collection_match(descs, xys, pairs, 0.8, cross)
        assert_same(got, want)
        n_int = sum(1 for a, b in pairs if case == "mixed" and a in (1, 3) and b in (1, 3)) * (2 if cross else 1)
        assert m.ctx.last_real_tc_pairs() == len(pairs) * (2 if cross else 1) - n_int and m.ctx.last_tc_pairs() == n_int
        assert m.ctx.exactness_errors() == 0                            # incl. the bound self-check of every re-scored candidate


def test_real_valued_full_size_fused_vs_oracle(ora):
    """8192 real-valued features per image: the re-scoring runs INSIDE the filter kernel (fused); every list equals the oracle's and the
    fallback handles only a small fraction of the queries.  The exact CUDA-core kernel (round-1 path, B200M_REAL_TC=0) agrees."""
    descs, xys = _real_images(3, 8192, 303)
    descs[2] = descs[2][:7003]; xys[2] = xys[2][:7003]
    pairs = [(0, 1), (1, 0), (2, 0), (1, 2), (1, 1)]
    got, m = run(descs, xys, pairs)
    want = ora.collection_match(descs, xys, pairs, 0.8)
    assert_same(got, want)
    assert m.ctx.last_real_tc_pairs() == len(pairs) and m.ctx.exactness_errors() == 0
    assert m.ctx.last_fallback_rows() < 0.01 * sum(len(descs[j]) for _, j in pairs), m.ctx.last_fallback_rows()
    mx = _fresh_matcher({"B200M_REAL_TC": "0"})
    got2 = dict(mx.Match({i: (descs[i], xys[i]) for i in range(3)}, pairs))
    assert mx.ctx.last_real_tc_pairs() == 0
    assert_same(got2, want)
    mx.ctx.close()


# ---------------------------------------------------------------------------------------------- round 2: Surface 1 on the tensor cores
@pytest.mark.parametrize("kind", ["u8", "f32"])
def test_arraymatcher_tensorcore_knn_8192(ora, kind):
    """ArrayMatcherB200.SearchNeighbours(NN = 2) on 128-D integer-valued descriptors runs the tcgen05 kernel (MODE_KNN) on the resident,
    prepared database: distances and both neighbours' indices against ArrayMatcher_bruteForce of the oracle, at 8192 x 8192 and ragged."""
    ds, _ = synth.sift_images(2, 8192, np.uint8, seed=311, pool_factor=1.0)
    if kind == "f32":
        ds = [d.astype(np.float32) for d in ds]
    for db, q in ((ds[0], ds[1]), (ds[0][:7001], ds[1][:333]), (ds[1][:17], ds[0][:4000])):
        m = ArrayMatcherB200(matching.L2_VECTORIZED)
        assert m.Build(db)
        for rep in range(2):                     # the second call reuses the scratch
            ok, idx, dist = m.SearchNeighbours(q, NN=2)
            assert ok and m.ctx.last_tc_pairs() == 1 and m.ctx.exactness_errors() == 0
        okr, ridx, rdist = ora.knn(db, q, 2, metric="l2_vectorized")
        assert okr and np.array_equal(dist, rdist)
        strict1 = rdist[:, 0] < rdist[:, 1]
        assert np.array_equal(idx[strict1, 0], ridx[strict1, 0])
        # second neighbour: unique whenever the third distance is larger; compare where the oracle's own second is unambiguous
        ok3, ridx3, rdist3 = ora.knn(db, q, 3, metric="l2_vectorized") if len(db) >= 3 else (False, None, None)
        if ok3:
            strict2 = strict1 & (rdist3[:, 1] < rdist3[:, 2])
            assert np.array_equal(idx[strict2, 1], ridx3[strict2, 1])
    # a real-valued query batch against an integer database falls back to the exact kernel, same answers as the oracle
    m = ArrayMatcherB200(matching.L2_VECTORIZED)
    if kind == "f32":
        assert m.Build(ds[0][:3000])
        qr = synth.real_valued([ds[1][:500]])[0]
        ok, idx, dist = m.SearchNeighbours(qr, NN=2)
        okr, ridx, rdist = ora.knn(ds[0][:3000], qr, 2, metric="l2_vectorized")
        assert ok and m.ctx.last_tc_pairs() == 0 and np.array_equal(dist, rdist)
