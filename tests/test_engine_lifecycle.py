"""Engine context lifecycle: the last-call record (b200m_last_*) describes the last matching or k-NN call and no earlier one, the
k-NN scratch grows and shrinks without changing a result, and a context can be created, used on every surface and destroyed
several times in one process."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from alicevision_b200 import ArrayMatcherB200, EMatcherType, ImageCollectionMatcherB200, matching, synth

pytestmark = pytest.mark.gpu

# x_R^T F x_L = 0 for a camera moving by t = (1000, 800, 1) (F = [t]x): the right epipole (1000, 800) lies inside a 2000 x 2000 image
F = np.array([[0, -1, 800], [1, 0, -1000], [-800, 1000, 0]], np.float64)
EPIPOLE = np.array([1000, 800, 1], np.float64)


def guided_match_model(ctx, left: int, right: int) -> int:
    """b200m_guided_match_model with F on two resident views, every right feature within the epipolar threshold; returns the match count."""
    res = C.c_void_p()
    matching._check(ctx.lib.b200m_guided_match_model(ctx._h, C.c_uint32(left), C.c_uint32(right), C.c_int(matching.MODEL_FUNDAMENTAL),
                                                     F.ctypes.data_as(C.c_void_p), C.c_double(1e12), C.c_double(0.64), C.byref(res)),
                    "b200m_guided_match_model")
    off = C.c_void_p()
    matching._check(ctx.lib.b200m_result_get(res, None, C.byref(off), None), "b200m_result_get")
    n = C.cast(off, C.POINTER(C.c_int64))[1]
    ctx.lib.b200m_result_free(res)
    return n


def same_knn(got, want) -> bool:
    """Equal distances, and equal first neighbours wherever the oracle's first is strictly closer than its second."""
    (ok, idx, dist), (okr, ridx, rdist) = got, want
    strict = rdist[:, 0] < rdist[:, 1]
    return ok and okr and np.array_equal(dist, rdist) and np.array_equal(idx[strict, 0], ridx[strict, 0])


def test_last_call_record_describes_the_last_call():
    descs, xys = synth.sift_images(2, 1500, np.uint8, seed=21, pool_factor=1.0)
    real = synth.real_valued(descs)
    ctx = matching.Context(0)
    am = ArrayMatcherB200(matching.L2_VECTORIZED, ctx)
    try:
        m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
        m.Match({v: (real[v], xys[v]) for v in range(2)}, [(0, 1)])
        assert ctx.last_real_tc_pairs() > 0 and ctx.last_records() > 0 and ctx.last_launches() > 0
        assert guided_match_model(ctx, 0, 1) > 0
        assert ctx.last_real_tc_pairs() == 0 and ctx.last_fallback_rows() == 0 and ctx.last_tc_pairs() == 0 and ctx.last_u8_tc_pairs() == 0
        assert ctx.last_records() > 0 and ctx.last_launches() > 0
        assert am.Build(descs[0])
        ok, _, _ = am.SearchNeighbours(descs[1], NN=2)
        assert ok and ctx.last_tc_pairs() == 1
        assert ctx.last_records() == 0 and ctx.last_real_tc_pairs() == 0 and ctx.last_launches() == 0 and ctx.last_gpu_ms() == 0
    finally:
        am._release()
        ctx.close()


def test_knn_scratch_grows_and_shrinks(ora):
    """One resident database, query batches that grow, shrink and grow again: the tensor-core path (integer-valued queries) and the
    exact path (real-valued queries, redone on the exact kernel after the tensor-core attempt) give the oracle's answers at every size."""
    ds, _ = synth.sift_images(2, 20000, np.uint8, seed=23, pool_factor=1.0)
    db = ds[0][:2000].astype(np.float32)
    queries = {"tc": ds[1].astype(np.float32), "exact": synth.real_valued([ds[1]])[0]}
    ctx = matching.Context(0)
    am = ArrayMatcherB200(matching.L2_VECTORIZED, ctx)
    try:
        assert am.Build(db)
        for path, q in queries.items():
            want = ora.knn(db, q, 2, metric="l2_vectorized")
            for n in (100, 5000, 300, 20000, 100):
                got = am.SearchNeighbours(q[:n], NN=2)
                assert ctx.last_tc_pairs() == (1 if path == "tc" else 0), (path, n)
                assert same_knn(got, (want[0], want[1][:n], want[2][:n])), (path, n)
            if path == "tc":
                assert ctx.exactness_errors() == 0     # the real-valued batches' tensor-core attempt does count (they are redone)
    finally:
        am._release()
        ctx.close()


def test_context_create_use_destroy(ora):
    """Three contexts in turn, each used once on every surface (upload + match, k-NN, guided matching from known poses, a-contrario
    RANSAC) and destroyed."""
    descs, xys = synth.sift_images(2, 1500, np.uint8, seed=29, pool_factor=1.0)
    pairs = [(0, 1)]
    want = ora.collection_match(descs, xys, pairs, ratio=0.8)
    want_knn = ora.knn(descs[0], descs[1], 2)
    corr = np.random.default_rng(5).uniform(0, 1000, (300, 4))
    for _ in range(3):
        ctx = matching.Context(0)
        am = ArrayMatcherB200(matching.L2_VECTORIZED, ctx)
        try:
            m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
            got = m.Match({v: (descs[v], xys[v]) for v in range(2)}, pairs)
            assert got.keys() == want.keys() and all(np.array_equal(got[k], want[k]) for k in want)
            assert am.Build(descs[0]) and same_knn(am.SearchNeighbours(descs[1], NN=2), want_knn)
            gf = ctx.guided_match_fast_pairs(pairs, [F], [EPIPOLE], [(2000, 2000)], 16.0, 0.64)
            assert list(gf) == pairs and ctx.last_launches() > 0
            acr = ctx.acransac_fundamental_pairs([corr], [(1000, 1000, 1000, 1000)], matching.mt19937_state(5489), 1000)
            assert len(acr) == 1 and acr[0]["iterations"] > 0
            assert ctx.exactness_errors() == 0
        finally:
            am._release()
            ctx.close()
