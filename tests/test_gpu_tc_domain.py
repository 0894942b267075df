"""The tensor-core search over its whole exactness domain (run with -m gpu on an H100).

The integer path (MODE_MATCH / MODE_KNN) is bit-exact for integer-valued rows with |v| <= 1024 and ||v||^2 < 2^22; the real-valued
filter (MODE_REAL) takes rows with |v| <= 1024, ||fp16(v)||^2 < 2^22 and at most REAL_MAX_ROWS = 131056 database rows.  The rest of the
suite only feeds it non-negative SIFT-like data; here it gets signed rows, magnitudes up to 1024, anti-correlated queries (whose distances
to every database row exceed those of an all-zero row, the padding of the last database tile), and every edge of the domain.

Integer-valued results are checked against an exact host reference (numpy, integer arithmetic) and, for representative cases, against the
oracle; real-valued results against the oracle, which follows the reference's SSE summation order.  Every test first asserts that the data
took the kernel it is meant to test (last_tc_pairs / last_real_tc_pairs), so that a silent fall-back to the exact kernel cannot pass it."""
import os

import numpy as np
import pytest

from alicevision_b200 import ArrayMatcherB200, EMatcherType, ImageCollectionMatcherB200, matching, synth

pytestmark = pytest.mark.gpu

NORM_LIMIT = 1 << 22          # ||v||^2 must stay below this (fp32-exact distances; three 11-bit half-norm limbs)
RANGE_LIMIT = 1024            # |v| <= 1024: 2v is exact in fp16
REAL_MAX_ROWS = 16 * 8191     # chunk ids of the real-valued filter ride in 13 mantissa bits, the all-ones id means "none"
DB_SIZES = [2, 16, 17, 100, 128, 129, 200, 255, 257, 1111]   # no padding, partial chunk, 1 to 7 pure-pad chunks in the last 128-row tile
Q_SIZES = [1, 127, 128, 129, 256, 257]                       # the 128- and 256-query work-item edges


# ---------------------------------------------------------------------------------------------- exact host reference
def sqdist(a, b):
    """||a||^2 + ||b||^2 - 2 a.b for integer-valued rows, as int64 [len(a), len(b)].  The product goes through float64 BLAS: every
    product and partial sum is an integer far below 2^53, so it is exact, and the result equals the reference's float distance
    because every distance is below 2^24."""
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64)
    dot = np.rint(a.astype(np.float64) @ b.T.astype(np.float64)).astype(np.int64)
    return (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * dot


def topk(d, k):
    """Indices and values of the k smallest entries per row, the lowest index first among equal values."""
    o = np.argsort(d, axis=1, kind="stable")[:, :k]
    return o, np.take_along_axis(d, o, axis=1)


def ratio_records(d, r):
    """RegionsMatcher::Match before de-duplication: top-2 per query, d1 < float(r)*float(r) * d2 in float (filters.hpp:60 with
    Square(r) in float, RegionsMatcher.hpp:150).  d: int64 [queries, database rows].  Returns MATCH_DTYPE records in query order."""
    nq, nb = d.shape
    out = np.zeros(0, matching.MATCH_DTYPE)
    if nq == 0 or nb < 2:                       # NN = 2 > rows: SearchNeighbours fails, no match (bruteForce.hpp:105)
        return out
    o, v = topk(d, 2)
    d1, d2 = v[:, 0].astype(np.float32), v[:, 1].astype(np.float32)
    keep = d1 < (np.float32(r) * np.float32(r)) * d2
    out = np.zeros(int(keep.sum()), matching.MATCH_DTYPE)
    out["i"] = o[keep, 0]; out["j"] = np.nonzero(keep)[0]
    out["ratio"] = d1[keep] / d2[keep]; out["dist"] = d1[keep]
    return out


def regions_match(d, xy_db, r):
    """RegionsMatcher::Match for database features in general position: IndMatch de-duplication (sorted by (i, j)), then the
    decorator's (every database feature keeps its match with the smallest query index; the set walks ascending database y)."""
    m = ratio_records(d, r)
    m = m[np.lexsort((m["j"], m["i"]))]
    m = m[np.r_[True, m["i"][1:] != m["i"][:-1]]] if len(m) else m
    return m[np.argsort(xy_db[m["i"], 1], kind="stable")]


def collection_match(descs, xys, pairs, r, cross):
    """ImageCollectionMatcher_generic::Match (cross: keep (i, j) of I->J iff (j, i) is in J->I's list), empty lists omitted."""
    res = {}
    for a, b in sorted({(int(p[0]), int(p[1])) for p in pairs}):
        if len(descs[a]) == 0 or len(descs[b]) == 0:
            continue
        fwd = regions_match(sqdist(descs[b], descs[a]), xys[a], r)
        if cross:
            rev = regions_match(sqdist(descs[a], descs[b]), xys[b], r)
            back = set(zip(rev["j"].tolist(), rev["i"].tolist()))
            fwd = fwd[np.array([(i, j) in back for i, j in zip(fwd["i"].tolist(), fwd["j"].tolist())], bool)] if len(fwd) else fwd
        if len(fwd):
            res[(a, b)] = fwd
    return res


def assert_same(got, want, what=""):
    missing, extra = sorted(set(want) - set(got)), sorted(set(got) - set(want))
    assert not missing and not extra, f"{what}: pairs missing {missing[:8]}, unexpected {extra[:8]}"
    for k in want:
        g, w = got[k], want[k]
        assert len(g) == len(w), f"{what}: pair {k} has {len(g)} matches, expected {len(w)}"
        for f in ("i", "j", "dist", "ratio"):
            assert np.array_equal(g[f], w[f]), f"{what}: {f} differs for pair {k}"


def as_dict(res):
    pid, off, mat = res
    return {(int(a), int(b)): mat[off[k]:off[k + 1]] for k, (a, b) in enumerate(pid.tolist()) if off[k + 1] > off[k]}


def assert_integer_domain(*arrays):
    for a in arrays:
        v = np.asarray(a, np.float64)
        assert np.array_equal(v, np.rint(v)) and np.abs(v).max() <= RANGE_LIMIT
        n = (np.asarray(a, np.int64) ** 2).sum(1)
        assert n.max() < NORM_LIMIT, n.max()


def fp16_norms(a):
    h = np.asarray(a, np.float32).astype(np.float16).astype(np.float64)
    return (h * h).sum(1)


def assert_real_domain(*arrays):
    for a in arrays:
        assert np.abs(a).max() <= RANGE_LIMIT and fp16_norms(a).max() < NORM_LIMIT and len(a) <= REAL_MAX_ROWS
        assert not np.array_equal(a, np.rint(a))


def n_directed(descs, pairs, cross):
    """Directed pairs that reach a search kernel: both views non-empty and at least two database rows."""
    n = 0
    for a, b in {(int(p[0]), int(p[1])) for p in pairs}:
        for i, j in ((a, b), (b, a)) if cross else ((a, b),):
            n += len(descs[i]) >= 2 and len(descs[j]) >= 1
    return n


@pytest.fixture
def ctx():
    """A context of the test's own: exactness_errors() counts over the context's life.  It is destroyed with the last object that uses
    it (an ArrayMatcherB200 kept alive by a failure's traceback must not outlive its context)."""
    return matching.Context(0)


def _fresh_matcher(env: dict, ratio=0.8, cross=False):
    """An ImageCollectionMatcherB200 on its own engine context created under `env` (the context reads its switches at creation)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        c = matching.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return ImageCollectionMatcherB200(ratio, cross, EMatcherType.BRUTE_FORCE_L2_B200, c)


# ---------------------------------------------------------------------------------------------- signed integer-valued data
def _family(kind, n_db, n_q, seed):
    """(database rows, query rows) as int64, every row inside the integer domain.
    anti:    database 160 + U[-15, 15], queries -(160 + U[-15, 15]): a.b < 0 for every pair, so that h = ||b||^2/2 - a.b of every real
             row (up to 2^21 + 2^22) exceeds that of a zero row.
    centred: SIFT-like rows minus 64 with planted correspondences.
    sparse:  three components of magnitude 1000..1024 with random signs on 16 dimensions (+ a little noise elsewhere); half of the
             queries are perturbed copies of database rows, a quarter negated copies (anti-aligned), a quarter fresh rows."""
    rng = np.random.default_rng(seed)
    if kind == "anti":
        return 160 + rng.integers(-15, 16, (n_db, 128)), -(160 + rng.integers(-15, 16, (n_q, 128)))
    if kind == "centred":
        d, _ = synth.sift_images(2, max(n_db, n_q), np.int16, seed=seed, pool_factor=1.0)
        return d[0][:n_db].astype(np.int64) - 64, d[1][:n_q].astype(np.int64) - 64

    def sparse(n):
        x = rng.integers(-2, 3, (n, 128))
        for r in range(n):
            pos = rng.choice(16, 3, replace=False)
            x[r, pos] = rng.choice([-1, 1], 3) * rng.integers(1000, 1025, 3)
        return x
    db = sparse(n_db)
    q = sparse(n_q)
    src = rng.integers(0, n_db, n_q)
    half, quarter = n_q // 2, n_q // 4
    q[:half] = np.clip(db[src[:half]] + rng.integers(-2, 3, (half, 128)), -RANGE_LIMIT, RANGE_LIMIT)
    q[half:half + quarter] = -db[src[half:half + quarter]]
    return db, q[rng.permutation(n_q)]


FAMILIES = ["anti", "centred", "sparse"]
_views_cache = {}


def signed_views(kind):
    """Views 0..9: database images of DB_SIZES rows, views 10..15: query images of Q_SIZES rows (prefixes of one pool each),
    fp32 storage, positions in general position; the pair list is every (database, query) combination."""
    if kind not in _views_cache:
        db, q = _family(kind, max(DB_SIZES), max(Q_SIZES), seed=1000 + FAMILIES.index(kind))
        assert_integer_domain(db, q)
        rng = np.random.default_rng(7)
        descs = [np.ascontiguousarray(db[:m], np.float32) for m in DB_SIZES] + [np.ascontiguousarray(q[:m], np.float32) for m in Q_SIZES]
        xys = [synth.positions(len(d), rng) for d in descs]
        pairs = np.array([(a, len(DB_SIZES) + b) for a in range(len(DB_SIZES)) for b in range(len(Q_SIZES))], np.uint32)
        _views_cache[kind] = (descs, xys, pairs)
    return _views_cache[kind]


@pytest.mark.parametrize("variant", [1, 2, 3, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_signed_integer_collection_vs_exact_reference(ctx, family, variant):
    """ImageCollectionMatcherB200 on signed / large-magnitude integer-valued fp32 rows, every database size against every query size, all four
    tensor-core variants, cross matching off and on, ratios 0.8 and 1.0: the final lists and the raw match records equal the exact reference."""
    descs, xys, pairs = signed_views(family)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    ctx.set_tc_variant(variant)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    kept = 0
    for cross in (False, True):
        for r in (0.8, 1.0):
            m.distRatio, m.crossMatching = r, cross
            what = f"cross={cross} ratio={r}"
            got = as_dict(m.match_uploaded(pairs))
            assert ctx.last_tc_pairs() == n_directed(descs, pairs, cross), what
            want = collection_match(descs, xys, pairs, r, cross)
            assert_same(got, want, what)
            kept += sum(len(v) for v in want.values())
            if not cross:
                # raw records (no de-duplication): one per query that passes the ratio test, in no particular order
                raw = as_dict(m.match_uploaded(pairs, matching.STAGE_RAW))
                want_raw = {}
                for a, b in pairs.tolist():
                    rec = ratio_records(sqdist(descs[b], descs[a]), r)
                    if len(rec):
                        want_raw[(a, b)] = rec
                assert_same({k: v[np.argsort(v["j"], kind="stable")] for k, v in raw.items()}, want_raw, what + " raw")
            assert ctx.exactness_errors() == 0, what
    assert kept > 0


@pytest.mark.parametrize("family", FAMILIES)
def test_signed_integer_collection_vs_oracle(ctx, ora, family):
    """The default kernel on the same views against the oracle (which also confirms the host reference above)."""
    descs, xys, pairs = signed_views(family)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    for cross in (False, True):
        for r in (0.8, 1.0):
            want = ora.collection_match(descs, xys, pairs, r, cross)
            what = f"cross={cross} ratio={r}"
            assert_same(collection_match(descs, xys, pairs, r, cross), want, what + " host reference")
            m.distRatio, m.crossMatching = r, cross
            assert_same(as_dict(m.match_uploaded(pairs)), want, what)
            assert ctx.last_tc_pairs() == n_directed(descs, pairs, cross) and ctx.exactness_errors() == 0, what


@pytest.mark.parametrize("family", FAMILIES)
def test_signed_integer_arraymatcher_knn(ctx, family):
    """ArrayMatcherB200.SearchNeighbours(NN = 2) (MODE_KNN) on ragged signed databases: distances equal the exact top-2, indices wherever
    the reference's order is unambiguous."""
    db, q = _family(family, max(DB_SIZES), 300, seed=2000 + FAMILIES.index(family))
    assert_integer_domain(db, q)
    qf = np.ascontiguousarray(q, np.float32)
    for mi in (2, 16, 17, 100, 129, 257, 1111):
        am = ArrayMatcherB200(matching.L2_VECTORIZED, ctx)
        assert am.Build(np.ascontiguousarray(db[:mi], np.float32))
        ok, idx, dist = am.SearchNeighbours(qf, NN=2)
        assert ok and ctx.last_tc_pairs() == 1 and ctx.exactness_errors() == 0, mi
        o, v = topk(sqdist(q, db[:mi]), 3)
        assert np.array_equal(dist, v[:, :2].astype(np.float32)), mi
        d3 = v[:, 2] if mi >= 3 else np.full(len(q), np.iinfo(np.int64).max)
        strict1 = v[:, 0] < v[:, 1]
        strict2 = strict1 & (v[:, 1] < d3)
        assert np.array_equal(idx[strict1, 0], o[strict1, 0]) and np.array_equal(idx[strict2, 1], o[strict2, 1]), mi


# ---------------------------------------------------------------------------------------------- signed real-valued data (MODE_REAL)
REAL_DB_SIZES = [2, 17, 129, 200, 257, 1111]
REAL_Q_SIZES = [1, 129, 257]


def _real_family(kind, seed):
    rng = np.random.default_rng(seed)
    n_db, n_q = max(REAL_DB_SIZES), max(REAL_Q_SIZES)
    if kind == "anti":       # large norms (~3.3e6 of the 4.19e6 limit), every query anti-correlated with every database row
        noise = lambda n: np.clip(rng.normal(0, 0.37, (n, 128)), -1, 1)
        db = 160 + rng.integers(-15, 16, (n_db, 128)) + noise(n_db)
        q = -(160 + rng.integers(-15, 16, (n_q, 128)) + noise(n_q))
        rs = (1.0,)
    else:                    # centred SIFT-like rows with real noise, scaled to roughly unit norm (every bound of the filter is relative)
        d, _ = synth.sift_images(2, n_db, np.float32, seed=seed, pool_factor=1.0)
        d = [(x - 64.0) / 512.0 for x in synth.real_valued(d)]
        db, q = d[0], d[1][:n_q]
        rs = (0.8, 1.0)
    db, q = np.ascontiguousarray(db, np.float32), np.ascontiguousarray(q, np.float32)
    assert_real_domain(db, q)
    rng2 = np.random.default_rng(9)
    descs = [db[:m] for m in REAL_DB_SIZES] + [q[:m] for m in REAL_Q_SIZES]
    xys = [synth.positions(len(x), rng2) for x in descs]
    pairs = np.array([(a, len(REAL_DB_SIZES) + b) for a in range(len(REAL_DB_SIZES)) for b in range(len(REAL_Q_SIZES))], np.uint32)
    return descs, xys, pairs, rs


@pytest.mark.parametrize("rescoring", ["standalone", "in_kernel"])
@pytest.mark.parametrize("kind", ["anti", "centred_unit"])
def test_signed_real_valued_vs_oracle(ora, kind, rescoring):
    """Signed real-valued rows on the tensor-core filter, ragged sizes, with the stand-alone re-scoring kernel (short database images) and
    with the re-scoring inside the filter kernel (B200M_REAL_FUSED_ROWS=0 lowers the average database rows it needs from 6144 to 0)."""
    descs, xys, pairs, rs = _real_family(kind, seed=3000 + (kind == "anti"))
    m = _fresh_matcher({"B200M_REAL_FUSED_ROWS": "0"} if rescoring == "in_kernel" else {})
    try:
        m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
        m.wait_uploads()
        kept = 0
        for r in rs:
            m.distRatio = r
            got = as_dict(m.match_uploaded(pairs))
            assert m.ctx.last_real_tc_pairs() == n_directed(descs, pairs, False) and m.ctx.last_tc_pairs() == 0
            want = ora.collection_match(descs, xys, pairs, r)
            assert_same(got, want)
            kept += sum(len(v) for v in want.values())
        assert kept > 0 and m.ctx.exactness_errors() == 0
    finally:
        m.ctx.close()


# ---------------------------------------------------------------------------------------------- domain edges
def greedy_squares(target, rng, n=124):
    """n signed integer components, |v| <= 1024, whose squares sum to exactly `target` (greedy: the largest square that fits)."""
    v = np.zeros(n, np.int64)
    rest, k = int(target), 0
    while rest:
        s = min(int(np.sqrt(rest)), RANGE_LIMIT)
        while s * s > rest:
            s -= 1
        v[k] = s; rest -= s * s; k += 1
    assert k <= n
    return v * rng.choice([-1, 1], n)


def _edge_views(real, seed):
    """Two 300-row centred SIFT-like views (integer-valued, or real-valued with noise), view 1 holding planted copies of view 0."""
    d, xy = synth.sift_images(2, 300, np.float32, seed=seed, pool_factor=1.0)
    if real:
        d = synth.real_valued(d)
    return [np.ascontiguousarray(x - np.float32(64)) for x in d], xy


def _run_pairs(ctx, descs, xys, r=0.8):
    m = ImageCollectionMatcherB200(r, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    return dict(m.Match({0: (descs[0], xys[0]), 1: (descs[1], xys[1])}, [(0, 1), (1, 0)]))


@pytest.mark.parametrize("value", [1024, -1024, 1025, -1025])
def test_integer_component_range_edge(ctx, ora, value):
    """|v| = 1024 is inside the integer domain (tensor cores), one component of magnitude 1025 sends the view to the exact kernel."""
    descs, xys = _edge_views(False, seed=401)
    descs[0][5, 3] = value
    descs[1][7] = descs[0][5]; descs[1][7, 40] += 1                   # a near copy in the other view: the edge row is matched
    inside = abs(value) <= RANGE_LIMIT
    if inside:
        assert_integer_domain(*descs)
    got = _run_pairs(ctx, descs, xys)
    assert ctx.last_tc_pairs() == (2 if inside else 0) and ctx.exactness_errors() == 0
    want = ora.collection_match(descs, xys, [(0, 1), (1, 0)], 0.8)
    assert_same(got, want)
    assert_same(got, collection_match(descs, xys, [(0, 1), (1, 0)], 0.8, False))
    assert 5 in want[(0, 1)]["i"]


@pytest.mark.parametrize("norm", [NORM_LIMIT - 1, NORM_LIMIT])
def test_integer_norm_edge(ctx, ora, norm):
    """||v||^2 = 2^22 - 1 is inside the integer domain, 2^22 is not: collection pairs and the ArrayMatcher path."""
    descs, xys = _edge_views(False, seed=402)
    rng = np.random.default_rng(4)
    row = np.concatenate([np.zeros(4, np.int64), greedy_squares(norm, rng)])[rng.permutation(128)]
    assert int((row * row).sum()) == norm and np.abs(row).max() <= RANGE_LIMIT
    descs[0][5] = row
    near = row.copy(); near[np.argmax(np.abs(near))] //= 2            # well inside the domain, and still nearest to row 5
    descs[1][7] = near
    inside = norm < NORM_LIMIT
    if inside:
        assert_integer_domain(*descs)
    got = _run_pairs(ctx, descs, xys)
    assert ctx.last_tc_pairs() == (2 if inside else 0) and ctx.exactness_errors() == 0
    want = ora.collection_match(descs, xys, [(0, 1), (1, 0)], 0.8)
    assert_same(got, want)
    assert_same(got, collection_match(descs, xys, [(0, 1), (1, 0)], 0.8, False))
    am = ArrayMatcherB200(matching.L2_VECTORIZED, ctx)
    assert am.Build(descs[0])
    ok, idx, dist = am.SearchNeighbours(descs[1], NN=2)
    assert ok and ctx.last_tc_pairs() == (1 if inside else 0) and ctx.exactness_errors() == 0
    o, v = topk(sqdist(descs[1], descs[0]), 2)
    assert np.array_equal(dist, v.astype(np.float32)) and idx[7, 0] == 5


@pytest.mark.parametrize("value", [1024.0, -1024.0, 1024.25, -1024.5])
def test_real_component_range_edge(ctx, ora, value):
    """The same range edge for a real-valued view: |v| = 1024 takes the tensor-core filter (MODE_REAL), anything above the exact kernel
    (even when, like 1024.25, it rounds to 1024 in fp16)."""
    descs, xys = _edge_views(True, seed=403)
    descs[0][5, 3] = value
    descs[1][7] = descs[0][5]; descs[1][7, 40] += np.float32(0.25)
    inside = abs(value) <= RANGE_LIMIT
    if inside:
        assert_real_domain(*descs)
    got = _run_pairs(ctx, descs, xys)
    assert ctx.last_real_tc_pairs() == (2 if inside else 0) and ctx.last_tc_pairs() == 0 and ctx.exactness_errors() == 0
    want = ora.collection_match(descs, xys, [(0, 1), (1, 0)], 0.8)
    assert_same(got, want)
    assert 5 in want[(0, 1)]["i"]


@pytest.mark.parametrize("norm", [NORM_LIMIT - 1, NORM_LIMIT])
def test_real_norm_edge(ctx, ora, norm):
    """||fp16(v)||^2 = 2^22 - 1 takes MODE_REAL, 2^22 the exact kernel.  The edge row is four components of 0.5 (the view is real-valued)
    plus integers, all exact in fp16, so its fp16 norm is exactly `norm`."""
    descs, xys = _edge_views(True, seed=404)
    rng = np.random.default_rng(5)
    row = np.concatenate([np.full(4, 0.5), greedy_squares(norm - 1, rng)])[rng.permutation(128)].astype(np.float32)
    assert fp16_norms(row[None])[0] == norm
    descs[0][5] = row
    near = row.copy(); near[np.argmax(np.abs(near))] *= np.float32(0.5); near -= np.float32(0.125) * np.sign(near)
    descs[1][7] = near
    inside = norm < NORM_LIMIT
    if inside:
        assert_real_domain(*descs)
    got = _run_pairs(ctx, descs, xys)
    assert ctx.last_real_tc_pairs() == (2 if inside else 0) and ctx.last_tc_pairs() == 0 and ctx.exactness_errors() == 0
    want = ora.collection_match(descs, xys, [(0, 1), (1, 0)], 0.8)
    assert_same(got, want)
    assert 5 in want[(0, 1)]["i"]


@pytest.mark.parametrize("rows", [REAL_MAX_ROWS, REAL_MAX_ROWS + 1])
def test_real_valued_database_row_limit(ctx, ora, rows):
    """A real-valued database of exactly 131056 rows takes MODE_REAL: its last chunk id, 8190, uses all 13 id bits of the packed chunk
    minima.  One row more and the pair goes to the exact kernel.  Queries are planted near rows all over the image, the last chunk included."""
    rng = np.random.default_rng(405)
    db = (synth.sift_pool(rows, rng).astype(np.float32) - np.float32(64)) + rng.normal(0, 0.37, (rows, 128)).astype(np.float32)
    src = np.concatenate([rng.integers(0, rows, 200), np.arange(rows - 40, rows)])
    q = np.concatenate([db[src] + rng.normal(0, 1.0, (len(src), 128)).astype(np.float32),
                        synth.sift_pool(60, rng).astype(np.float32) - np.float32(64) + np.float32(0.5)])
    descs = [np.ascontiguousarray(db), np.ascontiguousarray(q, np.float32)]
    assert_real_domain(descs[1])
    assert np.abs(db).max() <= RANGE_LIMIT and fp16_norms(db).max() < NORM_LIMIT
    xys = [synth.positions(len(d), rng) for d in descs]
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    got = dict(m.Match({0: (descs[0], xys[0]), 1: (descs[1], xys[1])}, [(0, 1)]))
    assert ctx.last_real_tc_pairs() == (1 if rows <= REAL_MAX_ROWS else 0) and ctx.last_tc_pairs() == 0 and ctx.exactness_errors() == 0
    want = ora.collection_match(descs, xys, [(0, 1)], 0.8)
    assert_same(got, want)
    assert (want[(0, 1)]["i"] >= REAL_MAX_ROWS - 16).any()          # the last chunk of a full-size view holds matches


# ---------------------------------------------------------------------------------------------- in-kernel exactness pass on short items
def test_fused_exactness_pass_on_short_database_images(ctx, ora):
    """One batch of nine pairs with 8192-row databases and three with 17-, 129- and 257-row databases.  The batch runs the exactness pass
    inside the search kernel when its database images average at least 6144 rows (engine.cu, `fused`; variants 2-4):
        (9 * 8192 + 17 + 129 + 257) / 12 = 74131 / 12 = 6177 >= 6144,
    so the short items, whose last tiles are mostly padding, go through the in-kernel pass too.  Their queries are anti-correlated with
    their databases."""
    big, _ = synth.sift_images(6, 8192, np.int16, seed=501, pool_factor=1.0)
    anti_db, anti_q = _family("anti", 257, 300, seed=502)
    views = [b.astype(np.int64) - 64 for b in big[:3]] + [b[:300].astype(np.int64) - 64 for b in big[3:]]   # 0-2 databases, 3-5 queries
    views += [anti_db[:17], anti_db[:129], anti_db, anti_q]                                                      # 6-8 databases, 9 queries
    assert_integer_domain(*views)
    descs = [np.ascontiguousarray(v, np.float32) for v in views]
    rng = np.random.default_rng(503)
    xys = [synth.positions(len(d), rng) for d in descs]
    pairs = np.array([(a, b) for a in range(3) for b in range(3, 6)] + [(6, 9), (7, 9), (8, 9)], np.uint32)
    rows = [len(descs[a]) for a, _ in pairs]
    assert sum(rows) // len(rows) >= 6144
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()                                               # resident views: the whole pair list is one batch
    for r in (0.8, 1.0):
        want = ora.collection_match(descs, xys, pairs, r)
        if r == 1.0:
            assert all((a, 9) in want for a in (6, 7, 8))
        for variant in (2, 3, 4):
            ctx.set_tc_variant(variant)
            m.distRatio = r
            got = as_dict(m.match_uploaded(pairs))
            assert ctx.last_tc_pairs() == len(pairs) and ctx.exactness_errors() == 0, variant
            assert_same(got, want, f"variant={variant} ratio={r}")
