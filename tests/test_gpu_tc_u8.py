"""The u8 search kernel (l2_tc.cuh, U8): integer-valued pairs whose two views are both stored as uchar run on the 8-bit tensor cores with
exact int32 distances (run with -m gpu on an H100).

Every test compares the final match lists with the oracle (RegionsMatcher::Match through collection_match, bit-exact: indices,
distances, ratios), asserts how many directed pairs took the u8 kernel (last_u8_tc_pairs) and the tensor cores at all (last_tc_pairs),
so that a silent change of path cannot pass, and that the exactness pass found no error."""
import numpy as np
import pytest

from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

pytestmark = pytest.mark.gpu

NORM_LIMIT = 1 << 22          # integer tensor-core domain: ||v||^2 < 2^22 (larger norms go to the exact kernels)


def as_dict(res):
    pid, off, mat = res
    return {(int(a), int(b)): mat[off[k]:off[k + 1]] for k, (a, b) in enumerate(pid.tolist()) if off[k + 1] > off[k]}


def assert_same(got, want, what=""):
    assert sorted(got) == sorted(want), f"{what}: pairs {sorted(set(got) ^ set(want))[:8]} differ"
    for k in want:
        g, w = got[k], want[k]
        assert len(g) == len(w), f"{what}: pair {k} has {len(g)} matches, expected {len(w)}"
        for f in ("i", "j", "dist", "ratio"):
            assert np.array_equal(g[f], w[f]), f"{what}: {f} differs for pair {k}"


def n_directed(descs, pairs, cross, select=lambda a, b: True):
    """Directed pairs that reach a search kernel (both views non-empty, at least two database rows) and satisfy `select`."""
    n = 0
    for a, b in {(int(p[0]), int(p[1])) for p in pairs}:
        for i, j in ((a, b), (b, a)) if cross else ((a, b),):
            n += len(descs[i]) >= 2 and len(descs[j]) >= 1 and select(i, j)
    return n


def check(ctx, ora, descs, xys, pairs, ratios=(0.8, 1.0), crosses=(False, True), u8=None):
    """Resident views (one batch per call), every ratio and cross setting against the oracle.  u8(i, j): whether directed pair (i, j)
    is expected on the u8 kernel (default: all); every directed pair is expected on the tensor cores."""
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    kept = 0
    for cross in crosses:
        for r in ratios:
            what = f"cross={cross} ratio={r}"
            m.distRatio, m.crossMatching = r, cross
            got = as_dict(m.match_uploaded(pairs))
            assert ctx.last_tc_pairs() == n_directed(descs, pairs, cross), what
            assert ctx.last_u8_tc_pairs() == n_directed(descs, pairs, cross, u8 or (lambda a, b: True)), what
            assert ctx.exactness_errors() == 0, what
            want = ora.collection_match(descs, xys, pairs, r, cross)
            assert_same(got, want, what)
            kept += sum(len(v) for v in want.values())
    assert kept > 0
    return m


@pytest.fixture
def ctx():
    return matching.Context(0)


def assert_u8_domain(*arrays):
    for a in arrays:
        v = np.asarray(a, np.int64)
        assert v.min() >= 0 and v.max() <= 255 and (v * v).sum(1).max() < NORM_LIMIT


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_full_size_fused(ctx, ora, dtype):
    """8192 x 8192 (the benchmark's image size): the in-kernel exactness pass (work items of >= 6144 database rows), uchar views as
    uploaded (uint8) and integer-valued fp32 views staged as uchar."""
    descs, xys = synth.sift_images(2, 8192, dtype, seed=601, pool_factor=1.0)
    assert_u8_domain(*descs)
    check(ctx, ora, descs, xys, np.array([(0, 1)], np.uint32), ratios=(0.8,))


DB_SIZES = [2, 5, 16, 17, 100, 129, 200, 255, 257, 1111]     # <= 16 (second chunk minimum = padding), partial chunks, 1..7 pad chunks
Q_SIZES = [1, 15, 127, 129, 255, 257, 300]                    # the 128- and 256-query work-item edges


def ragged_views(seed):
    """Views 0..9: database images of DB_SIZES rows, 10..16: query images of Q_SIZES rows (prefixes of two planted SIFT images)."""
    d, _ = synth.sift_images(2, max(DB_SIZES), np.uint8, seed=seed, pool_factor=1.0)
    descs = [d[0][:m] for m in DB_SIZES] + [d[1][:m] for m in Q_SIZES]
    rng = np.random.default_rng(seed)
    xys = [synth.positions(len(x), rng) for x in descs]
    pairs = np.array([(a, len(DB_SIZES) + b) for a in range(len(DB_SIZES)) for b in range(len(Q_SIZES))], np.uint32)
    return descs, xys, pairs


def test_ragged_sizes_unfused(ctx, ora):
    """Short database images (the stand-alone exactness pass, verify_pack_kernel) of sizes that are not multiples of 16, 128 or 256,
    m_i <= 16 included, against queries across the work-item edges.  Variant 3 leaves the same pairs on the fp16 kernel."""
    descs, xys, pairs = ragged_views(602)
    assert_u8_domain(*descs)
    m = check(ctx, ora, descs, xys, pairs)
    ctx.set_tc_variant(3)
    m.distRatio, m.crossMatching = 0.8, False
    got = as_dict(m.match_uploaded(pairs))
    assert ctx.last_u8_tc_pairs() == 0 and ctx.last_tc_pairs() == n_directed(descs, pairs, False) and ctx.exactness_errors() == 0
    assert_same(got, ora.collection_match(descs, xys, pairs, 0.8), "variant 3")


def test_zero_and_near_saturated_rows(ctx, ora):
    """All-zero rows and rows of 64 components in 250..255 (norms up to 64 * 255^2 = 4161600, just inside 2^22), scattered over
    chunks and tiles of both views, with near copies in the other view."""
    rng = np.random.default_rng(603)
    d, xys = synth.sift_images(2, 1500, np.uint8, seed=603, pool_factor=1.0)
    db, q = d[0].copy(), d[1].copy()
    for rows in (db, q):
        rows[rng.choice(len(rows), 40, replace=False)] = 0
    hot = rng.choice(len(db), 60, replace=False)
    for r in hot:
        v = np.zeros(128, np.uint8)
        v[rng.choice(128, 64, replace=False)] = rng.integers(250, 256, 64)
        db[r] = v
    for k, r in enumerate(hot[:30]):                       # near copies among the queries
        v = db[r].astype(np.int64)
        v[rng.integers(0, 128)] ^= 1
        q[k * 37 % len(q)] = np.clip(v, 0, 255)
    assert_u8_domain(db, q)
    assert (db * db.astype(np.int64)).sum(1).max() > 4_000_000
    check(ctx, ora, [db, q], xys, np.array([(0, 1)], np.uint32))


def test_duplicate_rows_in_different_chunks(ctx, ora):
    """Copies of a database row in different 16-row chunks and tiles (and twice in one chunk), queried by near copies: the chunk minima
    tie, and the lowest chunk id, then the lowest row, must win as in the reference (whose ratio test then rejects the equal pair)."""
    rng = np.random.default_rng(604)
    d, xys = synth.sift_images(2, 2000, np.uint8, seed=604, pool_factor=1.0)
    db, q = d[0].copy(), d[1].copy()
    for k, src in enumerate(rng.choice(len(db), 12, replace=False)):
        for dst in rng.choice(len(db), 3, replace=False).tolist() + [src ^ 1]:
            db[dst] = db[src]
        v = db[src].astype(np.int64)
        v[rng.integers(0, 128)] += 1
        q[k] = np.clip(v, 0, 255)
        q[12 + k] = db[src]
    assert_u8_domain(db, q)
    check(ctx, ora, [db, q], xys, np.array([(0, 1)], np.uint32))


def test_mixed_batch_u8_and_signed_pairs(ctx, ora):
    """One batch of uchar-range fp32 views (staged as uchar) and signed integer-valued fp32 views (stored as fp32): u8/u8 pairs run the
    u8 kernel, u8/signed pairs the fp16 kernel; both count as tensor-core pairs.  The database images are long enough for the in-kernel
    exactness pass on both lists."""
    d, xys = synth.sift_images(5, 6200, np.float32, seed=605, pool_factor=1.0)
    descs = d[:3] + [np.ascontiguousarray(x - np.float32(64)) for x in d[3:]]    # views 3, 4: signed
    assert_u8_domain(*descs[:3])
    assert min(x.min() for x in descs[3:]) < 0
    pairs = np.array([(0, 1), (0, 3), (1, 2), (2, 4)], np.uint32)
    check(ctx, ora, descs, xys, pairs, ratios=(0.8,), u8=lambda a, b: a < 3 and b < 3)
