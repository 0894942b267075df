"""The u8 search kernel's per-thread chunks (l2_tc.cuh U8, common.cuh chunk_row): chunk 8t + 4h + q of a database image is rows
128t + 64h + 8j + 2q + e (j = 0..7, e = 0, 1), the 16 columns one thread holds, not 16 consecutive rows (run with -m gpu on an H100).

Every test compares the final match lists with the oracle (RegionsMatcher::Match through collection_match, bit-exact: indices,
distances, ratios) and asserts that the pairs took the u8 kernel (last_u8_tc_pairs) and that the exactness pass found no error."""
import numpy as np
import pytest

from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

pytestmark = pytest.mark.gpu

FUSED_ROWS = 6144             # database images at least this long (on average over a launch) are re-scored inside the search kernel


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


def check(ctx, ora, descs, xys, pairs, n_u8, n_tc=None, ratios=(0.8, 1.0)):
    """Resident views, one call per ratio, against the oracle; n_u8 / n_tc: directed pairs expected on the u8 kernel / the tensor cores."""
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    wants = []
    for r in ratios:
        m.distRatio = r
        got = as_dict(m.match_uploaded(pairs))
        assert ctx.last_u8_tc_pairs() == n_u8 and ctx.last_tc_pairs() == (n_u8 if n_tc is None else n_tc), f"ratio={r}"
        assert ctx.exactness_errors() == 0, f"ratio={r}"
        want = ora.collection_match(descs, xys, pairs, r, False)
        assert_same(got, want, f"ratio={r}")
        wants.append(want)
    return wants


@pytest.fixture
def ctx():
    return matching.Context(0)


def chunk_rows(t, h, q):
    """The 16 database rows of chunk 8t + 4h + q, ascending."""
    return [128 * t + 64 * h + 8 * j + 2 * q + e for j in range(8) for e in range(2)]


def near(v, d, off=0):
    """A copy of row v at squared distance d: components off .. off + d - 1 moved by one."""
    w = v.astype(np.int16)
    w[off:off + d] += np.where(w[off:off + d] < 255, 1, -1)
    return w.astype(np.uint8)


def two_images(m_db, m_q, seed):
    d, xys = synth.sift_images(2, max(m_db, m_q), np.uint8, seed=seed, pool_factor=1.0)
    rng = np.random.default_rng(seed)
    return d[0][:m_db].copy(), d[1][:m_q].copy(), [synth.positions(m_db, rng), synth.positions(m_q, rng)]


# (squared distance of the nearer row, of the other row, which row of the pair is the nearer one)
CASES = [(1, 9, 0), (1, 9, 1), (3, 4, 0), (2, 2, 0), (0, 0, 0), (0, 5, 1)]


def plant_row_pairs(db, q, m_db):
    """Per 64-row block, one query per case of CASES with its two nearest rows planted as a row pair: (x, x + 8), one per-thread chunk,
    in even blocks and (x, x + 2), neighbouring rows of different chunks, in odd ones.  Returns {query: nearer row} of the cases the
    reference keeps at ratio 0.8 and at ratio 1.0."""
    last = m_db // 128 - 1
    keep08, keep10, n = {}, {}, 0
    for blk, (t, h) in enumerate([(0, 0), (0, 1), (5, 0), (5, 1), (last, 0), (last, 1)]):
        base, step = 128 * t + 64 * h, 2 if blk % 2 else 8
        firsts = [base + 2 * step * i + c for i in range(32 // step) for c in range(step)]       # disjoint pairs (x, x + step) of the block
        for ci, (d_lo, d_hi, which) in enumerate(CASES):
            x = firsts[(5 * ci + blk) % len(firsts)]
            assert (x + step in chunk_rows(t, h, x % 8 // 2)) == (step == 8) and x in chunk_rows(t, h, x % 8 // 2)
            lo, hi = (x, x + step) if which == 0 else (x + step, x)
            db[lo] = near(q[n], d_lo)
            db[hi] = near(q[n], d_hi, off=d_lo if d_hi == d_lo else 0)         # equidistant rows differ unless both are exact copies
            if d_lo < 0.64 * d_hi:
                keep08[n] = lo
            if d_lo < d_hi:
                keep10[n] = lo
            n += 1
    return keep08, keep10


@pytest.mark.parametrize("m_db", [8192, 1000])       # in-kernel exactness pass / verify_pack_kernel
def test_best_and_second_inside_and_across_chunks(ctx, ora, m_db):
    """Best and second-best rows x, x + 8 (one per-thread chunk: the second distance comes from the re-scoring) and x, x + 2 (neighbouring
    rows, different chunks: it comes from the second chunk minimum), in either order: near copies, equidistant rows and exact duplicates
    (which the reference drops even at ratio 1.0)."""
    db, q, xys = two_images(m_db, 256, 611)
    keep08, keep10 = plant_row_pairs(db, q, m_db)
    wants = check(ctx, ora, [db, q], xys, np.array([(0, 1)], np.uint32), 1)
    for want, keep in zip(wants, (keep08, keep10)):
        w = want[(0, 1)]
        assert len(keep) >= 18 and set(zip(w["i"].tolist(), w["j"].tolist())) >= {(r, n) for n, r in keep.items()}


@pytest.mark.parametrize("m_db", [8192, 128 * 9 + 65])
def test_nearest_neighbour_at_every_chunk_position(ctx, ora, m_db):
    """A planted nearest neighbour at each of the 16 positions of a chunk, in both halves of the first and of the last tile (partial
    when m_db is not a multiple of 128: rows past the end are skipped), for every quad lane."""
    db, q, xys = two_images(m_db, 512, 612)
    last = (m_db - 1) // 128
    rows = [r for t in (0, last) for h in (0, 1) for ql in range(4) for r in chunk_rows(t, h, ql) if r < m_db]
    assert len(set(rows)) == len(rows) and len(rows) <= len(q)
    for n, r in enumerate(rows):
        db[r] = near(q[n], 1 + n % 3)
    wants = check(ctx, ora, [db, q], xys, np.array([(0, 1)], np.uint32), 1, ratios=(0.8,))
    w = wants[0][(0, 1)]
    assert set(zip(w["i"].tolist(), w["j"].tolist())) >= {(r, n) for n, r in enumerate(rows)}


def ragged(sizes, seed):
    """Database images of `sizes` rows (prefixes of one SIFT image with planted correspondences) against one 300-row query image."""
    d, _ = synth.sift_images(2, max(max(sizes), 300), np.uint8, seed=seed, pool_factor=1.0)
    descs = [d[0][:m] for m in sizes] + [d[1][:300]]
    rng = np.random.default_rng(seed)
    xys = [synth.positions(len(x), rng) for x in descs]
    return descs, xys, np.array([(a, len(sizes)) for a in range(len(sizes))], np.uint32)


TAILS = (1, 2, 15, 17, 63, 65, 127)


def test_pad_rows_inside_chunks_unfused(ctx, ora):
    """Database sizes 128k + {1, 2, 15, 17, 63, 65, 127} and <= 16: in the last tile pad rows and real rows share chunks (a chunk of the
    last tile is real up to some position and padding from there on), stand-alone exactness pass."""
    sizes = [2, 3, 9, 16] + [128 * k + r for k in (0, 1, 6) for r in TAILS if 128 * k + r >= 2]
    descs, xys, pairs = ragged(sizes, 613)
    check(ctx, ora, descs, xys, pairs, len(pairs))


def test_pad_rows_inside_chunks_fused(ctx, ora):
    """The same tails on database images long enough for the in-kernel exactness pass."""
    sizes = [FUSED_ROWS + r for r in TAILS]
    descs, xys, pairs = ragged(sizes, 614)
    check(ctx, ora, descs, xys, pairs, len(pairs), ratios=(0.8,))


def test_both_chunk_layouts_in_one_packing_launch(ctx, ora):
    """One batch of short images with u8/u8 pairs (u8 kernel, per-thread chunks) and u8/signed pairs (fp16 kernel, contiguous chunks):
    verify_pack_kernel re-scores candidates of both layouts in one launch."""
    d, xys = synth.sift_images(4, 900, np.float32, seed=615, pool_factor=1.0)
    descs = d[:3] + [np.ascontiguousarray(d[3] - np.float32(64))]                 # view 3: signed, stored as fp32
    pairs = np.array([(0, 1), (0, 3), (1, 2), (3, 2), (2, 0)], np.uint32)
    check(ctx, ora, descs, xys, pairs, 3, n_tc=5)
