"""Every decision of the real-valued filter (MODE_REAL, verify.cuh rescore_real) against the oracle.

The fp16 tensor-core GEMM only filters real-valued rows; the bound of verify.cuh real_bound (eta from the fp16 rounding, sigma = 2^-14 S
for the fp32 accumulation) then decides each query on its two best chunks, on a third chunk, or leaves it undecided for the exact
fallback: exact_rows_pairs_kernel for the first FB_PER_PAIR = 64 queries of a pair, exact_rows_kernel for the overflow list.  Random
SIFT-like rows almost never reach the last two branches, so the inputs here are built for them:

* fp16 twins: rows that differ but round to the same fp16 row, so the filter cannot tell them apart and their chunk minima are
  ordered by chunk id, while which one is truly closer is placed on purpose;
* rows of 150 + N(0, s), s <= 1: every distance lies far inside sigma, so every query is undecided.

A float64 model of the decision (below) states which branch each query takes, with a margin of sigma and of the chunk id's 2^-10
relative truncation for what the device may differ by; on the GPU (run with -m gpu on an H100) every list must equal the oracle's bit
for bit, and the number of queries sent to the fallback must lie between the model's certainly and possibly undecided counts."""
import os

import numpy as np
import pytest

from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

CHUNK = 16
FB_PER_PAIR = 64
PAIR_CAP = 4096


# ---------------------------------------------------------------------------------------------- float64 model of the decision
def fp16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float64)


def ref_l2(q, rows):
    """The reference's L2_Vectorized<float>: four lanes s_l += (a - b)^2 over components l, l + 4, ..., then ((s0 + s1) + s2) + s3."""
    d = np.asarray(q, np.float32)[None, :] - np.asarray(rows, np.float32)
    d2 = (d * d).astype(np.float32)
    s = np.zeros((len(rows), 4), np.float32)
    for t in range(d.shape[1] // 4):
        s += d2[:, 4 * t:4 * t + 4]
    return ((s[:, 0] + s[:, 1]) + s[:, 2]) + s[:, 3]


class Model:
    """The decision of rescore_real for every query of one directed pair (database `db`, queries `q`) at ratio r, in float64."""

    def __init__(self, db, q, r, block=1024):
        db = np.asarray(db, np.float64); q = np.asarray(q, np.float64)
        hd, hq = fp16(db), fp16(q)
        err_d = np.sqrt(((db - hd) ** 2).sum(1)) * (1 + 2.0 ** -9)
        err_q = np.sqrt(((q - hq) ** 2).sum(1)) * (1 + 2.0 ** -9)
        nd, nq_ = (hd * hd).sum(1), (hq * hq).sum(1)
        self.eta = (err_q + err_d.max()) * (1 + 2.0 ** -10)
        S = 0.5 * (nq_ + nd.max()) + np.sqrt(nq_ * nd.max())
        self.sigma = S / 16384.0
        r2 = float(np.float32(np.float32(r) * np.float32(r)))
        m = len(db); nch = (m + CHUNK - 1) // CHUNK
        self.cls = []          # per query: "two", "third", "undecided", "dropped" (pre-test) or "either"
        self.certain, self.possible = 0, 0
        for b0 in range(0, len(q), block):
            F = nq_[b0:b0 + block, None] + nd[None, :] - 2.0 * hq[b0:b0 + block] @ hd.T           # filter value ||fp16(a) - fp16(b)||^2
            T = (q[b0:b0 + block] ** 2).sum(1)[:, None] + (db * db).sum(1)[None, :] - 2.0 * q[b0:b0 + block] @ db.T   # reference distance
            T = np.maximum(T, 0.0)
            pad = nch * CHUNK - m
            Fc = np.pad(F, ((0, 0), (0, pad)), constant_values=np.inf).reshape(len(F), nch, CHUNK)
            Tc = np.pad(T, ((0, 0), (0, pad)), constant_values=np.inf).reshape(len(T), nch, CHUNK)
            cmF, cmT = Fc.min(2), Tc.min(2)
            order = np.argsort(cmF, axis=1, kind="stable")
            for k in range(len(F)):
                self._classify(b0 + k, cmF[k], cmT[k], order[k], np.sort(T[k])[1], r2)
        self.cls = np.array(self.cls)

    def _classify(self, qi, cmF, cmT, order, s2, r2):
        sig, eta = self.sigma[qi], self.eta[qi]
        rel = 2.0 ** -16                                  # the reference's own float summation against the float64 distance

        def lower(x):
            v = np.maximum(np.sqrt(np.maximum(x - sig, 0.0)) - eta, 0.0)
            return v * v * (1 - 2.0 ** -16)

        def upper(x):
            v = np.sqrt(x * (1 + 2.0 ** -9) + sig) + eta
            return v * v * (1 + 2.0 ** -16)

        v = [cmF[order[k]] if k < len(order) else np.inf for k in range(4)]
        lo = [max(x - sig, 0.0) * (1 - 2.0 ** -10) for x in v]        # what the device's packed minimum may be
        hi = [x + sig for x in v]
        s2_lo = s2 * (1 - rel)

        def u_of(x, k):
            """An upper bound of the second smallest distance among the rows of any k chunks whose filter minima are <= x: the
            (k - 1)-th largest reference chunk minimum among those chunks (the middle one of three chosen is at most the second largest)."""
            sel = np.sort(cmT[cmF <= x])
            return sel[-(k - 1)] * (1 + rel) if len(sel) >= k else np.inf

        pre_certain = lower(hi[0]) < r2 * upper(lo[1]) * (1 - 1e-6)
        pre_possible = lower(lo[0]) < r2 * upper(hi[1]) * (1 + 1e-6)
        und_certain = pre_certain and lower(hi[3]) < s2_lo
        und_possible = pre_possible and lower(lo[3]) < u_of(hi[2], 3)
        third_certain = pre_certain and lower(hi[2]) < s2_lo and not und_possible
        two_certain = pre_certain and lower(lo[2]) >= u_of(hi[1], 2)
        self.certain += und_certain
        self.possible += und_possible
        self.cls.append("undecided" if und_certain else "third" if third_certain else "two" if two_certain
                        else "dropped" if not pre_possible else "either")


# ---------------------------------------------------------------------------------------------- constructions
def skeleton(rng, n=128):
    """An fp16-exact row in [64, 128): multiples of 1/16."""
    return (64 + rng.integers(0, 64 * 16 - 64, n) / 16.0).astype(np.float64)


def planted_query(rng, twins=3, clear_best=True, last_bits=False):
    """One query and its planted rows (the query first, then the rows in the chunk order they must take):
    clear_best: A at distance 128 (fp16-exact), then the fp16 twins B, C, D ... = s - j * eps on the 64 components where s = q + 2,
    distance ~256, the later twin truly closer.  Without a clear best: s = q + 0.5, twins at exactly equal distance (eps = 1/64: every partial sum is
    exact) or, last_bits, twins whose distances differ by j * 2^-12 * ~1 (a few float ulps)."""
    q = skeleton(rng)
    comps = rng.permutation(128)[:64]
    s = q.copy(); s[comps] += 2.0 if clear_best else 0.5      # without a clear best: distances ~16, deep inside sigma
    rows = []
    if clear_best:
        a = q.copy(); a[rng.permutation(128)[:32]] += 2.0
        rows.append(a)
        for j in range(twins):
            rows.append(s - 0.01 * j * (np.arange(128)[:, None] == comps[None, :]).any(1))
    else:
        for j in range(twins):
            t = s.copy()
            if last_bits:
                t[comps[:4]] -= 0.01
                t[comps[4 + j]] -= j * 2.0 ** -12
            else:
                t[comps[16 * (j % 4):16 * (j % 4) + 16]] -= 1.0 / 64.0
            rows.append(t)
    for x in rows[1 if clear_best else 0:]:
        assert np.array_equal(fp16(x), s)                    # twins: one fp16 row
    return q, rows


def far_rows(rng, n):
    """Rows at distance >= ~2000 from every planted query: fp16-exact skeleton rows elsewhere in [64, 128)."""
    return np.stack([skeleton(rng) for _ in range(n)])


def build_pair(rng, planted, n_chunks_min=8, extra_queries=None, extra_rows=None):
    """Database and queries for a list of planted (query, rows): planted row j of query k in chunk (k * width + j), row k % 16 inside it;
    the other rows of the database are far skeleton rows (or `extra_rows`), the queries are the planted ones then `extra_queries`."""
    width = max(len(r) for _, r in planted)
    n_chunks = max(n_chunks_min, width * len(planted) + 2)
    db = far_rows(rng, n_chunks * CHUNK)
    if extra_rows is not None:
        fill = np.setdiff1d(np.arange(len(db)), [16 * (k * width + j) + k % 16 for k, (_, rs) in enumerate(planted) for j in range(len(rs))])
        db[fill[:len(extra_rows)]] = extra_rows[:len(fill)]
    for k, (_, rs) in enumerate(planted):
        for j, x in enumerate(rs):
            db[16 * (k * width + j) + k % 16] = x
    qs = np.stack([p[0] for p in planted])
    if extra_queries is not None:
        qs = np.concatenate([qs, extra_queries])
    return db.astype(np.float32), qs.astype(np.float32)


def sift_real(n, seed):
    d, _ = synth.sift_images(2, n, np.float32, seed=seed, pool_factor=1.0)
    return synth.real_valued(d, seed=seed)


def noise_view(rng, m, s=0.25):
    return (150 + rng.normal(0, s, (m, 128))).astype(np.float32)


def case_third_chunk(seed=1):
    rng = np.random.default_rng(seed)
    return build_pair(rng, [planted_query(rng, twins=2) for _ in range(20)])


def case_undecided_kept(seed=2):
    rng = np.random.default_rng(seed)
    return build_pair(rng, [planted_query(rng, twins=3) for _ in range(20)])


def case_undecided_dropped(seed=3, last_bits=False):
    rng = np.random.default_rng(seed)
    return build_pair(rng, [planted_query(rng, twins=4, clear_best=False, last_bits=last_bits) for _ in range(20)])


def case_per_pair(k, seed=4):
    """k planted undecided queries among SIFT-like real-valued queries that the filter decides."""
    rng = np.random.default_rng(seed + k)
    a, b = sift_real(600, seed + k)
    return build_pair(rng, [planted_query(rng, twins=3) for _ in range(k)], n_chunks_min=40, extra_queries=b, extra_rows=a)


# ---------------------------------------------------------------------------------------------- CPU: every construction falls in its class
def test_model_classifies_the_constructions():
    for build, cls in ((case_third_chunk, "third"), (case_undecided_kept, "undecided"), (case_undecided_dropped, "undecided")):
        db, q = build()
        m = Model(db, q, 0.8)
        assert (m.cls == cls).all(), (build.__name__, m.cls)
    db, q = case_undecided_dropped(last_bits=True)
    assert (Model(db, q, 1.0).cls == "undecided").all()


def test_twins_place_the_true_second_neighbour():
    """The answers of the constructions depend on the branch: the third-chunk case's second neighbour is the later twin (the earlier
    one if the third chunk were skipped), the undecided-kept case's is the fourth chunk's twin, the equal twins tie exactly, and the
    last-bit twins differ."""
    rng = np.random.default_rng(9)
    for twins in (2, 3):
        q, rows = planted_query(rng, twins=twins)
        d = ref_l2(q, np.stack(rows))
        assert d[0] == 128 and (np.diff(d[1:]) < 0).all() and d[0] < np.float32(0.64) * d[-1]
    q, rows = planted_query(rng, twins=4, clear_best=False)
    assert len(set(ref_l2(q, np.stack(rows)).tolist())) == 1
    q, rows = planted_query(rng, twins=4, clear_best=False, last_bits=True)
    d = ref_l2(q, np.stack(rows))
    assert len(set(d.tolist())) > 1 and np.abs(d / d.min() - 1).max() < 1e-4


@pytest.mark.parametrize("k", [1, 5, 65])
def test_model_counts_the_planted_undecided_queries(k):
    db, q = case_per_pair(k)
    m = Model(db, q, 0.8)
    assert m.certain == k and (m.cls[:k] == "undecided").all()
    assert m.possible - k <= 0.02 * (len(q) - k), (m.certain, m.possible)     # a few SIFT-like queries sit within the model's margin


def test_model_everything_undecided():
    rng = np.random.default_rng(5)
    db, q = noise_view(rng, 1000), noise_view(rng, 300)
    m = Model(db, q, 0.8)
    assert (m.sigma > 300).all() and m.certain > 0.9 * len(q) and m.possible == len(q)
    assert Model(db[:50], q, 0.8).possible == len(q)            # 4 chunks, the last one partial
    assert Model(db[:48], q, 0.8).possible == 0                 # 3 chunks: no fourth minimum, decided after the third


# ---------------------------------------------------------------------------------------------- GPU
def _has_cuda_device():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


gpu = pytest.mark.skipif(not _has_cuda_device(), reason="needs a CUDA device (an H100)")

RUNS = {"fused": "0", "stand_alone": "1000000000"}   # B200M_REAL_FUSED_ROWS: in-kernel re-scoring from 0 database rows, or never


def fresh_context(fused_rows):
    old = os.environ.get("B200M_REAL_FUSED_ROWS")
    os.environ["B200M_REAL_FUSED_ROWS"] = fused_rows
    try:
        return matching.Context(0)
    finally:
        if old is None:
            os.environ.pop("B200M_REAL_FUSED_ROWS", None)
        else:
            os.environ["B200M_REAL_FUSED_ROWS"] = old


def as_dict(res):
    pid, off, mat = res
    return {(int(a), int(b)): mat[off[k]:off[k + 1]] for k, (a, b) in enumerate(pid.tolist()) if off[k + 1] > off[k]}


def assert_same(got, want, what):
    assert sorted(got) == sorted(want), f"{what}: pairs {sorted(set(got) ^ set(want))[:8]} differ"
    for k in want:
        for f in ("i", "j", "dist", "ratio"):
            assert np.array_equal(got[k][f], want[k][f]), f"{what}: {f} differs for pair {k}"


def run(ora, descs, pairs, run_name, ratios=(0.8,), cross=False, n_real=None, log=None):
    """One context of the run's kind: every ratio against the oracle, the real-valued pair count, no exactness error, and the fallback
    count inside the model's bounds.  Returns the fallback counts."""
    ctx = fresh_context(RUNS[run_name])
    rng = np.random.default_rng(0)
    xys = [synth.positions(len(d), rng) for d in descs]
    m = ImageCollectionMatcherB200(0.8, cross, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    directed = sorted({(int(a), int(b)) for a, b in pairs} | ({(int(b), int(a)) for a, b in pairs} if cross else set()))
    counts = []
    for r in ratios:
        what = f"{run_name} r={r} cross={cross}"
        m.distRatio = r
        got = as_dict(m.match_uploaded(np.asarray(pairs, np.uint32)))
        assert ctx.last_real_tc_pairs() == (len(directed) if n_real is None else n_real), what
        assert ctx.exactness_errors() == 0, what
        assert_same(got, ora.collection_match(descs, xys, pairs, r, cross), what)
        models = [Model(descs[a], descs[b], r) for a, b in directed]
        lo, hi = sum(x.certain for x in models), sum(x.possible for x in models)
        fb = ctx.last_fallback_rows()
        if log is not None:
            log.append((what, fb, lo, hi))
        print(f"{what}: fallback rows {fb}, model [{lo}, {hi}]")
        assert lo <= fb <= hi, (what, fb, lo, hi)
        counts.append(fb)
    ctx.close()
    return counts


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("run_name", list(RUNS))
def test_twin_branches(ora, run_name):
    """Third chunk, undecided and kept, undecided and dropped (also at ratio 1.0, decided by the last bit), as one pair each."""
    descs, pairs = [], []
    for db, q in (case_third_chunk(), case_undecided_kept(), case_undecided_dropped(), case_undecided_dropped(seed=6, last_bits=True)):
        pairs.append((len(descs), len(descs) + 1)); descs += [db, q]
    run(ora, descs, pairs, run_name, ratios=(0.8, 1.0))


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("run_name", list(RUNS))
def test_per_pair_fallback_counts(ora, run_name):
    """One pair with K planted undecided queries: groups of 4 with a remainder, an exactly full 64-slot list, the first overflow entries;
    with more than 64 the overflow kernel must have run.  Cross matching on the 65-query pair."""
    for k in (1, 3, 4, 5, 63, 64, 65, 200):
        db, q = case_per_pair(k)
        (fb,) = run(ora, [db, q], [(0, 1)], run_name)
        assert fb >= k
    db, q = case_per_pair(65)
    run(ora, [db, q], [(0, 1)], run_name, cross=True)


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("run_name", list(RUNS))
def test_everything_undecided(ora, run_name):
    """150 + N(0, 1/4): every query goes to the fallback.  8192 x 8192 (8128 overflow entries), ragged pairs with m_i = 1000 and
    m_i = 50 (< 64, four chunks), and a self pair."""
    rng = np.random.default_rng(7)
    big = [noise_view(rng, 8192), noise_view(rng, 8192)]
    (fb,) = run(ora, big, [(0, 1)], run_name)
    assert fb > FB_PER_PAIR
    small = [noise_view(rng, 1000), noise_view(rng, 50), noise_view(rng, 300)]
    run(ora, small, [(0, 2), (1, 2), (0, 0)], run_name, ratios=(0.8, 1.0))


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("run_name", list(RUNS))
def test_mixed_storage(ora, run_name):
    """An integer-valued database view (stored as uchar) against real-valued queries whose rows are all undecided (the fallback's
    converting tile load), and the reverse direction (the query side read through view_elem)."""
    rng = np.random.default_rng(8)
    ints = np.rint(150 + rng.normal(0, 1, (700, 128))).astype(np.float32)
    reals = noise_view(rng, 300)
    run(ora, [ints, reals], [(0, 1), (1, 0)], run_name)


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("run_name", list(RUNS))
def test_more_than_one_batch(ora, run_name):
    """More than PAIR_CAP directed pairs of small real-valued views, each with a few rows every query of which is undecided: the two
    per-batch buffer sets must not leak fallback lists or counters into each other."""
    rng = np.random.default_rng(9)
    n = 66
    sift = sift_real(40 * n, 10)[0]
    descs = []
    for v in range(n):
        x = sift[40 * v:40 * v + 50].copy() if 40 * v + 50 <= len(sift) else sift[-50:].copy()
        x[[3, 19, 35, 48, 9, 25, 41, 49, 13, 29]] = noise_view(rng, 10)     # in all four chunks
        descs.append(np.ascontiguousarray(x))
    pairs = [(i, j) for i in range(n) for j in range(n) if i != j]
    assert len(pairs) > PAIR_CAP
    run(ora, descs, pairs, run_name)
