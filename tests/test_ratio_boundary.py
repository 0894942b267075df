"""The ratio test at its float32 boundary on every search path.

The reference keeps a match when  d1 < fl(fl(r * r) * d2)  for L2 (matching/filters.hpp:60 with Square(r) in float,
RegionsMatcher.hpp:150) and when  (float)d1 < fl(r * (float)d2)  for Hamming (ratio not squared).  Pairs of integer distances where
fl(r * r) * d2 rounds exactly onto d1, where a double product would land on the other side of d1, or where r * r squared in double
would change the outcome, decide whether a kernel uses the same float operations and the same strict comparison.  Random data
essentially never produces them, so the CPU part here finds them, builds descriptor sets whose best row sits at exactly d1 and whose
second row sits at exactly d2, and pins them to the oracle; the GPU part (run with -m gpu on an H100) sends the same sets through every
search path and compares each list with the oracle and with the float32 predicate."""
import os

import numpy as np
import pytest

import oracle
from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

RATIOS = (0.6, 0.8, 0.95, 1.0)
D2_MAX = 1 << 21            # stays inside every integer domain below (uchar, signed |v| <= 1024, quarter units)
HAMMING_BITS = 486          # AKAZE MLDB descriptors: 486 used bits of 64 bytes
DB_ROWS = 48                # three 16-row chunks


# ---------------------------------------------------------------------------------------------- finder
def l2_keeps(d1, d2, r):
    """The reference's L2 predicate in float32."""
    r = np.float32(r)
    return np.float32(d1) < np.float32(r * r) * np.float32(d2)


def hamming_keeps(d1, d2, r):
    return np.float32(d1) < np.float32(r) * np.float32(d2)


def l2_boundary_pairs(r, d2_max=D2_MAX, per_kind=3):
    """Integer (d1, d2), d1 <= d2 <= d2_max, of three kinds, the first `per_kind` hits of each (smallest d2 first):
    "exact":  fl(fl(r r) d2) == d1;
    "double": the float and the double product of the same float operands fall on different sides of d1;
    "square": r * r squared in double instead of float changes the outcome."""
    r32 = np.float32(r)
    rr = np.float32(r32 * r32)
    d2 = np.arange(1, d2_max + 1, dtype=np.int64)
    pf = (rr * d2.astype(np.float32)).astype(np.float64)          # float product
    pd = np.float64(rr) * d2.astype(np.float64)                    # double product of the same operands (exact here)
    psq = (np.float64(r32) * np.float64(r32)) * d2                 # r squared in double
    return {"exact": _exact(pf, d2, per_kind), "double": _between(pf, pd, d2, per_kind), "square": _between(pf, psq, d2, per_kind)}


def _exact(pf, d2, n):
    hit = (pf == np.floor(pf)) & (pf <= d2)
    return [(int(a), int(b)) for a, b in zip(pf[hit], d2[hit])][:n]


def _between(pf, px, d2, n):
    """The integers d1 <= d2 with (d1 < pf) != (d1 < px): d1 in [min, max) of the two products."""
    c = np.ceil(np.minimum(pf, px))
    hit = (c < np.maximum(pf, px)) & (c <= d2)
    return [(int(a), int(b)) for a, b in zip(c[hit], d2[hit])][:n]


def hamming_boundary_pairs(r, dmax=HAMMING_BITS, per_kind=3):
    """The same kinds for Hamming distances (ratio not squared): "exact" fl(r d2) == d1, "double" float vs double product."""
    r32 = np.float32(r)
    d2 = np.arange(1, dmax + 1, dtype=np.int64)
    pf = (r32 * d2.astype(np.float32)).astype(np.float64)
    return {"exact": _exact(pf, d2, per_kind), "double": _between(pf, np.float64(r32) * d2, d2, per_kind)}


def fixture_pairs(hamming=False):
    """(r, d1, d2) to realise: every hit of the finder and its two integer neighbours d1 - 1, d1 + 1 (one of which flips the outcome)."""
    out = []
    for r in RATIOS:
        kinds = hamming_boundary_pairs(r, per_kind=2) if hamming else l2_boundary_pairs(r, per_kind=2)
        for hits in kinds.values():
            for d1, d2 in hits:
                for a in (d1 - 1, d1, d1 + 1):
                    if 0 <= a <= d2 and (r, a, d2) not in out:
                        out.append((r, a, d2))
    return out


def test_finder_hits_the_known_float_facts():
    """The first hits are the float32 facts the kernels must reproduce (computed independently of the finder)."""
    assert {(9, 25), (18, 50), (36, 100)} <= set(l2_boundary_pairs(0.6, per_kind=50)["exact"])
    assert {(361, 400), (722, 800)} <= set(l2_boundary_pairs(0.95, per_kind=50)["exact"])
    assert not any(l2_keeps(d1, d2, 0.6) for d1, d2 in [(9, 25), (18, 50), (36, 100)])
    assert not any(l2_keeps(d1, d2, 0.95) for d1, d2 in [(361, 400), (722, 800)])
    assert l2_keeps(1015193, 1586239, 0.8) and not 1015193 < np.float64(np.float32(0.8)) ** 2 * 1586239
    assert all(not l2_keeps(d, d, 1.0) for d in (1, 7, 1 << 20))
    assert not hamming_keeps(3, 5, 0.6) and not hamming_keeps(4, 5, 0.8) and not hamming_keeps(19, 20, 0.95)
    for r in (0.6, 0.8, 0.95):
        r32 = np.float32(r); rr = np.float32(r32 * r32)
        kinds = l2_boundary_pairs(r)
        for d1, d2 in kinds["exact"]:
            assert np.float32(rr * np.float32(d2)) == d1 and not l2_keeps(d1, d2, r)
        for d1, d2 in kinds["double"]:
            assert l2_keeps(d1, d2, r) != (d1 < np.float64(rr) * d2)
        for d1, d2 in kinds["square"]:
            assert l2_keeps(d1, d2, r) != (d1 < np.float64(r32) ** 2 * d2)
        for d1, d2 in hamming_boundary_pairs(r)["exact"]:
            assert np.float32(r32 * np.float32(d2)) == d1 and not hamming_keeps(d1, d2, r)


# ---------------------------------------------------------------------------------------------- realiser
def squares(d, kmax):
    """Positive integers with sum of squares == d, each <= kmax (greedy; at most a few dozen terms below D2_MAX)."""
    out = []
    while d > 0:
        k = min(kmax, int(np.sqrt(d)))
        while k * k > d:
            k -= 1
        out.append(k); d -= k * k
    return out


def offset_row(base, d, kmax, lo, hi, rng):
    """base + a component offset whose squared norm is exactly d, every component inside [lo, hi]."""
    ks = squares(d, kmax)
    comps = rng.permutation(len(base))[:len(ks)]
    assert len(ks) <= len(base)
    row = base.copy()
    for c, k in zip(comps, ks):
        s = 1 if rng.random() < 0.5 else -1
        if not lo <= row[c] + s * k <= hi:
            s = -s
        row[c] += s * k
        assert lo <= row[c] <= hi
    assert int(((row - base) ** 2).sum()) == d
    return row


DOMAINS = {   # storage of one row as integers; value = integer * scale
    "u8": dict(dim=128, kmax=230, lo=0, hi=255, base=(0, 20), scale=1, dtype=np.uint8),
    "signed": dict(dim=128, kmax=1000, lo=-1024, hi=1024, base=(-20, 20), scale=1, dtype=np.float32),
    "real": dict(dim=128, kmax=1800, lo=-2000, hi=2000, base=(-40, 40), scale=0.25, dtype=np.float32),   # quarter units: fp16-exact
    "f64d": dict(dim=64, kmax=1000, lo=-1024, hi=1024, base=(-20, 20), scale=1, dtype=np.float32),
    "u144": dict(dim=144, kmax=230, lo=0, hi=255, base=(0, 20), scale=1, dtype=np.uint8),
}


def realise(cases, domain, seed, same_chunk):
    """One (database view, query view) per case (r, d1, d2): the query, in the database the best row at exactly d1 and the second at exactly
    d2 (units of scale^2), every other row at d2 + max(d2 // 2, 16).  same_chunk: both rows in chunk 1, else in chunks 2 and 0."""
    D = DOMAINS[domain]
    rng = np.random.default_rng(seed)
    descs = []
    for (r, d1, d2) in cases:
        q = rng.integers(D["base"][0], D["base"][1] + 1, D["dim"]).astype(np.int64)
        if domain == "real":
            q[rng.integers(0, D["dim"])] |= 1                                    # at least one non-integer value: a real-valued view
        far = d2 + max(d2 // 2, 16)
        db = np.stack([offset_row(q, far, D["kmax"], D["lo"], D["hi"], rng) for _ in range(DB_ROWS)])
        ia, ib = (20, 27) if same_chunk else (37, 5)
        db[ia] = offset_row(q, d1, D["kmax"], D["lo"], D["hi"], rng)
        db[ib] = offset_row(q, d2, D["kmax"], D["lo"], D["hi"], rng)
        descs += [(db * D["scale"]).astype(D["dtype"]), (q[None] * D["scale"]).astype(D["dtype"])]
    return descs


def realise_hamming(cases, seed, same_chunk):
    rng = np.random.default_rng(seed)
    descs = []
    for (r, d1, d2) in cases:
        q = rng.integers(0, 2, 512, dtype=np.uint8); q[HAMMING_BITS:] = 0
        def at(d):
            v = q.copy(); v[rng.permutation(HAMMING_BITS)[:d]] ^= 1
            return v
        far = min(HAMMING_BITS, d2 + max(d2 // 2, 16))
        assert far > d2
        db = np.stack([at(far) for _ in range(DB_ROWS)])
        ia, ib = (20, 27) if same_chunk else (37, 5)
        db[ia], db[ib] = at(d1), at(d2)
        descs += [np.packbits(db, axis=1, bitorder="little"), np.packbits(q[None], axis=1, bitorder="little")]
    return descs


def xys_for(descs, seed):
    rng = np.random.default_rng(seed)
    return [synth.positions(len(d), rng) for d in descs]


def expected(cases, hamming=False, scale=1.0):
    """{(I, J): (d1, keep)} of the float32 predicate, view 2k = database, 2k + 1 = query."""
    out = {}
    for k, (r, d1, d2) in enumerate(cases):
        f1, f2 = np.float32(d1 * scale * scale), np.float32(d2 * scale * scale)
        out[(2 * k, 2 * k + 1)] = (f1, bool(hamming_keeps(f1, f2, r) if hamming else l2_keeps(f1, f2, r)))
    return out


def check_against_predicate(lists, cases, r, hamming=False, scale=1.0):
    """The lists of one ratio: exactly the cases of that ratio the predicate keeps, each at distance d1 with ratio d1 / d2."""
    want = {k: v for k, v in expected(cases, hamming, scale).items() if cases[k[0] // 2][0] == r}
    kept = {k for k, (_, keep) in want.items() if keep}
    assert {k for k in lists if k in want} == kept
    for k in kept:
        assert len(lists[k]) == 1 and lists[k]["dist"][0] == want[k][0] and lists[k]["j"][0] == 0


def pairs_of(cases, r=None):
    return np.array([(2 * k, 2 * k + 1) for k, c in enumerate(cases) if r is None or c[0] == r], np.uint32)


def test_realised_fixtures_cover_every_kind():
    """Every ratio has fixtures, the three L2 kinds and the two Hamming kinds occur, and kept and dropped cases both occur."""
    for hamming in (False, True):
        cases = fixture_pairs(hamming)
        assert {c[0] for c in cases} == set(RATIOS)
        keeps = [bool(hamming_keeps(d1, d2, r) if hamming else l2_keeps(d1, d2, r)) for r, d1, d2 in cases]
        assert any(keeps) and not all(keeps)
    for r in RATIOS[:3]:
        assert all(l2_boundary_pairs(r)[k] for k in ("exact", "double", "square"))
        assert all(hamming_boundary_pairs(r)[k] for k in ("exact",))
    assert any(hamming_boundary_pairs(r)["double"] for r in RATIOS)


@pytest.mark.parametrize("domain", list(DOMAINS))
def test_realiser_builds_exact_distances(domain):
    D = DOMAINS[domain]
    cases = fixture_pairs()
    descs = realise(cases, domain, 11, same_chunk=False)
    for k, (r, d1, d2) in enumerate(cases):
        db = descs[2 * k].astype(np.float64) / D["scale"]; q = descs[2 * k + 1].astype(np.float64)[0] / D["scale"]
        d = ((db - q) ** 2).sum(1)
        assert d[37] == d1 and d[5] == d2 and (np.delete(d, [5, 37]) > d2).all()
    if domain == "real":
        for x in descs:
            assert np.array_equal(x.astype(np.float16).astype(np.float32), x) and np.abs(x).max() < 512
        assert not np.array_equal(descs[0], np.rint(descs[0]))
    elif D["dtype"] == np.float32:
        assert max(np.abs(x).max() for x in descs) <= 1024
    if domain in ("u8", "signed", "real"):      # the tensor-core domain: ||v||^2 < 2^22
        assert max(((x.astype(np.float64)) ** 2).sum(1).max() for x in descs) < 1 << 22


def undecided_boundary_pair(seed, copies=10):
    """One pair in which every query is undecided (real-valued filter) and most queries sit on the ratio boundary.  Database: 1024 rows
    of 150 + N(0, 1), then per query its best row at exactly d1 and its second at exactly d2 (quarter units around 150: fp16-exact, exact
    float distances in units of 1/16).  Queries: `copies` of every boundary case whose d2 / 16 stays below the background distances
    (~180), each on its own base.  sigma ~ 350 exceeds every distance, so every query goes to the fallback: far more than 64 of them,
    so both the per-pair list and the overflow list decide boundary cases.  Returns (db, queries, cases)."""
    rng = np.random.default_rng(seed)
    cases = [c for c in fixture_pairs() if c[2] <= 800] * copies
    db = [(150 + rng.normal(0, 1, (1024, 128))).astype(np.float32)]
    qs = []
    for (r, d1, d2) in cases:
        q = 600 + rng.integers(-8, 9, 128).astype(np.int64)
        q[rng.integers(0, 128)] |= 1
        rows = np.stack([offset_row(q, d1, 60, 520, 680, rng), offset_row(q, d2, 60, 520, 680, rng)])
        db.append((rows * 0.25).astype(np.float32)); qs.append(q * 0.25)
    perm = np.random.default_rng(seed + 1).permutation(1024 + 2 * len(cases))
    db = np.concatenate(db)[perm]
    return np.ascontiguousarray(db), np.stack(qs).astype(np.float32), cases


def test_undecided_boundary_construction():
    db, q, cases = undecided_boundary_pair(61)
    assert len(q) > 2 * 64 and {c[0] for c in cases} >= {0.6, 0.95, 1.0}
    for x in (db, q):
        assert np.abs(x).max() < 256 and fp16_norm_max(x) < 1 << 22
    assert np.array_equal(q.astype(np.float16).astype(np.float32), q)
    d = ((q.astype(np.float64)[:, None, :] - db.astype(np.float64)[None]) ** 2).sum(2)
    top = np.sort(d, 1)
    assert np.array_equal(top[:, 0] * 16, [c[1] for c in cases]) and np.array_equal(top[:, 1] * 16, [c[2] for c in cases])
    assert (top[:, 2] > 60).all()


def fp16_norm_max(x):
    h = x.astype(np.float16).astype(np.float64)
    return (h * h).sum(1).max()


def test_oracle_keeps_exactly_what_the_float_predicate_keeps(ora):
    """Pins the fixtures to the reference before any GPU runs: RegionsMatcher::Match through collection_match keeps exactly the pairs the
    float32 predicate keeps, with distance d1, for every ratio, L2 (integer and quarter-unit rows) and Hamming."""
    for domain, scale, same in (("u8", 1.0, True), ("signed", 1.0, False), ("real", 0.25, True)):
        cases = fixture_pairs()
        descs = realise(cases, domain, 21, same)
        xys = xys_for(descs, 21)
        for r in RATIOS:
            check_against_predicate(ora.collection_match(descs, xys, pairs_of(cases, r), r), cases, r, scale=scale)
    cases = fixture_pairs(hamming=True)
    descs = realise_hamming(cases, 22, True)
    xys = xys_for(descs, 22)
    for r in RATIOS:
        check_against_predicate(ora.collection_match(descs, xys, pairs_of(cases, r), r, False, True), cases, r, hamming=True)


# ---------------------------------------------------------------------------------------------- GPU: every search path
def _has_cuda_device():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


gpu = pytest.mark.skipif(not _has_cuda_device(), reason="needs a CUDA device (an H100)")


def as_dict(res):
    pid, off, mat = res
    return {(int(a), int(b)): mat[off[k]:off[k + 1]] for k, (a, b) in enumerate(pid.tolist()) if off[k + 1] > off[k]}


def assert_same(got, want, what=""):
    assert sorted(got) == sorted(want), f"{what}: pairs {sorted(set(got) ^ set(want))[:8]} differ"
    for k in want:
        for f in ("i", "j", "dist", "ratio"):
            assert np.array_equal(got[k][f], want[k][f]), f"{what}: {f} differs for pair {k}"


def fresh_context(env):
    """A context created under `env` (the context reads its switches at creation)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return matching.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def run_path(ctx, ora, descs, cases, counters, hamming=False, scale=1.0, what=""):
    """Every ratio through one context: the oracle's lists, the float32 predicate, the path counters and no exactness error."""
    t = EMatcherType.BRUTE_FORCE_HAMMING_B200 if hamming else EMatcherType.BRUTE_FORCE_L2_B200
    xys = xys_for(descs, 5)
    m = ImageCollectionMatcherB200(0.8, False, t, ctx)
    m.upload({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    m.wait_uploads()
    P = ora if descs[0].shape[1] in (64 if hamming else 128,) else oracle.Oracle("port")   # the compiled reference is 128-D only
    for r in RATIOS:
        pairs = pairs_of(cases, r)
        m.distRatio = r
        got = as_dict(m.match_uploaded(pairs))
        for name, want in counters(len(pairs)).items():
            assert getattr(ctx, name)() == want, f"{what} r={r}: {name}"
        assert ctx.exactness_errors() == 0, f"{what} r={r}"
        assert_same(got, P.collection_match(descs, xys, pairs, r, False, hamming), f"{what} r={r}")
        check_against_predicate(got, cases, r, hamming, scale)


def tc(n): return {"last_tc_pairs": n, "last_u8_tc_pairs": 0, "last_real_tc_pairs": 0}
def u8(n): return {"last_tc_pairs": n, "last_u8_tc_pairs": n, "last_real_tc_pairs": 0}
def real(n): return {"last_tc_pairs": 0, "last_real_tc_pairs": n}
def none(n): return {"last_tc_pairs": 0, "last_real_tc_pairs": 0}


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("same_chunk", [True, False], ids=["same_chunk", "two_chunks"])
def test_integer_paths(ora, same_chunk):
    """The u8 kernel (uchar views), the fp16 kernel on signed integer views under variant 4 and variants 1-3, and the exact CUDA-core
    kernels (f32 and u8) decide every boundary pair as the reference does."""
    cases = fixture_pairs()
    du8 = realise(cases, "u8", 31, same_chunk)
    dsg = realise(cases, "signed", 32, same_chunk)
    ctx = matching.Context(0)
    run_path(ctx, ora, du8, cases, u8, what="u8 kernel")
    run_path(ctx, ora, dsg, cases, tc, what="fp16 kernel")
    for v in (1, 2, 3):
        ctx.set_tc_variant(v)
        run_path(ctx, ora, dsg, cases, tc, what=f"fp16 kernel, variant {v}")
    ctx.set_tc_variant(4)
    ctx.set_force_exact(True)
    run_path(ctx, ora, dsg, cases, none, what="exact f32")
    run_path(ctx, ora, du8, cases, none, what="exact u8")
    ctx.close()


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "stand_alone"])
def test_real_valued_paths(ora, fused):
    """Quarter-unit rows (fp16-exact, exact float distances in units of 1/16) on the real-valued filter, re-scoring fused and stand-alone,
    with the two rows in one chunk and in two."""
    ctx = fresh_context({"B200M_REAL_FUSED_ROWS": "0" if fused else "1000000000"})
    cases = fixture_pairs()
    for same in (True, False):
        run_path(ctx, ora, realise(cases, "real", 41 + same, same), cases, real, scale=0.25, what=f"real same_chunk={same}")
    ctx.close()


@pytest.mark.gpu
@gpu
def test_hamming_and_generic_paths(ora):
    """The Hamming kernel (ratio not squared) and the generic exact kernel (float 64-D, uchar 144-D)."""
    ctx = matching.Context(0)
    hc = fixture_pairs(hamming=True)
    for same in (True, False):
        run_path(ctx, ora, realise_hamming(hc, 51 + same, same), hc, none, hamming=True, what=f"hamming same_chunk={same}")
    cases = fixture_pairs()
    run_path(ctx, ora, realise(cases, "f64d", 53, False), cases, none, what="generic float 64-D")
    run_path(ctx, ora, realise(cases, "u144", 54, True), cases, none, what="generic uchar 144-D")
    ctx.close()


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "stand_alone"])
def test_real_valued_fallback_kernels(ora, fused):
    """Boundary pairs among queries that are all undecided: both fallback kernels (per-pair list and overflow list) apply the ratio test."""
    db, q, cases = undecided_boundary_pair(61)
    ctx = fresh_context({"B200M_REAL_FUSED_ROWS": "0" if fused else "1000000000"})
    xys = xys_for([db, q], 6)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({0: (db, xys[0]), 1: (q, xys[1])})
    m.wait_uploads()
    for r in (0.6, 0.95, 1.0):
        m.distRatio = r
        got = as_dict(m.match_uploaded(np.array([(0, 1)], np.uint32)))
        assert ctx.last_real_tc_pairs() == 1 and ctx.exactness_errors() == 0 and ctx.last_fallback_rows() == len(q), r
        assert_same(got, ora.collection_match([db, q], xys, [(0, 1)], r), f"r={r}")
        keep = {j for j, (rc, d1, d2) in enumerate(cases) if l2_keeps(np.float32(d1 / 16), np.float32(d2 / 16), r)}
        got_j = set(got[(0, 1)]["j"].tolist()) if (0, 1) in got else set()
        assert got_j == keep, r
    ctx.close()
