"""Vocabulary-tree producer at the shape AliceVision ships (vlfeat_K80L3.SIFT.tree: 80 children per node, 512,000 words), on
posting lists longer than a warp and on hundreds of documents.

References written here from the definitions, numpy and fractions only (no oracle code):
* `quantize_ref`: VocabularyTree::quantize (voctree/VocabularyTree.hpp:169-196) with L2 (voctree/distance.hpp:24-37): children in
  ascending order up to the first invalid one, diff = double(a) - double(c), each square rounded on its own and the squares summed
  in index order, strict '<' against DBL_MAX;
* the integer scores (commonPoints, strongCommonPoints, classic) from Counters, and inversedWeightedCommonPoints in float32 over the
  common words in ascending word id (VocabularyTree.cpp:192-247).
Every scene asserts, from its own data, the structure it exists for: children past 32 and 64, a first invalid child in every 32-wide
chunk, ties within one lane and across lanes, near-ties that only the summation order decides, posting lists longer than 64
documents, more than 256 documents.  Every deliberate fault of the references changes a result on the scenes.
CPU: the references equal the port oracle; the port equals the compiled reference at K = 33, 64 and 80 (L = 2 and 3), stored in
tests/golden/reference_outputs.npz for machines without the reference.  GPU (-m gpu): K5 (`quantize_kernel`), K6
(`score_postings_kernel`) and K6b (`doc_starts_kernel`, `weighted_pairs_kernel`) equal the references and the oracle bit for bit."""
import collections
import functools
import os
from concurrent.futures import ThreadPoolExecutor
from fractions import Fraction

import numpy as np
import pytest

import oracle
from alicevision_b200 import synth

F32 = np.float32
DBL_MAX = np.finfo(np.float64).max
METHODS = ["strongCommonPoints", "commonPoints", "classic", "inversedWeightedCommonPoints"]
FIRST_INVALID = (0, 31, 32, 33, 63, 64, 79)          # chunk 1 (0, 31), chunk 2 (32, 33, 63), chunk 3 (64, 79)
SAME_LANE = ((5, 37), (6, 70), (40, 72))              # lane l evaluates children l, l + 32, l + 64: one lane holds both
CROSS_LANE = ((31, 32), (10, 43), (3, 68), (33, 66))  # two lanes, one child each
NEAR_TIE_AT = ((2, 34), (9, 73), (4, 37), (45, 78), (30, 63))


# ---------------------------------------------------------------------------------------------- references
def _pairwise(t):
    while t.shape[-1] > 1:
        t = t[..., 0::2] + t[..., 1::2]
    return t[..., 0]


def _dists(x, C, fault):
    """(m, d) rows against (m, k, d) centres -> (m, k) distances in the reference's operation order (or a faulty one)."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _dists_unchecked(x, C, fault)


def _dists_unchecked(x, C, fault):
    if fault == "float32":
        diff = np.subtract(x.astype(F32)[:, None, :], C, dtype=F32)
        return np.add.accumulate(np.multiply(diff, diff), axis=-1, dtype=F32)[..., -1]
    diff = np.subtract(x.astype(np.float64)[:, None, :], C, dtype=np.float64)
    sq = np.multiply(diff, diff, out=diff)
    if fault == "pairwise":
        return _pairwise(sq)
    if fault == "reversed":
        sq = sq[..., ::-1]
    return np.add.accumulate(sq, axis=-1, out=sq)[..., -1]


def _descend(k, levels, centers, valid, x, fault):
    n = len(x)
    ar = np.arange(k)
    idx = np.full(n, -1, np.int64)
    chosen = np.zeros((n, levels), np.int64); limit = np.zeros((n, levels), np.int64)
    for level in range(levels):
        first = (idx + 1) * k
        nodes = first[:, None] + ar
        v = valid[nodes].astype(bool)
        lim = np.where(v.all(1), k, np.argmin(v, axis=1))                 # the first invalid child ends the scan
        eligible = v if fault == "skip_invalid" else ar[None, :] < lim[:, None]
        D = _dists(x, centers[nodes], fault)
        cand = eligible & ((D <= np.inf) if fault == "le_max" else (D < DBL_MAX))   # NaN is never below anything
        m = np.where(cand, D, np.inf).min(1)
        hit = cand & (D == m[:, None])
        pick = (k - 1 - np.argmax(hit[:, ::-1], 1)) if fault == "last_tie" else np.argmax(hit, 1)
        best = np.where(hit.any(1), pick, 0)                              # nothing below DBL_MAX: best_child stays first_child
        idx = first + best
        chosen[:, level] = best; limit[:, level] = lim
    return idx, chosen, limit


def quantize_ref(k, levels, centers, valid, descs, fault=None, path=False, chunk=256):
    """VocabularyTree::quantize for every row.  fault: None, or one deliberate error ("pairwise", "reversed", "float32" summation,
    "skip_invalid" children instead of stopping, "last_tie" index, "le_max": an infinite distance taken as a candidate).
    path=True also returns the child chosen and the scan limit at every level."""
    x = np.asarray(descs)
    word_start = sum(k ** (l + 1) for l in range(levels - 1))
    parts = [(s, x[s:s + chunk]) for s in range(0, len(x), chunk)]
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:               # numpy releases the GIL in its loops
        res = list(ex.map(lambda p: _descend(k, levels, centers, valid, p[1], fault), parts))
    if not res:
        res = [(np.zeros(0, np.int64), np.zeros((0, levels), np.int64), np.zeros((0, levels), np.int64))]
    words = (np.concatenate([r[0] for r in res]) - word_start).astype(np.int32)
    if path:
        return words, np.concatenate([r[1] for r in res]), np.concatenate([r[2] for r in res])
    return words


def exact_dist(a, c):
    """Squared L2 in rational arithmetic; classifies scenes, never the expected answer (the reference's rounding is the spec)."""
    return sum((Fraction(float(p)) - Fraction(float(q))) ** 2 for p, q in zip(a, c))


def count_scores(docs):
    """docs: {id: words}.  Returns ids (ascending), vocabulary, the count matrix and, for every ordered pair (diagonal included),
    commonPoints = sum min(c_a, c_b), strongCommonPoints = #{c_a = c_b = 1}, classic = n_a + n_b - 2 sum min."""
    ids = sorted(docs)
    cnt = [collections.Counter(np.asarray(docs[i]).tolist()) for i in ids]
    vocab = np.array(sorted(set().union(*cnt)), np.int64)
    col = {w: j for j, w in enumerate(vocab.tolist())}
    C = np.zeros((len(ids), len(vocab)), np.int64)
    for r, c in enumerate(cnt):
        for w, m in c.items():
            C[r, col[w]] = m
    common = np.stack([np.minimum(C[a], C).sum(1) for a in range(len(ids))]) if ids else np.zeros((0, 0), np.int64)
    ones = (C == 1).astype(np.int64)
    strong = ones @ ones.T
    nf = C.sum(1)
    return ids, vocab, C, common, strong, nf[:, None] + nf[None, :] - 2 * common


def weighted_scores(C, vocab, w, descending=False):
    """inversedWeightedCommonPoints score of every pair: (1.f / min(c_a, c_b)) * w[word] over the common words in ascending word id,
    accumulated in float32 (descending=True: the deliberate wrong order)."""
    n = len(C)
    S = np.zeros((n, n), F32)
    nz = C > 0
    for a in range(n):
        for b in range(a, n):
            both = nz[a] & nz[b]
            if both.any():
                t = (F32(1) / np.minimum(C[a, both], C[b, both]).astype(F32)) * w[vocab[both]]
                S[a, b] = S[b, a] = np.add.accumulate(t[::-1] if descending else t, dtype=F32)[-1]
    return S


def distances(method, common, strong, classic, wsc):
    """The `distance` Database::find ranks by, as float32: -score, or the classic L1 count."""
    if method == "inversedWeightedCommonPoints":
        return -wsc
    return {"commonPoints": -common.astype(F32), "strongCommonPoints": -strong.astype(F32), "classic": classic.astype(F32)}[method]


def check_weights(w, docs, num_words):
    """Database::computeTfIdfWeights: log(N / Ni) with the quotient of the float N and Ni, 1 for unused words; equal to
    float64 log of that quotient to within one float ulp."""
    ni = np.zeros(num_words, np.int64)
    for d in docs.values():
        ni[np.unique(np.asarray(d, np.int64))] += 1
    used = ni > 0
    q = F32(len(docs)) / ni[used].astype(F32)
    want = np.log(q.astype(np.float64))
    got = w[used].astype(np.float64)
    assert np.all(np.abs(got - want) <= np.spacing(np.abs(w[used])).astype(np.float64) + 1e-300)
    assert np.all(w[~used] == 1.0)


# ---------------------------------------------------------------------------------------------- scenes
Scene = collections.namedtuple("Scene", "name tree k levels centers valid descs words")


@functools.lru_cache(None)
def base_tree(k, levels):
    c, v = synth.vocabulary_tree(k, levels, seed=500 + k + levels)
    c.setflags(write=False); v.setflags(write=False)
    return c, v


@functools.lru_cache(None)
def sift_rows(n, seed):
    return synth.sift_images(1, n, np.uint8, seed=seed, pool_factor=1.0)[0][0]


def _scene(name, tree, k, levels, c, v, descs):
    return Scene(name, tree, k, levels, c, v, descs, [quantize_ref(k, levels, c, v, d) for d in descs])


def _below(k, levels, c, v, node, child, rng, noise=0.3):
    """A query near a descendant of `child` of `node` (-1 = the root): the centre of one of its children when there is a level
    below, else the child's own centre, plus real-valued noise."""
    n = (node + 1) * k + child
    first_of = lambda i: (i + 1) * k                                   # noqa: E731
    if first_of(n) < len(c):
        n = first_of(n) + int(rng.integers(k))
    return (c[n] + rng.normal(0, noise, c.shape[1])).astype(F32)


@functools.lru_cache(None)
def spread_scene(k):
    """A K-way L = 2 tree (SIFT-like centres): u8, integer-valued float and real-valued float rows."""
    c, v = base_tree(k, 2)
    u8 = sift_rows(3000, 40 + k)
    descs = [u8, u8.astype(F32), synth.real_valued([u8[:1500]], seed=k)[0]]
    s = _scene(f"spread{k}", ("base", k, 2), k, 2, c, v, descs)
    _, ch, _ = quantize_ref(k, 2, c, v, np.concatenate(descs[::2]), path=True)
    for level in range(2):
        assert (ch[:, level] == k - 1).any() and (k <= 32 or (ch[:, level] >= 32).any()) and (k <= 64 or (ch[:, level] >= 64).any())
    return s


@functools.lru_cache(None)
def big_scene():
    """The full K = 80, L = 3 tree: 10^5 u8 rows (and the same rows as integer-valued float), 2 x 10^4 real-valued rows, and
    0, 1, 3, 4, 5 rows (K5 runs 4 warps per block)."""
    c, v = base_tree(80, 3)
    assert len(c) == 518480 and c.nbytes > 265e6
    u8 = sift_rows(100000, 7)
    real = synth.real_valued([sift_rows(20000, 8)], seed=8)[0]
    descs = [real] + [u8[:n] for n in (0, 1, 3, 4, 5)] + [real[:n] for n in (1, 3, 4, 5)]
    s = _scene("big", ("base", 80, 3), 80, 3, c, v, descs)
    w = quantize_ref(80, 3, c, v, u8)
    s.descs.extend([u8, u8.astype(F32)]); s.words.extend([w, w])         # the same values: the same words
    _, ch, _ = quantize_ref(80, 3, c, v, u8[:20000], path=True)
    assert all((ch[:, level] >= 64).any() and len(np.unique(ch[:, level])) == 80 for level in range(3))
    assert len(np.unique(w)) > 20000
    return s


def _invalid_queries(k, levels, c, v, nodes, rng, per=12):
    """Queries whose truly nearest child of `node` lies after its first invalid child c0 (c0 = 79: the invalid child itself)."""
    q = []
    for node, c0 in nodes:
        for _ in range(per):
            after = c0 + 1 + int(rng.integers(k - 1 - c0)) if c0 < k - 1 else c0
            q.append(_below(k, levels, c, v, node, after, rng))
    return np.array(q, F32)


def _assert_first_invalid_hit(s, nodes_by_level):
    """Every (level, c0) is met by some row whose scan stops at c0 and whose word a kernel skipping the invalid child changes
    (c0 = 79: a kernel that evaluates the invalid child)."""
    x = s.descs[0]
    _, ch, lim = quantize_ref(s.k, s.levels, s.centers, s.valid, x, path=True)
    skip = quantize_ref(s.k, s.levels, s.centers, s.valid, x, fault="skip_invalid")
    allv = quantize_ref(s.k, s.levels, s.centers, np.ones_like(s.valid), x)
    for level, c0s in nodes_by_level.items():
        for c0 in c0s:
            rows = lim[:, level] == c0
            wrong = skip if c0 < s.k - 1 else allv
            assert (rows & (wrong != s.words[0])).any(), (s.name, level, c0)


@functools.lru_cache(None)
def invalid_scenes():
    """First invalid child at every c0 in FIRST_INVALID: at the root of seven K80 L2 trees, and under chosen nodes of levels 1 and
    2 of the K80 L3 tree; every other child valid, the query's nearest child after c0."""
    out = []
    rng = np.random.default_rng(11)
    c, v0 = base_tree(80, 2)
    for c0 in FIRST_INVALID:
        v = v0.copy(); v[c0] = 0
        x = _invalid_queries(80, 2, c, v, [(-1, c0)] * 2, rng)
        s = _scene(f"invalid_root{c0}", ("invalid_root", c0), 80, 2, c, v, [x, np.clip(np.rint(x), 0, 255).astype(np.uint8)])
        _assert_first_invalid_hit(s, {0: [c0]})
        out.append(s)
    c, v = base_tree(80, 3)
    v = v.copy()
    lvl1 = [(n, c0) for n, c0 in zip((3, 17, 29, 41, 52, 66, 77), FIRST_INVALID)]
    lvl2 = [(80 + 80 * g + h, c0) for (g, h), c0 in zip(((1, 70), (12, 33), (30, 2), (44, 64), (50, 31), (71, 40), (79, 79)), FIRST_INVALID)]
    for node, c0 in lvl1 + lvl2:
        v[(node + 1) * 80 + c0] = 0
    x = _invalid_queries(80, 3, c, v, lvl1 + lvl2, rng)
    s = _scene("invalid_deep", ("invalid_deep",), 80, 3, c, v, [x])
    _assert_first_invalid_hit(s, {1: FIRST_INVALID, 2: FIRST_INVALID})
    out.append(s)
    # a K80 L2 tree whose nodes keep between 1 and 80 valid children (a valid prefix, as in a trained tree)
    c, v = base_tree(80, 2)
    v = np.ones_like(v)
    cnt = rng.integers(1, 81, 81)
    cnt[:3] = 71, 1, 80                                  # the root keeps 71; node 0 one child, node 1 all 80
    for node in range(-1, 80):
        v[(node + 1) * 80 + cnt[node + 1]:(node + 2) * 80] = 0
    u8 = sift_rows(3000, 12)
    s = _scene("valid_prefix", ("valid_prefix",), 80, 2, c, v, [u8, synth.real_valued([u8[:1000]], seed=12)[0]])
    _, ch, lim = quantize_ref(80, 2, c, v, u8, path=True)
    assert cnt.min() == 1 and cnt.max() == 80 and (lim[:, 1] < 32).any() and ((lim[:, 1] > 32) & (lim[:, 1] < 64)).any() and ((lim[:, 1] > 64) & (lim[:, 1] < 80)).any()
    assert (ch[:, 0] >= 64).any() and (lim[:, 1] == 80).any()
    out.append(s)
    return out


@functools.lru_cache(None)
def tie_scene():
    """Bit-identical centres at SAME_LANE and CROSS_LANE pairs (i, j), i < j, at the root and under node 7: the lower index wins."""
    c, v = base_tree(80, 2)
    c = c.copy()
    rng = np.random.default_rng(13)
    q = []
    for i, j in SAME_LANE + CROSS_LANE:
        c[j] = c[i]
        c[8 * 80 + j] = c[8 * 80 + i]                    # children of node 7 start at (7 + 1) * 80
    for i, j in SAME_LANE + CROSS_LANE:
        q += [_below(80, 2, c, v, -1, i, rng) for _ in range(6)] + [_below(80, 2, c, v, 7, i, rng, noise=0.05) for _ in range(6)]
    x = np.array(q, F32)
    s = _scene("ties", ("ties",), 80, 2, c, v, [x, np.clip(np.rint(x), 0, 255).astype(np.uint8)])
    _, ch, _ = quantize_ref(80, 2, c, v, x, path=True)
    _, chl, _ = quantize_ref(80, 2, c, v, x, fault="last_tie", path=True)
    for level in range(2):
        for i, j in SAME_LANE + CROSS_LANE:
            assert ((ch[:, level] == i) & (chl[:, level] == j)).any(), (level, i, j)
    return s


def _near_tie(rng, dim=128, tries=4000):
    """A centre A, its copy B with two components swapped, and a real-valued query x with x_p = x_q: the exact distances tie, the
    reference's sequential sum ranks B first, pairwise and reversed summation rank A first."""
    while True:
        mag = 10.0 ** rng.uniform(-2, 4, (tries, dim))
        A = (rng.standard_normal((tries, dim)) * mag).astype(F32)
        x = (A + 0.1 * mag * rng.standard_normal((tries, dim))).astype(F32)
        p = rng.integers(0, dim // 2, tries); q = rng.integers(dim // 2, dim, tries)
        r = np.arange(tries)
        x[r, q] = x[r, p]
        B = A.copy(); B[r, p], B[r, q] = A[r, q], A[r, p]
        AB = np.stack([A, B], 1)
        d = {f: _dists(x, AB, f) for f in (None, "pairwise", "reversed")}
        ok = (d[None][:, 1] < d[None][:, 0]) & (d["pairwise"][:, 0] <= d["pairwise"][:, 1]) & (d["reversed"][:, 0] <= d["reversed"][:, 1])
        for t in np.flatnonzero(ok):
            if exact_dist(x[t], A[t]) == exact_dist(x[t], B[t]):
                return A[t], B[t], x[t]


@functools.lru_cache(None)
def near_tie_scene():
    """NEAR_TIE_AT pairs (a, b) at the root, in different chunks, one lane or two: exactly tied, decided by the rounding of the
    sequential sum in favour of b; the exact order, pairwise and reversed summation all pick a."""
    c, v = base_tree(80, 2)
    c = c.copy()
    rng = np.random.default_rng(17)
    q = []
    for a, b in NEAR_TIE_AT:
        c[a], c[b], x = _near_tie(rng)
        q.append(x)
    x = np.array(q, F32)
    s = _scene("near_ties", ("near_ties",), 80, 2, c, v, [x])
    _, ch, _ = quantize_ref(80, 2, c, v, x, path=True)
    for f in ("pairwise", "reversed"):
        _, chf, _ = quantize_ref(80, 2, c, v, x, fault=f, path=True)
        assert np.array_equal(chf[:, 0], [a for a, _ in NEAR_TIE_AT]), f
    assert np.array_equal(ch[:, 0], [b for _, b in NEAR_TIE_AT])
    for r, (a, b) in enumerate(NEAR_TIE_AT):
        assert exact_dist(x[r], c[a]) == exact_dist(x[r], c[b])          # exact order: a tie, the lower index a
    return s


@functools.lru_cache(None)
def nonfinite_scene():
    """Rows with NaN, +-inf and +-3e38 on the K80 L3 tree, u8 rows of all 0 and all 255; and a K80 L2 tree whose root child 0 has
    an infinite component, so that an infinite row sees NaN there and +inf everywhere else."""
    c, v = base_tree(80, 3)
    base = sift_rows(16, 19).astype(F32)
    rows = []
    for val in (np.nan, np.inf, -np.inf, 3e38, -3e38):
        r = base.copy()[:3]
        r[0, :] = val; r[1, 0] = val; r[2, 127] = val
        rows.append(r)
    alt = base[:1].copy(); alt[0, ::2] = 3e38; alt[0, 1::2] = -3e38
    x = np.concatenate(rows + [alt, base[3:]]).astype(F32)
    u8 = np.array([np.zeros(128), np.full(128, 255)] + list(base[:4]), np.uint8)
    s = _scene("nonfinite", ("base", 80, 3), 80, 3, c, v, [x, u8])
    assert s.words[0][0] == 0 and s.words[0][3] == 0                   # all-NaN, all-+inf rows: every level keeps its first child
    c2, v2 = base_tree(80, 2)
    c2 = c2.copy(); c2[0, 0] = np.inf
    y = sift_rows(8, 20).astype(F32); y[:4, 0] = np.inf
    s2 = _scene("inf_centre", ("inf_centre",), 80, 2, c2, v2, [y])
    assert (s2.words[0][:4] < 80).all() and (quantize_ref(80, 2, c2, v2, y, fault="le_max")[:4] >= 80).all()
    return [s, s2]


def quantiser_scenes(big=True):
    out = [spread_scene(k) for k in (31, 32, 33, 64, 80)] + invalid_scenes() + [tie_scene(), near_tie_scene()] + nonfinite_scene()
    return out + [big_scene()] if big else out


SCENE_NAMES = ["spread31", "spread32", "spread33", "spread64", "spread80", "invalid", "ties", "near_ties", "nonfinite", "big"]


def scenes_named(name):
    return {"invalid": invalid_scenes, "ties": lambda: [tie_scene()], "near_ties": lambda: [near_tie_scene()], "nonfinite": nonfinite_scene,
            "big": lambda: [big_scene()]}.get(name, lambda: [spread_scene(int(name[6:]))])()


@functools.lru_cache(None)
def word_db():
    """300 documents (three 128-wide block columns of K6b) under sparse, large ids on the 512,000-word vocabulary: empty documents
    first, in the middle and last in id order, a stop word in every other document, posting lists of exactly 31, 32, 33, 64 and 65
    documents, counts of 1 and above, documents of thousands of words."""
    rng = np.random.default_rng(23)
    ids = np.unique(np.r_[0, 0xFFFFFFFF, rng.choice(1 << 32, 400, replace=False)])[:299]
    ids = np.unique(np.r_[ids, 0xFFFFFFFF])
    assert len(ids) == 300
    n_words = 80 ** 3
    pool = rng.choice(n_words, 6000, replace=False)
    stop, exact = pool[:1], pool[1:6]
    pool = pool[6:]
    zipf = 1.0 / np.arange(1, len(pool) + 1) ** 0.9
    zipf /= zipf.sum()
    docs = {}
    for r, i in enumerate(ids):
        if r in (0, 150, 299):
            docs[int(i)] = np.zeros(0, np.int32)
            continue
        m = int(rng.choice([40, 200, 600, 4000], p=[0.3, 0.4, 0.25, 0.05]))
        docs[int(i)] = np.r_[rng.choice(pool, m, p=zipf), stop.repeat(rng.integers(1, 4))]
    full = [i for i in docs if len(docs[i])]
    for w, L in zip(exact, (31, 32, 33, 64, 65)):
        for i in rng.choice(full, L, replace=False):
            docs[int(i)] = np.r_[docs[int(i)], np.full(rng.integers(1, 3), w)]
    docs = {i: rng.permutation(d).astype(np.int32) for i, d in docs.items()}
    ids_, vocab, C, common, strong, classic = count_scores(docs)
    post = (C > 0).sum(0)
    assert len(ids_) > 256 and post.max() == 297 > 64 and all((post[np.searchsorted(vocab, w)] == L) for w, L in zip(exact, (31, 32, 33, 64, 65)))
    assert [r for r in range(300) if not C[r].any()] == [0, 150, 299] and ids_[0] == 0 and ids_[-1] == 0xFFFFFFFF
    assert (common != strong).any() and (C > 1).any() and max(len(d) for d in docs.values()) > 3000
    return docs


@functools.lru_cache(None)
def e2e_views(k, levels, n, m, seed):
    """n SIFT-like documents of about m rows from a shared pool, so that documents overlap; sparse ids, a few shorter documents
    (one empty) so that nmax = 1000 cuts some and not others."""
    descs, _ = synth.sift_images(n, m, np.uint8, seed=seed, pool_factor=1.0)
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(1 << 20, n, replace=False))
    d = {int(i): x for i, x in zip(ids, descs)}
    d[int(ids[3])] = d[int(ids[3])][:0]
    d[int(ids[n // 2])] = d[int(ids[n // 2])][:700]
    d[int(ids[-1])] = d[int(ids[-1])][:1000]
    return d


def e2e_scene():
    return e2e_views(80, 3, 64, 1500, 29)


@functools.lru_cache(None)
def e2e_words(nmax):
    c, v = base_tree(80, 3)
    d = e2e_scene()
    rows = [x[:nmax] if nmax else x for x in d.values()]
    w = quantize_ref(80, 3, c, v, np.concatenate(rows))
    out, o = {}, 0
    for i, x in zip(d, rows):
        out[i] = w[o:o + len(x)]; o += len(x)
    ids, vocab, C, *_ = count_scores(out)
    _, ch, _ = quantize_ref(80, 3, c, v, np.concatenate(rows)[:20000], path=True)
    assert (C > 0).sum(0).max() > 32 and all((ch[:, level] >= 64).any() for level in range(3))
    return out


@pytest.fixture(scope="module", autouse=True)
def _release_caches():
    yield
    for f in (base_tree, sift_rows, spread_scene, big_scene, invalid_scenes, tie_scene, near_tie_scene, nonfinite_scene, word_db, e2e_views, e2e_words):
        f.cache_clear()


def kind():
    return "ref" if oracle.VoctreeOracle.available("ref") else "port"


def ref_output(key, compute):
    live = oracle.VoctreeOracle.available("ref")
    return oracle.reference_output("voctree.scale." + key, compute if live else None, live)


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_quantize_ref_equals_port(name):
    P = oracle.VoctreeOracle("port")
    for s in scenes_named(name):
        for d, w in zip(s.descs, s.words):
            assert np.array_equal(P.quantize(s.k, s.levels, s.centers, s.valid, d), w), s.name


REF_ROWS = 4000


@pytest.mark.parametrize("name", ["spread33", "spread64", "spread80", "invalid", "ties", "near_ties", "nonfinite", "big"])
def test_port_equals_reference_quantize(name, tmp_path):
    """The compiled reference (its own VocabularyTree::load and quantize) on the quantiser scenes at K = 33, 64, 80, L = 2 and 3:
    live when built, else its stored words."""
    P = oracle.VoctreeOracle("port")
    R = oracle.VoctreeOracle("ref") if oracle.VoctreeOracle.available("ref") else None
    for s in scenes_named(name):
        for dt in (np.uint8, F32):
            parts = [d[:REF_ROWS] for d in s.descs if d.dtype == dt and len(d)]
            if not parts:
                continue
            x = np.concatenate(parts)
            got = ref_output(f"quantize.{s.name}.{np.dtype(dt).name}", lambda: R.quantize(s.k, s.levels, s.centers, s.valid, x, str(tmp_path / "t.tree")))
            assert np.array_equal(got, P.quantize(s.k, s.levels, s.centers, s.valid, x)), s.name
            assert np.array_equal(got, np.concatenate([w[:REF_ROWS] for d, w in zip(s.descs, s.words) if d.dtype == dt and len(d)]))


E2E = {"k33": (33, 2, 24, 400, 31), "k64": (64, 2, 24, 400, 37), "k80l3": (80, 3, 64, 1500, 29)}


@pytest.mark.parametrize("shape", sorted(E2E))
@pytest.mark.parametrize("method", METHODS)
def test_port_equals_reference_image_matching(shape, method, tmp_path):
    """populateDatabase + computeTfIdfWeights + find + convertAllMatchesToPairList: ranked ids, scores, weights and the pair list."""
    k, levels, n, m, seed = E2E[shape]
    c, v = base_tree(k, levels)
    d = e2e_views(k, levels, n, m, seed)
    P = oracle.VoctreeOracle("port")
    R = oracle.VoctreeOracle("ref") if oracle.VoctreeOracle.available("ref") else None
    for nmax, nq in ((0, 0), (1000, 10)):
        def stored(ids, mids, sc, w, pairs):
            # the weights do not depend on the method: stored with the first one; the unused words keep the default weight 1
            used = np.flatnonzero(w != 1.0) if method == METHODS[0] else np.zeros(0, np.int64)
            return ids, mids, sc, used, w[used], pairs
        a = ref_output(f"{shape}.{method}.{nmax}.{nq}", lambda: stored(*R.image_matching(k, levels, c, v, d, nmax, nq, method, str(tmp_path / "t.tree"))))
        ids, mids, sc, w, pairs = P.image_matching(k, levels, c, v, d, nmax, nq, method)
        for x, y in zip(a, stored(ids, mids, sc, w, pairs)):
            assert np.array_equal(x, y)
        assert len(pairs) > 0 and mids.shape == (n, nq or n)


@pytest.mark.parametrize("nmax", [0, 1000])
def test_references_equal_port_scores(nmax):
    """The Counter and float32 references give the port's (id -> distance) map for every query, its weights, and a ranking that
    is the port's wherever the distances do not tie."""
    c, v = base_tree(80, 3)
    d = e2e_scene()
    P = oracle.VoctreeOracle("port")
    docs = e2e_words(nmax)
    ids, vocab, C, common, strong, classic = count_scores(docs)
    for method in METHODS:
        qid, mids, sc, w, _ = P.image_matching(80, 3, c, v, d, nmax, 0, method)
        check_weights(w, docs, 80 ** 3)
        wsc = weighted_scores(C, vocab, w) if method == METHODS[3] else None
        D = distances(method, common, strong, classic, wsc)
        assert np.array_equal(qid, ids)
        pos = {i: r for r, i in enumerate(ids)}
        for r in range(len(ids)):
            cols = [pos[int(i)] for i in mids[r]]
            assert sorted(cols) == list(range(len(ids))) and np.array_equal(sc[r], D[r, cols])
            assert np.all(np.diff(sc[r]) >= 0)
    assert (strong != common).any() and (weighted_scores(C, vocab, w) != 0).sum() > len(ids)


def test_tree_file_at_k80_l3(tmp_path):
    """A K80 L3 tree (518,480 nodes, 265 MB) through VocabularyTree.save: the product's loader reads it back byte for byte, the
    reference's loader (oracle) reads the same bytes and gives the reference words."""
    from alicevision_b200 import voctree
    c, v = base_tree(80, 3)
    v = v.copy(); v[[5, 80 + 17 * 80 + 40]] = 0
    t = voctree.VocabularyTree(80, 3, c, v)
    assert (t.levels(), t.splits(), t.words()) == (3, 80, 512000)
    a = str(tmp_path / "a.tree")
    t.save(a)
    raw = np.fromfile(a, np.uint8)
    assert raw[:12].view(np.uint32).tolist() == [80, 3, 518480] and len(raw) == 12 + c.nbytes + len(v)
    assert np.array_equal(raw[12:12 + c.nbytes].view(F32).reshape(c.shape), c) and np.array_equal(raw[12 + c.nbytes:], v)
    t2 = voctree.VocabularyTree(file=a)
    assert (t2.levels(), t2.splits(), t2.words()) == (3, 80, 512000)
    b = str(tmp_path / "b.tree")
    t2.save(b)
    assert np.array_equal(np.fromfile(b, np.uint8), raw)
    x = sift_rows(3000, 41)
    want = quantize_ref(80, 3, c, v, x)
    O = oracle.VoctreeOracle(kind())
    o = str(tmp_path / "o.tree")
    assert np.array_equal(O.quantize(80, 3, c, v, x, o), want)
    if O.kind == "ref":
        assert np.array_equal(np.fromfile(o, np.uint8), raw)             # the reference loaded exactly the product's bytes
    if matching_has_gpu():
        assert np.array_equal(t2.quantize(x), want)


def matching_has_gpu():
    from alicevision_b200 import matching
    return matching.load_library().b200m_device_count() > 0


@pytest.mark.parametrize("fault", ["pairwise", "skip_invalid", "last_tie", "float32", "le_max"])
def test_quantize_faults_are_caught(fault):
    """Each deliberate fault of quantize_ref changes at least one word on the scenes: the scenes can tell them apart."""
    changed = 0
    for s in quantiser_scenes(big=False):
        for d, w in zip(s.descs, s.words):
            changed += int((quantize_ref(s.k, s.levels, s.centers, s.valid, d, fault=fault) != w).sum())
    assert changed > 0


def test_weighted_order_fault_is_caught():
    docs = word_db()
    ids, vocab, C, *_ = count_scores(docs)
    w = np.ones(80 ** 3, F32)
    ni = (C > 0).sum(0)
    w[vocab] = np.log(F32(len(ids)) / ni.astype(F32))
    assert (weighted_scores(C, vocab, w, descending=True) != weighted_scores(C, vocab, w)).any()


# ---------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def gpu_trees():
    """One device tree per distinct (centres, valid), shared by every test and database of the module: the K80 L3 tree's device
    copy is made once."""
    from alicevision_b200 import voctree
    cache = {}

    def get(key, k, levels, c, v):
        if key not in cache:
            cache[key] = voctree.VocabularyTree(k, levels, c, v)
        return cache[key]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_gpu_quantize(name, gpu_trees, tmp_path):
    O = oracle.VoctreeOracle(kind())
    for s in scenes_named(name):
        t = gpu_trees(s.tree, s.k, s.levels, s.centers, s.valid)
        for d, w in zip(s.descs, s.words):
            got = t.quantize(d)
            assert got.dtype == np.int32 and np.array_equal(got, w), s.name
        x = [d for d in s.descs if d.dtype == F32 and len(d)]
        if x:
            assert np.array_equal(t.quantize(x[0]), O.quantize(s.k, s.levels, s.centers, s.valid, x[0], str(tmp_path / "t.tree"))), s.name


def _check_db(db, docs, method, num_words):
    ids, vocab, C, common, strong, classic = count_scores(docs)
    w = db.computeTfIdfWeights()
    check_weights(w, docs, num_words)
    q, mids, sc = db.find_all(0, method)
    assert np.array_equal(q, ids)
    S = db.last_scores()
    if method == METHODS[3]:
        assert not S.any()
        D = -weighted_scores(C, vocab, w)
    else:
        assert np.array_equal(S, strong if method == "strongCommonPoints" else common)
        D = distances(method, common, strong, classic, None)
    pos = {i: r for r, i in enumerate(ids)}
    for r in range(len(ids)):
        cols = [pos[int(i)] for i in mids[r]]
        assert sorted(cols) == list(range(len(ids))) and np.array_equal(sc[r], D[r, cols]) and np.all(np.diff(sc[r]) >= 0)
    return q, mids, sc, w


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_gpu_word_database(method, gpu_trees):
    """insert_words skips the quantiser: K6 over posting lists of up to 297 documents, K6b over 300 documents with empty ones
    first, in the middle and last, and weighted scores at b - a >= 256 (the third block column)."""
    from alicevision_b200 import voctree
    c, v = base_tree(80, 3)
    t = gpu_trees(("base", 80, 3), 80, 3, c, v)
    docs = word_db()
    db = voctree.Database(t)
    for i in sorted(docs, reverse=True):
        db.insert_words(i, docs[i])
    assert db.size() == 300 and np.array_equal(db.document(max(docs)), docs[max(docs)])
    q, mids, sc, w = _check_db(db, docs, method, 80 ** 3)
    if method == METHODS[3]:
        ids = sorted(docs)
        far = [(r, mids[r][sc[r] < 0]) for r in range(5)]
        assert any((np.searchsorted(ids, m) - r >= 256).any() for r, m in far)
    empty = voctree.Database(t)
    for i in (4, 9, 2):
        empty.insert_words(i, np.zeros(0, np.int32))
    q, mids, sc = empty.find_all(0, method)
    assert np.array_equal(q, [2, 4, 9]) and not sc.any()


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_gpu_end_to_end_k80_l3(method, gpu_trees, tmp_path):
    """64 overlapping documents of up to 1,500 rows through Database.insert and conditionVocTree on the K80 L3 tree, against the
    references and the oracle (ranked ids against the oracle only: partial_sort's order among tied scores is libstdc++'s)."""
    from alicevision_b200 import voctree
    c, v = base_tree(80, 3)
    t = gpu_trees(("base", 80, 3), 80, 3, c, v)
    d = e2e_scene()
    O = oracle.VoctreeOracle(kind())
    for nmax in (0, 1000):
        docs = e2e_words(nmax)
        db = voctree.Database(t)
        for i in sorted(d):
            db.insert(i, d[i], nmax)
        for i in d:
            assert np.array_equal(db.document(i), docs[i])
        _check_db(db, docs, method, 80 ** 3)
        for nq in (0, 10):
            ids, omids, osc, ow, opairs = O.image_matching(80, 3, c, v, d, nmax, nq, method, str(tmp_path / "t.tree"))
            q, mids, sc = db.find_all(nq, method)
            assert np.array_equal(db.computeTfIdfWeights(), ow)
            assert np.array_equal(q, ids) and np.array_equal(mids, omids) and np.array_equal(sc, osc)
            pairs, _ = voctree.conditionVocTree(t, d, nmax, nq, method)
            assert np.array_equal(pairs, opairs) and len(pairs) > 0
