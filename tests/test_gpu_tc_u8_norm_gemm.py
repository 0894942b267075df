"""The u8 norm-GEMM search kernel (l2_tc.cuh, NG): u8 pairs whose query view has no component above 127 and whose database view
(at least 128 rows) has every squared norm within the limbs' capacity fold the database norms into the 8-bit GEMM (run with -m gpu
on an H100).

Every GPU test compares the final match lists with the oracle (bit-exact: indices, distances, ratios) and with a second context
created under B200M_U8_NORM_GEMM=0, which runs the same pairs on the u8 kernel: the records must be equal element for element.  It
asserts how many directed pairs took the norm-GEMM kernel (last_u8_norm_gemm_pairs), the u8 kernels (last_u8_tc_pairs) and the
tensor cores (last_tc_pairs), so that a silent change of path cannot pass, and that the exactness pass found no error."""
import numpy as np
import pytest

from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

# common.cuh: squared-norm capacity of the 32 limbs (127 + 128 * 31 * 255) and the pad rows' norm (all limbs 255)
LIMB_CAP = 127 + 128 * 31 * 255
LIMB_PAD = 255 + 128 * 31 * 255
BN = 128                      # database rows per tile: smaller databases stay on the u8 kernel


def limbs(n):
    """The limb encoding of common.cuh u8_limb, restated: l_0 = n mod 128, floor(n / 128) filled into l_1..l_31 up to 255 each."""
    q = n >> 7
    return [n & 127] + [int(min(255, max(0, q - 255 * (k - 1)))) for k in range(1, 32)]


def weights():
    return [-1] + [-128] * 31


# ---------------------------------------------------------------------------------------------- CPU: the encoding
def test_limbs_encode_every_norm_up_to_capacity():
    """sum w_k l_k = -n for every n in [0, LIMB_CAP], every limb in 0..255 and l_0 < 128; the pad limbs give -LIMB_PAD, below every
    real row's value; and the largest s32 accumulator magnitude of a gated pair stays below 2^24 (h = s / 2 exact in fp32)."""
    w = np.array(weights(), np.int64)
    ns = np.concatenate([np.arange(0, 70000), np.arange(LIMB_CAP - 70000, LIMB_CAP + 1), np.random.default_rng(1).integers(0, LIMB_CAP + 1, 20000)])
    L = np.array([limbs(int(n)) for n in ns], np.int64)
    assert L.min() >= 0 and L.max() <= 255 and L[:, 0].max() <= 127
    assert np.array_equal(L @ w, -ns)
    assert int(np.full(32, 255) @ w) == -LIMB_PAD and LIMB_PAD > LIMB_CAP
    assert 2 * 127 * 255 * 128 + LIMB_PAD < 1 << 24
    # the s8 weight bytes of the constant A tile (l2_tc.cuh): chunk 0 = 0x808080FF, 0x80808080 x 3
    assert bytes(np.array(weights()[:4], np.int8).view(np.uint8)) == (0x808080FF).to_bytes(4, "little")


def test_doubling_a_word_doubles_its_bytes():
    """The in-place doubling of the query tile shifts 32-bit words left by one: exact for every byte <= 127, not above."""
    rng = np.random.default_rng(2)
    b = rng.integers(0, 128, (4096, 4), dtype=np.uint8)
    w = b.view("<u4")
    assert np.array_equal(((w << 1) & 0xFFFFFFFF).astype("<u4").view(np.uint8).reshape(-1, 4), 2 * b.astype(np.uint16))
    b[0, 0] = 128
    w = b.view("<u4")
    assert not np.array_equal(((w << 1) & 0xFFFFFFFF).astype("<u4").view(np.uint8).reshape(-1, 4), 2 * b.astype(np.uint16))


def row_with_norm(n, rng):
    """A uchar row with squared norm exactly n (n up to 128 * 255^2): greedy largest squares, shuffled."""
    v, rest = [], n
    while rest:
        x = min(255, int(np.sqrt(rest)))
        v.append(x)
        rest -= x * x
    assert len(v) <= 128 and sum(x * x for x in v) == n
    r = np.zeros(128, np.uint8)
    r[rng.permutation(128)[:len(v)]] = v
    return r


def test_row_with_norm():
    rng = np.random.default_rng(3)
    for n in (0, 1, LIMB_CAP, LIMB_CAP + 1, 128 * 255 * 255):
        assert int((row_with_norm(n, rng).astype(np.int64) ** 2).sum()) == n


# ---------------------------------------------------------------------------------------------- GPU
def as_dict(res):
    pid, off, mat = res
    return {(int(a), int(b)): mat[off[k]:off[k + 1]].copy() for k, (a, b) in enumerate(pid.tolist()) if off[k + 1] > off[k]}


def assert_same(got, want, what):
    assert sorted(got) == sorted(want), f"{what}: pairs {sorted(set(got) ^ set(want))[:8]} differ"
    for k in want:
        g, w = got[k], want[k]
        assert len(g) == len(w), f"{what}: pair {k} has {len(g)} matches, expected {len(w)}"
        for f in ("i", "j", "dist", "ratio"):
            assert np.array_equal(g[f], w[f]), f"{what}: {f} differs for pair {k}"


class Engine:
    """One context created under `env` (read at creation) with `views` {id: (desc, xy)} uploaded."""

    def __init__(self, mp, env, views):
        for k, v in env.items():
            mp.setenv(k, v)
        self.ctx = matching.Context(0)
        self.m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, self.ctx)
        self.m.upload(dict(sorted(views.items())))
        self.m.wait_uploads()

    def run(self, pairs, ratio, cross):
        self.m.distRatio, self.m.crossMatching = ratio, cross
        pid, off, mat = self.m.match_uploaded(np.asarray(pairs, np.uint32).reshape(-1, 2))
        c = self.ctx
        counts = dict(tc=c.last_tc_pairs(), u8=c.last_u8_tc_pairs(), ng=c.last_u8_norm_gemm_pairs(), real=c.last_real_tc_pairs(),
                      batches=c.last_batches(), errors=c.exactness_errors(), fallback=c.last_fallback_rows())
        return (pid, off, mat), counts


@pytest.fixture
def engines():
    """The default context (norm-GEMM kernel on) and one under B200M_U8_NORM_GEMM=0, built by open(views)."""
    made = []

    def open_(views):
        out = []
        for env in ({}, {"B200M_U8_NORM_GEMM": "0"}):
            with pytest.MonkeyPatch.context() as mp:
                out.append(Engine(mp, env, views))
        made.extend(out)
        return out

    yield open_
    for e in made:
        e.ctx.close()


def directed(descs, pairs, cross):
    """Directed pairs (database, query) that reach a search kernel: at least two database rows and a non-empty query view."""
    ps = {(int(a), int(b)) for a, b in np.asarray(pairs).reshape(-1, 2)}
    return [(i, j) for a, b in ps for i, j in (((a, b), (b, a)) if cross else ((a, b),)) if len(descs[i]) >= 2 and len(descs[j]) >= 1]


def ng_eligible(descs, i, j):
    """Directed pair (database i, query j) on the norm-GEMM kernel: the engine's gates (engine.cu pair_class)."""
    db, q = np.asarray(descs[i], np.int64), np.asarray(descs[j], np.int64)
    return len(db) >= BN and len(q) >= 1 and q.max() <= 127 and (db * db).sum(1).max() <= LIMB_CAP


def check(ora, on, off, descs, xys, pairs, ratios=(0.8, 1.0), crosses=(False, True), ng=None):
    """Every ratio and cross setting: the oracle's lists on the default context, the same bytes on the u8 kernel's context, and the
    number of directed pairs on each path.  ng(i, j): whether directed pair (i, j) is expected on the norm-GEMM kernel (default: the
    gates restated).  Every view here is stored as uchar, so every directed pair that reaches a search kernel is a u8 pair."""
    ng = ng or (lambda i, j: ng_eligible(descs, i, j))
    kept = 0
    for cross in crosses:
        for r in ratios:
            what = f"cross={cross} ratio={r}"
            d = directed(descs, pairs, cross)
            n_ng = sum(ng(i, j) for i, j in d)
            res, c = on.run(pairs, r, cross)
            res0, c0 = off.run(pairs, r, cross)
            assert (c["tc"], c["u8"], c["ng"], c["errors"]) == (len(d), len(d), n_ng, 0), (what, c)
            assert (c0["tc"], c0["u8"], c0["ng"], c0["errors"]) == (len(d), len(d), 0, 0), (what, c0)
            for a, b in zip(res, res0):
                assert np.array_equal(a, b), f"{what}: the norm-GEMM kernel's records differ from the u8 kernel's"
            want = ora.collection_match(descs, xys, pairs, r, cross)
            assert_same(as_dict(res), want, what)
            kept += sum(len(v) for v in want.values())
    assert kept > 0
    return kept


@pytest.mark.gpu
def test_full_size_fused(ora, engines):
    """8192 x 8192 (the benchmark's image size, in-kernel exactness pass) of RootSIFT-like uchar rows: every directed pair on the
    norm-GEMM kernel, at ratios 0.8 and 1.0, with and without cross matching."""
    descs, xys = synth.sift_images(2, 8192, np.uint8, seed=611, pool_factor=1.0)
    assert max(int(d.max()) for d in descs) <= 127
    on, off = engines({k: (d, x) for k, (d, x) in enumerate(zip(descs, xys))})
    check(ora, on, off, descs, xys, np.array([(0, 1)], np.uint32), ng=lambda i, j: True)


DB_SIZES = [1, 2, 3, 17, 127, 128, 129, 130, 200, 257, 1111]     # below one tile: the u8 kernel; partial last tiles of 1, 2, ... rows
Q_SIZES = [1, 2, 3, 17, 129, 300]


@pytest.mark.gpu
def test_ragged_sizes_unfused(ora, engines):
    """Short database images (the stand-alone exactness pass) of ragged sizes against ragged query images, both directions: the
    databases of fewer than 128 rows stay on the u8 kernel, the others take the norm-GEMM kernel with partial last tiles."""
    d, _ = synth.sift_images(2, max(DB_SIZES), np.uint8, seed=612, pool_factor=1.0)
    descs = [d[0][:m] for m in DB_SIZES] + [d[1][:m] for m in Q_SIZES]
    rng = np.random.default_rng(612)
    xys = [synth.positions(len(x), rng) for x in descs]
    pairs = np.array([(a, len(DB_SIZES) + b) for a in range(len(DB_SIZES)) for b in range(len(Q_SIZES))], np.uint32)
    on, off = engines({k: (x, p) for k, (x, p) in enumerate(zip(descs, xys))})
    d = directed(descs, pairs, True)
    assert 0 < sum(ng_eligible(descs, i, j) for i, j in d) < len(d)
    check(ora, on, off, descs, xys, pairs)


def gate_views(seed=613):
    """Queries with a component of exactly 127 (eligible) and 128 (not); databases of 600 rows holding a row of squared norm exactly
    LIMB_CAP (eligible) and LIMB_CAP + 1 (not), in their partial last tile."""
    rng = np.random.default_rng(seed)
    d, _ = synth.sift_images(4, 600, np.uint8, seed=seed, pool_factor=1.0)
    q127, q128, db_cap, db_over = (x.copy() for x in d)
    q127[5, 10] = q127[200, 99] = 127
    q128[7, 3] = 128
    db_cap[590] = row_with_norm(LIMB_CAP, rng)
    db_over[590] = row_with_norm(LIMB_CAP + 1, rng)
    return [q127[:300], q128[:300], db_cap, db_over]


@pytest.mark.gpu
@pytest.mark.parametrize("db,q,on_ng", [(2, 0, True), (3, 0, False), (2, 1, False), (3, 1, False)])
def test_gate_boundaries(ora, engines, db, q, on_ng):
    """Query max component 127 / 128 against database max norm LIMB_CAP / LIMB_CAP + 1, and with cross matching the reverse
    direction (the databases hold components of 255, so they are never norm-GEMM queries)."""
    descs = gate_views()
    assert int(descs[0].max()) == 127 and int(descs[1].max()) == 128
    assert int((descs[2].astype(np.int64) ** 2).sum(1).max()) == LIMB_CAP and int((descs[3].astype(np.int64) ** 2).sum(1).max()) == LIMB_CAP + 1
    rng = np.random.default_rng(614)
    xys = [synth.positions(len(x), rng) for x in descs]
    on, off = engines({k: (x, p) for k, (x, p) in enumerate(zip(descs, xys))})
    expect = {(db, q): on_ng, (q, db): False}
    check(ora, on, off, descs, xys, np.array([(db, q)], np.uint32), ng=lambda i, j: expect[(i, j)])


@pytest.mark.gpu
def test_pad_rows_never_win(ora, engines):
    """All-zero queries, whose nearest row is the one of smallest norm, against databases of rows with distinct squared norms just below
    and at the capacity (LIMB_CAP - 7 k), ending in partial last tiles of 1, 2, 3 and 17 rows: the smallest norm sits in the partial
    tile (or, reversed, the LIMB_CAP row does), and a pad row, whose value lies above LIMB_CAP, never wins and is never the second
    neighbour.  At ratio 1.0 every zero query keeps its match."""
    rng = np.random.default_rng(615)
    rows = np.array([row_with_norm(LIMB_CAP - 7 * k, rng) for k in range(145)])
    dbs = [rows[:m] for m in (129, 130, 131, 145)] + [np.ascontiguousarray(rows[::-1])]
    q = np.zeros((40, 128), np.uint8)
    q[20:] = np.minimum(synth.sift_pool(20, rng), 127)
    descs = dbs + [q]
    xys = [synth.positions(len(x), rng) for x in descs]
    on, off = engines({k: (x, p) for k, (x, p) in enumerate(zip(descs, xys))})
    pairs = np.array([(k, len(dbs)) for k in range(len(dbs))], np.uint32)
    kept = check(ora, on, off, descs, xys, pairs, crosses=(False,), ng=lambda i, j: True)
    assert kept >= 20 * len(dbs)


@pytest.mark.gpu
def test_duplicate_rows_in_different_chunks(ora, engines):
    """Copies of a database row in different chunks and tiles (and twice in one chunk), queried by exact and near copies: the chunk
    minima tie, and the lowest chunk id, then the lowest row, must win as in the reference."""
    rng = np.random.default_rng(616)
    d, xys = synth.sift_images(2, 2000, np.uint8, seed=616, pool_factor=1.0)
    db, q = d[0].copy(), d[1].copy()
    for k, src in enumerate(rng.choice(len(db), 12, replace=False)):
        for dst in rng.choice(len(db), 3, replace=False).tolist() + [src ^ 1]:
            db[dst] = db[src]
        v = db[src].astype(np.int64)
        v[rng.integers(0, 128)] += 1
        q[k] = np.clip(v, 0, 127)
        q[12 + k] = np.minimum(db[src], 127)
    assert int(q.max()) <= 127
    on, off = engines({0: (db, xys[0]), 1: (q, xys[1])})
    check(ora, on, off, [db, q], xys, np.array([(0, 1)], np.uint32), crosses=(False,), ng=lambda i, j: True)


# ---------------------------------------------------------------------------------------------- every kernel class in one list
PAIR_CAP = 4096
CLASSES = ["ng", "u8", "fp16", "real", "exact_f32", "exact_u8"]
K_DB, L_Q = 30, 50          # database / query views per class: 9000 directed pairs, three batches of PAIR_CAP


def class_view(rng, pool, cls, m):
    """m uchar-valued SIFT-like rows of class `cls`: up to len(pool) noisy copies of distinct pool rows, the rest fresh."""
    k = min(m, len(pool))
    a = pool[rng.choice(len(pool), k, replace=False)].astype(np.int16) + rng.integers(-4, 5, (k, 128), dtype=np.int16)
    b = synth.sift_pool(m - k, rng).astype(np.int16)
    d = np.ascontiguousarray(np.clip(np.concatenate([a, b]), 0, 255)[rng.permutation(m)].astype(np.uint8))
    if cls == "ng":                            # integer-valued fp32 in 0..127 (staged as uchar), databases of >= 128 rows
        return np.minimum(d, 127).astype(np.float32)
    if cls == "u8":                            # the same kind of rows, databases below one tile: the u8 kernel
        return d.astype(np.float32)
    if cls == "fp16":                          # signed integers: the fp16 kernel
        return d.astype(np.float32) - np.float32(64)
    if cls == "real":                          # real-valued: the filter kernel; noise rows fall back to the exact search
        x = d.astype(np.float32) + rng.normal(0, 0.37, d.shape).astype(np.float32)
        rows = [r for r in (3, 19, 35, 48, 9, 25, 41, 49) if r < m]
        x[rows] = (150 + rng.normal(0, 0.25, (len(rows), 128))).astype(np.float32)
        return np.ascontiguousarray(x)
    if cls == "exact_f32":                     # ||v||^2 >= 2^22: the exact kernels
        x = d.astype(np.float32); x[0] = 0; x[0, :8] = 1000
        return x
    x = d.copy(); x[0] = 255
    return x


def class_scene(seed=617):
    """Database view k of class c has id 6k + c, so the sorted pair list cycles through the classes every 6 database views."""
    rng = np.random.default_rng(seed)
    pool = synth.sift_pool(48, rng)
    descs, cls_of, pairs = {}, {}, []
    for k in range(K_DB):
        for c, cls in enumerate(CLASSES):
            v = len(CLASSES) * k + c
            m = int(rng.integers(128, 200)) if cls == "ng" else 50 if cls == "real" else int(rng.integers(2, 41))
            descs[v], cls_of[v] = class_view(rng, pool, cls, m), cls
    q0 = len(CLASSES) * K_DB
    for c, cls in enumerate(CLASSES):
        for k in range(L_Q):
            v = q0 + L_Q * c + k
            descs[v], cls_of[v] = class_view(rng, pool, cls, int(rng.integers(1, 41))), cls
            pairs += [(len(CLASSES) * a + c, v) for a in range(K_DB)]
    xys = {v: synth.positions(len(d), rng) for v, d in descs.items()}
    return descs, xys, cls_of, sorted(pairs)


def test_class_scene_batches():
    """Every PAIR_CAP batch of the sorted list holds every class."""
    _, _, cls_of, pairs = class_scene()
    assert len(pairs) == len(CLASSES) * K_DB * L_Q
    for b in range(0, len(pairs), PAIR_CAP):
        assert {cls_of[a] for a, _ in pairs[b:b + PAIR_CAP]} == set(CLASSES)


@pytest.mark.gpu
def test_every_kernel_class_in_every_batch(ora, engines):
    """One list across three batches whose every batch launches the norm-GEMM, u8, fp16, real-valued and exact f32 / u8 kernels into
    one candidate array: the oracle's lists, the same bytes with the norm-GEMM kernel switched off, and the per-class pair counts."""
    descs, xys, cls_of, pairs = class_scene()
    per = {c: sum(cls_of[a] == c for a, _ in pairs) for c in CLASSES}
    n = max(descs) + 1
    want = {}
    for keep_cls, dt in (({"ng", "u8", "fp16", "real", "exact_f32"}, np.float32), ({"exact_u8"}, np.uint8)):
        keep = {v for v, c in cls_of.items() if c in keep_cls}
        ds = [descs[v] if v in keep else np.zeros((0, 128), dt) for v in range(n)]
        xs = [xys[v] if v in keep else np.zeros((0, 2), np.float32) for v in range(n)]
        want.update(ora.collection_match(ds, xs, [p for p in pairs if p[0] in keep], 0.8))
    for c in CLASSES:
        assert sum(len(v) for k, v in want.items() if cls_of[k[0]] == c) > 0, c
    on, off = engines({v: (descs[v], xys[v]) for v in descs})
    res, c = on.run(pairs, 0.8, False)
    res0, c0 = off.run(pairs, 0.8, False)
    assert c["batches"] == c0["batches"] == 3
    assert (c["tc"], c["u8"], c["ng"], c["real"]) == (per["ng"] + per["u8"] + per["fp16"], per["ng"] + per["u8"], per["ng"], per["real"])
    assert (c0["tc"], c0["u8"], c0["ng"]) == (c["tc"], c["u8"], 0)
    assert c["errors"] == 0 and c0["errors"] == 0 and c["fallback"] > 0
    for a, b in zip(res, res0):
        assert np.array_equal(a, b)
    assert_same(as_dict(res), want, "classes")
