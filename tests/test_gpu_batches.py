"""The host batch loop of b200m_match_pairs (engine.cu): long pair lists split into batches, two buffer sets on three streams, the
pinned per-batch meta block and the per-batch kernel decisions, checked against the oracle (the GPU tests: run with -m gpu on an H100).

A batch closes before a directed pair that would exceed one of PAIR_CAP directed pairs, CAND_CAP candidate slots (sum of the query
rows m_j), ITEM_CAP work items or SLOT_CAP finishing slots (sum of the database rows m_i); while uploads are in flight the pair cap
starts at B200M_FIRST_BATCH and doubles from batch to batch.  `plan_batches` restates that rule; every GPU case asserts that the engine
ran the number of batches the plan predicts (b200m_last_batches), so a case built to cross a cap cannot quietly run as one batch.

Each scene keeps one side of every pair small (a few large views paired with many small ones), so the CPU oracle stays cheap.  The
results must equal the oracle's bit for bit (indices, distances, ratios) and be byte-identical across the finishing stage on the device
and on the host, the pipelined streams and one stream, and different batch compositions of the same list."""
import time

import numpy as np
import pytest

import oracle
from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

# the engine's batch limits (engine.cu) and the tensor-core work-item height
PAIR_CAP = 4096
CAND_CAP = 4 << 20
ITEM_CAP = CAND_CAP // 64 + PAIR_CAP
SLOT_CAP = 8 << 20
BM = 128
FUSED_ROWS = 6144            # average database rows of a batch's u8 pairs from which the u8 kernel runs the exactness pass itself


# ---------------------------------------------------------------------------------------------- the split rule
def plan_batches(sizes_i, sizes_j, cross=False, pair_cap=PAIR_CAP):
    """Directed pairs per batch for a list of (undirected) pairs in processing order: sizes_i[k] / sizes_j[k] are the rows of the
    database / query view of pair k.  Skipped pairs (an empty view, a database of fewer than 2 rows, mismatched types) take their place
    and count toward every cap like the others.  With cross matching both directions of a pair go into the same batch.  pair_cap is
    the first batch's pair cap: PAIR_CAP for resident views, B200M_FIRST_BATCH while uploads are in flight (doubled per batch)."""
    step = 2 if cross else 1
    plan, n, cand, items, slots = [], 0, 0, 0, 0
    for mi, mj in zip(sizes_i, sizes_j):
        dirs = ((mi, mj), (mj, mi))[:step]
        assert all(q <= CAND_CAP and d <= SLOT_CAP // 2 for d, q in dirs), "view too large for one batch"
        need_c = sum(q for _, q in dirs)
        need_i = sum(-(-q // BM) for _, q in dirs)
        need_s = sum(d for d, _ in dirs)
        over = dict(cand=cand + need_c > CAND_CAP, items=items + need_i > ITEM_CAP, slots=slots + need_s > SLOT_CAP, pairs=n + step > pair_cap)
        # ITEM_CAP never decides: items <= sum(m_j / BM + 1) <= CAND_CAP / BM + PAIR_CAP < ITEM_CAP while the other caps hold
        assert not over["items"] or over["cand"] or over["pairs"]
        if n and any(over.values()):
            plan.append(n)
            n, cand, items, slots = 0, 0, 0, 0
            pair_cap = min(PAIR_CAP, 2 * pair_cap)
        n += step; cand += need_c; items += need_i; slots += need_s
        assert items <= cand // BM + n <= CAND_CAP // BM + PAIR_CAP < ITEM_CAP
    if n:
        plan.append(n)
    return plan


def processing_order(pairs, upload_rank=None):
    """The engine's processing order: PairSet order (sorted, unique); while uploads are in flight, stably re-sorted by the later
    upload position of each pair's two views (upload_rank[view id])."""
    ps = sorted({(int(a), int(b)) for a, b in pairs})
    if upload_rank is not None:
        ps.sort(key=lambda p: max(upload_rank[p[0]], upload_rank[p[1]]))
    return ps


def plan_of(sizes, pairs, cross=False, upload_rank=None, pair_cap=PAIR_CAP):
    ps = processing_order(pairs, upload_rank)
    return plan_batches([sizes[a] for a, _ in ps], [sizes[b] for _, b in ps], cross, pair_cap)


def batches_of(plan, ps):
    """Split the (directed, non-cross) processing order `ps` by `plan`."""
    out, k = [], 0
    for n in plan:
        out.append(ps[k:k + n]); k += n
    return out


def fused_u8_pairs(sizes, batches):
    """The u8 kernel's per-batch choice: the exactness pass runs inside the kernel when the batch's u8 pairs average >= 6144 database
    rows (integer division); the pairs that take it.  All pairs here are u8 pairs unless skipped (no database rows to search)."""
    fused = set()
    for b in batches:
        live = [(a, q) for a, q in b if sizes[a] >= 2 and sizes[q] >= 1]
        if live and sum(sizes[a] for a, _ in live) // len(live) >= FUSED_ROWS:
            fused |= set(live)
    return fused


def n_directed(sizes, pairs, cross=False):
    """Directed pairs that reach a search kernel: a database of >= 2 rows and a non-empty query view."""
    ps = {(int(a), int(b)) for a, b in pairs}
    return sum(sizes[i] >= 2 and sizes[j] >= 1 for a, b in ps for i, j in (((a, b), (b, a)) if cross else ((a, b),)))


# ---------------------------------------------------------------------------------------------- CPU: the rule on hand-computed plans
def test_plan_pair_cap():
    assert plan_batches([10] * 4096, [10] * 4096) == [4096]
    assert plan_batches([10] * 4097, [10] * 4097) == [4096, 1]
    assert plan_batches([0, 1] * 2048 + [5], [7] * 4097) == [4096, 1]        # skipped pairs count toward the cap


def test_plan_cross_step():
    assert plan_batches([10] * 2048, [10] * 2048, cross=True) == [4096]
    assert plan_batches([10] * 2049, [10] * 2049, cross=True) == [4096, 2]


def test_plan_cand_cap():
    assert plan_batches([40] * 512, [8192] * 512) == [512]                  # sum m_j == CAND_CAP exactly
    assert plan_batches([40] * 513, [8192] * 513) == [512, 1]
    assert plan_batches([40] * 2, [CAND_CAP, 1]) == [1, 1]


def test_plan_slot_cap():
    assert plan_batches([8192] * 1024, [3] * 1024) == [1024]                # sum m_i == SLOT_CAP exactly
    assert plan_batches([8192] * 1025, [3] * 1025) == [1024, 1]
    assert plan_batches([8192] * 1025, [3] * 1025, cross=True) == [1022, 1022, 6]   # both directions: 8195 candidate slots per pair


def test_plan_first_batch_doubling():
    assert plan_batches([10] * 4097, [10] * 4097, pair_cap=1) == [1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 2]
    assert plan_batches([10] * 10000, [10] * 10000, pair_cap=16) == [16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 1824]
    assert plan_batches([10] * 7, [10] * 7, cross=True, pair_cap=1) == [2, 2, 4, 6]


def test_plan_item_cap_never_binds():
    """One-row queries (one work item per candidate slot) and 129-row queries (two items each) hit PAIR_CAP, not ITEM_CAP; the
    assertions inside plan_batches check the bound on every step."""
    assert plan_batches([2] * 4096, [1] * 4096) == [4096]
    n = CAND_CAP // 129
    assert plan_batches([2] * (n + 1), [129] * (n + 1)) == [4096] * (n // 4096) + [n % 4096 + 1]
    with pytest.raises(AssertionError, match="too large"):
        plan_batches([2], [CAND_CAP + 1])


def test_processing_order_and_fused_rule():
    sizes = {0: 8192, 1: 2000, 5: 3, 6: 2}
    pairs = [(0, 5), (1, 5), (0, 6), (1, 6)]
    assert processing_order(pairs) == [(0, 5), (0, 6), (1, 5), (1, 6)]
    rank = {5: 0, 6: 1, 0: 2, 1: 3}
    assert processing_order(pairs, rank) == [(0, 5), (0, 6), (1, 5), (1, 6)]
    rank = {0: 0, 5: 1, 1: 2, 6: 3}
    assert processing_order(pairs, rank) == [(0, 5), (1, 5), (0, 6), (1, 6)]
    ps = processing_order(pairs)
    assert fused_u8_pairs(sizes, batches_of([4], ps)) == set()                       # (8192 + 2000) / 2 < 6144
    assert fused_u8_pairs(sizes, batches_of([1, 3], ps)) == {(0, 5)}
    assert fused_u8_pairs(sizes, batches_of([2, 2], ps)) == {(0, 5), (0, 6)}


# ---------------------------------------------------------------------------------------------- the scenes
# view ids (one id space, u8 views): S small (2-40 rows, some empty / one-row), B: CAND_CAP scenes, C: SLOT_CAP scenes, M: 2000-row
S_DB, S_Q, S_EXTRA = range(0, 64), range(64, 128), 128
B_DB, B_Q = range(200, 265), range(300, 308)
C_DB, C_Q = range(400, 412), range(500, 757)
M_DB = range(760, 772)
N_IDS = 772


def world_sizes():
    rng = np.random.default_rng(8101)
    sizes = {}
    for v in list(S_DB) + list(S_Q) + [S_EXTRA] + list(B_DB):
        sizes[v] = int(rng.integers(2, 41))
    for v in (5, 17, 70, 111):
        sizes[v] = 0                         # empty views: skipped pairs on either side
    for v in (9, 30, 99, 230):
        sizes[v] = 1                         # one row: skipped as a database, searched as a query
    for v in B_Q:
        sizes[v] = 8192
    for v in C_DB:
        sizes[v] = 8192
    for v in C_Q:
        sizes[v] = int(rng.integers(1, 4))
    for v in M_DB:
        sizes[v] = 2000
    return sizes


def scene_lists():
    A = [(a, b) for a in S_DB for b in S_Q]                       # 4096 directed pairs
    A1 = sorted(A + [(0, S_EXTRA)])
    B = sorted([(a, b) for a in B_DB[:64] for b in B_Q] + [(B_DB[64], B_Q[0])])
    C = sorted([(a, b) for a in C_DB for b in C_Q[:256]] + [(C_DB[0], C_Q[256])])
    comp = [(a, b) for a in list(C_DB[:4]) + list(M_DB) for b in C_Q[:8]]
    return {
        # name: (pairs, cross, batches)
        "pair_cap": (A, False, 1),
        "pair_cap_plus_1": (A1, False, 2),
        "cross_2048": (A[:2048], True, 1),
        "cross_2049": (A[:2049], True, 2),
        "cand_cap": (B[:512], False, 1),
        "cand_cap_plus_1": (B, False, 2),
        "slot_cap": (C[:1025], False, 2),
        "many": (sorted(A1 + B + C), False, 6),
        "three": (sorted(A1 + C[:1025]), False, 3),
        "four": (sorted(A1 + B + C[:1025]), False, 4),
        "composition": (comp, False, 1),
    }


def upload_rank():
    """Upload order of the world: view ids ascending."""
    return {v: k for k, v in enumerate(range(N_IDS))}


def test_scene_plans():
    """Every scene of the GPU tests splits the way its name says, and sits exactly on the cap it is built for."""
    sizes = world_sizes()
    for name, (pairs, cross, want) in scene_lists().items():
        assert len(plan_of(sizes, pairs, cross)) == want, name
    L = scene_lists()
    assert sum(sizes[b] for _, b in L["cand_cap"][0]) == CAND_CAP
    assert sum(sizes[a] for a, _ in L["slot_cap"][0][:1024]) == SLOT_CAP
    assert plan_of(sizes, *L["pair_cap"][:2]) == [PAIR_CAP] and plan_of(sizes, *L["cross_2048"][:2]) == [PAIR_CAP]
    assert len(L["cross_2049"][0]) == 2049 and len(L["slot_cap"][0]) == 1025 and len(L["cand_cap_plus_1"][0]) == 513
    assert n_directed(sizes, L["pair_cap"][0]) < PAIR_CAP           # skipped pairs inside the full batch
    # PAIR_CAP, then CAND_CAP (one small pair + 511 of the 8192-row queries), then SLOT_CAP three times: each buffer set is used by
    # three batches
    assert plan_of(sizes, L["many"][0]) == [4096, 512, 1025, 1024, 1024, 2]
    assert all(1 <= sizes[b] <= 3 for _, b in L["slot_cap"][0]) and all(sizes[a] <= 40 for a, _ in L["cand_cap_plus_1"][0])
    # the composition list: one batch (unfused) when resident, batches of 1, 2, 4, ... in upload order (the first ones fused)
    comp = L["composition"][0]
    assert fused_u8_pairs(sizes, batches_of(plan_of(sizes, comp), processing_order(comp))) == set()
    rank = upload_rank()
    ps = processing_order(comp, rank)
    plan = plan_of(sizes, comp, upload_rank=rank, pair_cap=1)
    assert plan == [1, 2, 4, 8, 16, 32, 64, 1]
    assert fused_u8_pairs(sizes, batches_of(plan, ps)) == set(ps[:31])


# ---------------------------------------------------------------------------------------------- GPU
RATIO = 0.8
VARIANTS = {
    "device_finish": {"B200M_DEVICE_FINISH": "1", "B200M_PIPE_STREAMS": "1"},
    "host_finish": {"B200M_DEVICE_FINISH": "0", "B200M_PIPE_STREAMS": "1"},
    "one_stream": {"B200M_DEVICE_FINISH": "1", "B200M_PIPE_STREAMS": "0"},
}


def sift_view(rng, pool, m, planted):
    """m uchar-valued SIFT-like rows: `planted` of them noisy copies of rows of the shared pool, the rest fresh."""
    k = min(planted, m, len(pool))
    a = pool[rng.choice(len(pool), k, replace=False)].astype(np.int16) + rng.integers(-4, 5, (k, 128), dtype=np.int16)
    b = synth.sift_pool(m - k, rng).astype(np.int16) if m > k else np.zeros((0, 128), np.int16)
    return np.ascontiguousarray(np.clip(np.concatenate([a, b]), 0, 255)[rng.permutation(m)].astype(np.uint8))


def build_world():
    """Descriptors and positions of every view id (empty arrays for unused ids); small views draw 3/4 of their rows from a pool of
    96 shared rows, large views hold all of them, so most pairs keep matches."""
    sizes = world_sizes()
    rng = np.random.default_rng(8102)
    pool = synth.sift_pool(96, rng)
    descs, xys = [], []
    for v in range(N_IDS):
        m = sizes.get(v, 0)
        descs.append(sift_view(rng, pool, m, m if m < 96 else 96) if m <= 40 else sift_view(rng, pool, m, 96))
        xys.append(synth.positions(m, rng))
    return sizes, descs, xys


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


def restrict(answer, pairs):
    keep = {(int(a), int(b)) for a, b in pairs}
    return {k: v for k, v in answer.items() if k in keep}


class Run:
    """One b200m_match_pairs call: its result bytes, as a dict, and the context's per-call counters."""

    def __init__(self, ctx, matcher, pairs, cross):
        matcher.crossMatching = cross
        pid, off, mat = matcher.match_uploaded(np.asarray(pairs, np.uint32))
        self.bytes = pid.tobytes() + off.tobytes() + mat.tobytes()
        self.got = as_dict((pid, off, mat))
        self.batches, self.tc, self.u8 = ctx.last_batches(), ctx.last_tc_pairs(), ctx.last_u8_tc_pairs()
        self.ng = ctx.last_u8_norm_gemm_pairs()
        self.real, self.fallback, self.errors = ctx.last_real_tc_pairs(), ctx.last_fallback_rows(), ctx.exactness_errors()


def open_context(mp, env, views, hamming=False, wait=True):
    """A fresh context created under `env` (read at creation), with `views` {id: (desc, xy)} uploaded in id order."""
    for k, v in env.items():
        mp.setenv(k, v)
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(RATIO, False, EMatcherType.BRUTE_FORCE_HAMMING_B200 if hamming else EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload(dict(sorted(views.items())))
    if wait:
        m.wait_uploads()
    return ctx, m


@pytest.fixture(scope="module")
def world():
    return build_world()


@pytest.fixture(scope="module")
def answers(world, ora):
    """The oracle's lists, computed once: every non-cross pair of every scene in one call, the cross scene in another."""
    sizes, descs, xys = world
    L = scene_lists()
    plain = sorted({p for pairs, cross, _ in L.values() if not cross for p in pairs})
    return {False: ora.collection_match(descs, xys, plain, RATIO), True: ora.collection_match(descs, xys, L["cross_2049"][0], RATIO, cross=True)}


CAP_CASES = ["pair_cap", "pair_cap_plus_1", "cross_2048", "cross_2049", "cand_cap", "cand_cap_plus_1", "slot_cap", "many"]


@pytest.fixture(scope="module")
def cap_runs(world):
    """Every cap scene on one context per variant (device / host finishing, pipelined / one stream), views resident."""
    sizes, descs, xys = world
    L = scene_lists()
    views = {v: (descs[v], xys[v]) for v in range(N_IDS) if v in sizes}
    out = {}
    for name, env in VARIANTS.items():
        with pytest.MonkeyPatch.context() as mp:
            ctx, m = open_context(mp, env, views)
        try:
            out[name] = {case: Run(ctx, m, L[case][0], L[case][1]) for case in CAP_CASES}
        finally:
            ctx.close()
    return out


def check_run(r, want, sizes, pairs, cross, batches, what):
    assert r.batches == batches, f"{what}: {r.batches} batches, planned {batches}"
    n = n_directed(sizes, pairs, cross)
    assert (r.tc, r.u8, r.real, r.errors) == (n, n, 0, 0), what
    assert_same(r.got, want, what)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAP_CASES)
def test_caps_against_oracle(case, world, answers, cap_runs):
    """Scenes on, and one pair across, each cap: the planned batch count, every directed pair on the u8 kernel, the oracle's lists bit
    for bit (every pair the oracle keeps is non-empty), and byte-identical results with the finishing stage on the device and on the
    host and with every stage on one stream."""
    sizes = world[0]
    pairs, cross, want_batches = scene_lists()[case]
    plan = plan_of(sizes, pairs, cross)
    assert len(plan) == want_batches
    want = restrict(answers[cross], pairs)
    assert sum(len(v) for v in want.values()) > 0 and len(want) > 0.1 * len(pairs)
    ref = cap_runs["device_finish"][case]
    for name in VARIANTS:
        r = cap_runs[name][case]
        check_run(r, want, sizes, pairs, cross, len(plan), f"{case} {name}")
        assert r.bytes == ref.bytes, f"{case}: {name} differs from device_finish"


HOLD_S = 2.0                 # GPU sleep that holds an upload in flight (test_batch_composition)


@pytest.mark.gpu
def test_batch_composition(world, answers):
    """The same lists while the views are still uploading with B200M_FIRST_BATCH=1 (batches of 1, 2, 4, ... in upload order) and once
    they are resident give identical bytes.  In the composition list the big-database pairs of the first short batches run the u8
    kernel's in-kernel exactness pass, while the resident batch (average below 6144 rows) leaves it to verify_pack_kernel.

    The upload is held in flight on purpose: the context runs on a borrowed stream, a GPU sleep is queued on it before the upload,
    and the upload stream waits for that stream (the view buffers are allocated on it).  The uploader thread then blocks when it
    reuses its first staging buffer, so the job cannot finish before the sleep ends; the match call starts well inside the sleep.
    The first, resident call allocated the batch buffers and sized the view table, so nothing on the way synchronises the stream."""
    import torch
    sizes, descs, xys = world
    L = scene_lists()
    views = dict(sorted((v, (descs[v], xys[v])) for v in range(N_IDS) if v in sizes))
    assert sum(2 if len(d) else 1 for d, _ in views.values()) > 2 * 24     # more chunks than the uploader's staging ring
    rank = upload_rank()
    for case in ("composition", "many"):
        pairs = L[case][0]
        want = restrict(answers[False], pairs)
        pending_plan = plan_of(sizes, pairs, upload_rank=rank, pair_cap=1)
        resident_plan = plan_of(sizes, pairs)
        stream = torch.cuda.Stream(0)
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200M_FIRST_BATCH", "1")
            ctx = matching.Context(0, stream=stream.cuda_stream)
        try:
            m = ImageCollectionMatcherB200(RATIO, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
            m.upload(views)
            m.wait_uploads()
            resident = Run(ctx, m, pairs, False)
            t0 = time.perf_counter()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(int(HOLD_S * 2.0e9))    # SM cycles; the H100's clock is below 2 GHz
            m.upload(views)                               # replaces every view; its copies queue behind the sleep
            held = time.perf_counter() - t0
            uploading = Run(ctx, m, pairs, False)
        finally:
            ctx.close()
        assert held < HOLD_S / 2, f"{case}: the upload call took {held:.2f} s, the hold may have ended before the match call"
        check_run(uploading, want, sizes, pairs, False, len(pending_plan), f"{case} uploading")
        check_run(resident, want, sizes, pairs, False, len(resident_plan), f"{case} resident")
        assert uploading.bytes == resident.bytes, case
        if case == "composition":
            fused_up = fused_u8_pairs(sizes, batches_of(pending_plan, processing_order(pairs, rank)))
            fused_res = fused_u8_pairs(sizes, batches_of(resident_plan, processing_order(pairs)))
            assert fused_up and not fused_res and any(restrict(want, [p]) for p in fused_up)


@pytest.mark.gpu
def test_reused_context_equals_fresh(world, answers):
    """Three calls on one context (3, then 1, then 4 batches) return the lists of fresh contexts: nothing of a buffer set outlives
    its call."""
    sizes, descs, xys = world
    L = scene_lists()
    views = {v: (descs[v], xys[v]) for v in range(N_IDS) if v in sizes}
    seq = [("three", 3), ("pair_cap", 1), ("four", 4)]
    with pytest.MonkeyPatch.context() as mp:
        ctx, m = open_context(mp, {}, views)
    try:
        reused = [Run(ctx, m, L[case][0], False) for case, _ in seq]
    finally:
        ctx.close()
    for (case, nb), r in zip(seq, reused):
        with pytest.MonkeyPatch.context() as mp:
            ctx, m = open_context(mp, {}, views)
        try:
            fresh = Run(ctx, m, L[case][0], False)
        finally:
            ctx.close()
        pairs = L[case][0]
        want = restrict(answers[False], pairs)
        check_run(r, want, sizes, pairs, False, nb, f"{case} reused")
        check_run(fresh, want, sizes, pairs, False, nb, f"{case} fresh")
        assert r.bytes == fresh.bytes, case


# ---------------------------------------------------------------------------------------------- every kernel class in every batch
CLASSES = ["u8", "ng", "fp16", "real", "exact_f32", "exact_u8", "generic"]
K_DB, L_Q = 30, 50          # database / query views per class: 10500 directed pairs, three batches


def noise_rows(rng, n):
    """Rows of 150 + N(0, 1/4): every distance among them lies deep inside the real-valued filter's error bound (undecided)."""
    return (150 + rng.normal(0, 0.25, (n, 128))).astype(np.float32)


def class_view(rng, pool, gpool, cls, m):
    if cls == "generic":                                   # AKAZE-like float x 64: the generic exact kernel
        sel = rng.choice(len(gpool), m, replace=False)
        return np.ascontiguousarray((gpool[sel] + rng.normal(0, 2.5, (m, 64))).astype(np.float32))
    d = sift_view(rng, pool, m, m)
    if cls == "u8":                                        # integer-valued fp32 in 0..255: staged as uchar, u8 kernel
        return d.astype(np.float32)
    if cls == "ng":                                        # ... in 0..127 (databases of >= 128 rows): u8 norm-GEMM kernel
        return np.minimum(d, 127).astype(np.float32)
    if cls == "fp16":                                      # signed integers: fp16 kernel
        return d.astype(np.float32) - np.float32(64)
    if cls == "real":                                      # real-valued: filter kernel; noise rows in all four chunks fall back
        x = d.astype(np.float32) + rng.normal(0, 0.37, d.shape).astype(np.float32)
        rows = [r for r in (3, 19, 35, 48, 9, 25, 41, 49) if r < m]
        x[rows] = noise_rows(rng, len(rows))
        return np.ascontiguousarray(x)
    big = np.zeros(128, np.int32); big[:8] = 1000               # ||v||^2 = 8e6 >= 2^22: the exact kernels
    if cls == "exact_f32":
        x = d.astype(np.float32); x[0] = big
        return x
    x = d.copy(); x[0] = 255                                      # uchar row of norm 128 * 255^2 >= 2^22
    return x


def class_scene(seed=8201):
    """Database view k of class c has id 7k + c, so PairSet order cycles through the classes every 7 database views (350 pairs).
    The norm-GEMM class's database views have 128 to 160 rows (one full tile at least), every other class's at most 50."""
    rng = np.random.default_rng(seed)
    pool, gpool = synth.sift_pool(48, rng), rng.gamma(2.0, 20.0, (48, 64))
    descs, cls_of, pairs = {}, {}, []
    for k in range(K_DB):
        for c, cls in enumerate(CLASSES):
            v = len(CLASSES) * k + c
            m = 50 if cls == "real" else int(rng.integers(128, 161)) if cls == "ng" else int(rng.integers(2, 41))
            descs[v] = class_view(rng, pool, gpool, cls, m)
            cls_of[v] = cls
    q0 = len(CLASSES) * K_DB
    for c, cls in enumerate(CLASSES):
        for k in range(L_Q):
            v = q0 + L_Q * c + k
            descs[v] = class_view(rng, pool, gpool, cls, int(rng.integers(1, 41)))
            cls_of[v] = cls
            pairs += [(len(CLASSES) * a + c, v) for a in range(K_DB)]
    xys = {v: synth.positions(len(d), rng) for v, d in descs.items()}
    return descs, xys, cls_of, sorted(pairs)


def test_class_scene_batches():
    descs, _, cls_of, pairs = class_scene()
    sizes = {v: len(d) for v, d in descs.items()}
    plan = plan_of(sizes, pairs)
    assert len(plan) >= 3
    for b in batches_of(plan, processing_order(pairs)):
        assert {cls_of[a] for a, _ in b} == set(CLASSES)


def oracle_view_list(descs, xys, keep, dim, dtype):
    n = max(descs) + 1
    ds = [descs[v] if v in keep else np.zeros((0, dim), dtype) for v in range(n)]
    xs = [xys[v] if v in keep else np.zeros((0, 2), np.float32) for v in range(n)]
    return ds, xs


@pytest.mark.gpu
def test_every_kernel_class_in_every_batch(ora):
    """One L2 list across three batches (PAIR_CAP) whose every batch launches the u8, u8 norm-GEMM, fp16, real-valued (filter,
    re-scoring and per-pair fallback), exact f32 / u8 and generic kernels into one candidate array; the work items of all four
    tensor-core classes share each batch's item table."""
    descs, xys, cls_of, pairs = class_scene()
    sizes = {v: len(d) for v, d in descs.items()}
    plan = plan_of(sizes, pairs)
    per = {c: sum(cls_of[a] == c for a, _ in pairs) for c in CLASSES}
    want = {}
    groups = {"f32": ({"u8", "ng", "fp16", "real", "exact_f32"}, 128, np.float32, ora), "u8": ({"exact_u8"}, 128, np.uint8, ora),
              "generic": ({"generic"}, 64, np.float32, oracle.Oracle("port"))}
    for keep_cls, dim, dt, checker in groups.values():
        keep = {v for v, c in cls_of.items() if c in keep_cls}
        ds, xs = oracle_view_list(descs, xys, keep, dim, dt)
        want.update(checker.collection_match(ds, xs, [p for p in pairs if p[0] in keep], RATIO))
    for c in CLASSES:
        assert sum(len(v) for k, v in want.items() if cls_of[k[0]] == c) > 0, c
    with pytest.MonkeyPatch.context() as mp:
        ctx, m = open_context(mp, {}, {v: (descs[v], xys[v]) for v in descs})
    try:
        r = Run(ctx, m, pairs, False)
    finally:
        ctx.close()
    assert r.batches == len(plan) >= 3
    assert (r.tc, r.u8, r.ng, r.real) == (per["u8"] + per["ng"] + per["fp16"], per["u8"] + per["ng"], per["ng"], per["real"])
    assert r.errors == 0 and r.fallback > 0
    assert_same(r.got, want, "classes")


@pytest.mark.gpu
def test_hamming_list_over_two_batches(ora):
    """More than PAIR_CAP pairs of small MLDB views (the Hamming kernel) in one call."""
    rng = np.random.default_rng(8301)
    d, _ = synth.mldb_images(130, 40, seed=8301)
    descs = [x[:int(rng.integers(2, 41))] for x in d]
    xys = [synth.positions(len(x), rng) for x in descs]
    pairs = [(a, b) for a in range(65) for b in range(65, 130)]
    sizes = {v: len(x) for v, x in enumerate(descs)}
    plan = plan_of(sizes, pairs)
    assert plan == [4096, 129]
    want = ora.collection_match(descs, xys, pairs, RATIO, hamming=True)
    assert len(want) > 0.1 * len(pairs)
    with pytest.MonkeyPatch.context() as mp:
        ctx, m = open_context(mp, {}, {v: (descs[v], xys[v]) for v in range(130)}, hamming=True)
    try:
        r = Run(ctx, m, pairs, False)
    finally:
        ctx.close()
    assert r.batches == 2 and r.tc == 0 and r.errors == 0
    assert_same(r.got, want, "hamming")


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["query", "database"])
def test_view_too_large_for_one_batch(side):
    """A query view above CAND_CAP rows or a database view above SLOT_CAP / 2 rows is refused with B200M_ERR_UNSUPPORTED before
    anything is queued; the context then runs the next list normally (one-dimensional uchar views keep the upload small)."""
    rng = np.random.default_rng(8401)
    big = np.zeros(((CAND_CAP if side == "query" else SLOT_CAP // 2) + 1, 1), np.uint8)
    small = rng.integers(0, 255, (40, 1)).astype(np.uint8)
    ctx = matching.Context(0)
    try:
        m = ImageCollectionMatcherB200(RATIO, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
        m.upload({0: (small, None), 1: (big, None), 2: (small[:20].copy(), None)})
        m.wait_uploads()
        pair = (0, 1) if side == "query" else (1, 0)
        with pytest.raises(matching.B200MatchError, match=r"status 4\).*too large"):
            m.match_uploaded(np.array([pair, (0, 2)], np.uint32), matching.STAGE_DEVICE)
        m.match_uploaded(np.array([(0, 2)], np.uint32), matching.STAGE_DEVICE)
        assert ctx.last_batches() == 1
    finally:
        ctx.close()
