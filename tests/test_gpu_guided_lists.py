"""The three guided-matching pair-list calls on resident views - b200m_guided_match_fast_pairs (K9), b200m_guided_match_pairs (K7) and
b200m_guided_match_positions_pairs (position-only) - over one list of views: every descriptor storage class, a mixed pair each way,
an empty view, a pair with no common descriptor type, a duplicated pair, views with and without geometry positions.  They share the
list check, the batching rule (DESIGN.md K7) and the result assembly; this pins all three on the same inputs: every list equals its
oracle, the lists do not depend on the left-feature bound, launch counts follow the batch grouping, and a bad entry anywhere in a list
is rejected before anything runs."""
import ctypes as C

import numpy as np
import pytest

import oracle
import test_guided_fast as gft
from oracle import guided_fast as gfo
from oracle import guided_positions as gpo
from alicevision_b200 import synth

TH, RATIO, POS_TH = 16.0, 0.64, 4.0
EMPTY, NOPOS, F64, GEOM_ONLY = 13, 20, 21, 23


def _scenes():
    """views {id: (descriptors, upload positions or None, geometry positions or None, binary)} and the geometry of each scene
    {left id: (F, ep2, W, H)}.  Ids 3/4 and 7/10 are integer-valued fp32 (stored as uchar); 7/8 is uchar-stored left / real right,
    9/10 the reverse."""
    views, geo = {}, {}

    def add(a, b, s, dl, dr, geom):
        views[a] = (dl, s["xl"], s["ul"] if a in geom else None, False)
        views[b] = (dr, s["xr"], s["ur"] if b in geom else None, False)
        geo[a] = (s["F"], s["ep2"], s["W"], s["H"])

    for a, kind, geom_ids, seed in ((1, "u8", (1, 2), 3), (3, "f32", (), 5), (5, "real", (5,), 7), (7, "mixed", (8,), 9)):
        s = gft.two_view(kind, "outside", 1000, seed=seed, k1=-0.05)
        add(a, a + 1, s, s["dl"], s["dr"], geom_ids)
    s = gft.two_view("f32", "inside", 1000, seed=11, k1=-0.05)
    add(9, 10, s, synth.real_valued([s["dl"]])[0], s["dr"], (9, 10))
    s = gft.two_view("bin", "outside", 1000, seed=13, k1=-0.05)
    add(11, 12, s, s["dl"], s["dr"], (12,))
    views[11] = views[11][:3] + (True,); views[12] = views[12][:3] + (True,)
    d1, x1 = views[1][0], views[1][1]
    views[EMPTY] = (d1[:0], x1[:0], None, False)                                # empty, no positions
    views[NOPOS] = (d1, None, None, False)                                      # no positions of either kind
    f64 = np.ascontiguousarray(views[5][0][:, :64])
    views[F64] = (f64, views[5][1], None, False)                                # 64-component fp32: no descriptor call takes it
    views[F64 + 1] = (np.ascontiguousarray(views[6][0][:, :64]), views[6][1], None, False)
    geo[F64] = geo[5]
    views[GEOM_ONLY] = (d1, None, views[1][2], False)                           # geometry positions only
    geo[GEOM_ONLY] = geo[1]
    return views, geo


VIEWS, GEO = _scenes()
# uchar, uchar-stored fp32, real fp32, mixed both ways, binary, pairs with an empty view / no common type (empty lists, unchecked
# positions), and duplicates of a uchar and a mixed pair
PAIRS = [(1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (1, EMPTY), (EMPTY, 2), (1, 12), (EMPTY, NOPOS), (NOPOS, 12), (1, 2), (7, 8)]
RUN = [(1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (1, 2), (7, 8)]       # the pairs that are matched


def _geo(pair):
    return GEO.get(pair[0], GEO[1])


def _pos(v):
    d, xy, g, _ = VIEWS[v]
    return g if g is not None else xy.astype(np.float64)


def _skipped(a, b):
    (da, xa, _, ba), (db, xb, _, bb) = VIEWS[a], VIEWS[b]
    return len(da) == 0 or len(db) == 0 or ba != bb or da.dtype != db.dtype or da.shape[1] != db.shape[1]


def _want(call, a, b, decorate=False):
    if _skipped(a, b):
        return np.zeros(0, oracle.MATCH_DTYPE)
    (da, xa, ga, binary), (db, xb, gb, _) = VIEWS[a], VIEWS[b]
    F, ep2, W, H = _geo((a, b))
    if call == "fast":
        return gfo.best().guided_fast(da, _pos(a), db, _pos(b), F, ep2, W, H, TH, RATIO, binary=binary)
    if call == "guided":
        if ga is None and gb is None:
            return oracle.best().guided_match(da, xa, db, xb, F, TH, RATIO, binary=binary)
        return gfo.best().guided_match(da, _pos(a), db, _pos(b), F, TH, RATIO, binary=binary)
    m = gpo.GuidedPositionsOracle().guided_match_positions(_pos(a), _pos(b), F, POS_TH, 0)
    return oracle.best().decorator_dedup(m, xa, xb) if decorate and len(m) else m


def _upload(ctx, ids):
    from alicevision_b200 import matching
    for v in ids:
        d, xy, g, binary = VIEWS[v]
        code = matching.BIN if binary else matching._dtype_code(d, False)
        n = len(d)
        xy_p = np.ascontiguousarray(xy, np.float32).ctypes.data_as(C.c_void_p) if xy is not None and n else None
        matching._check(ctx.lib.b200m_upload_view(ctx._h, C.c_uint32(v), d.ctypes.data_as(C.c_void_p) if n else None, C.c_int(n),
                                                  C.c_int(d.shape[1]), C.c_int(code), xy_p), "b200m_upload_view")
        if g is not None:
            ctx.set_view_geometry(v, g)


def _call(ctx, call, pairs, decorate=False, wh=None):
    """One call over `pairs`; returns one list per pair, in input order."""
    geo = [_geo(p) for p in pairs]
    if call == "fast":
        whs = wh if wh is not None else [(g[2], g[3]) for g in geo]
        got = ctx.guided_match_fast_pairs(pairs, [g[0] for g in geo], [g[1] for g in geo], whs, TH, RATIO)
        assert list(got) == list(dict.fromkeys(map(tuple, pairs)))
        return [got[tuple(p)] for p in pairs]
    if call == "guided":
        return ctx.guided_match_pairs(pairs, [g[0] for g in geo], [TH] * len(pairs), RATIO)
    from alicevision_b200 import matching
    return ctx.guided_match_positions_pairs(pairs, [g[0] for g in geo], [POS_TH] * len(pairs), matching.MODEL_FUNDAMENTAL, decorate)


def _same(got, want):
    return len(got) == len(want) and np.array_equal(got["i"], want["i"]) and np.array_equal(got["j"], want["j"])


def _general_position(v):
    xy = VIEWS[v][1]
    return len(np.unique(xy[:, 0])) == len(xy) and len(np.unique(xy[:, 1])) == len(xy)


CALLS = [("fast", False), ("guided", False), ("positions", False), ("positions", True)]
# Launches per call at the default bounds: the matched pairs form one batch per kernel class - uchar {(1, 2), (3, 4), (1, 2)}, fp32
# {(5, 6)}, binary {(11, 12)}, mixed {(7, 8), (9, 10), (7, 8)} with two expansions (views 7 and 10, each once) - and the position-only
# call, which reads no descriptors, has one batch.  Per batch K9 counts 11 (three CUB scans of 2 launches each and 5 for its own
# kernels), K7 4 (guided_pairs_kernel and emit, one scan), the position-only call 4 (its kernel and emit, one scan) and one more for
# the device decorator when a left view of the batch is in general position; each expansion is one u8_to_f32_kernel.
DEFAULT_LAUNCHES = {("fast", False): 4 * 11 + 2, ("guided", False): 4 * 4 + 2, ("positions", False): 4}


@pytest.mark.gpu
def test_gpu_guided_lists_equal_oracle_at_any_left_bound(monkeypatch):
    """Every list equals its oracle; lists and last_records() are the same at the default bounds and with a left bound of 1 (every
    pair runs alone); last_launches() at the default bounds follows the batch grouping."""
    from alicevision_b200 import matching
    want = {(call, deco): [_want(call, a, b, deco) for a, b in PAIRS] for call, deco in CALLS}
    assert sum(len(w) > 0 for w in want[("fast", False)]) == len(RUN)
    assert sum(len(w) > 0 for w in want[("guided", False)]) == len(RUN)
    results = []
    for cap in (None, "1"):
        if cap:
            monkeypatch.setenv("B200M_GUIDED_FAST_LEFT_CAP", cap)
            monkeypatch.setenv("B200M_GUIDED_LEFT_CAP", cap)
        ctx = matching.Context(0)
        try:
            _upload(ctx, sorted(VIEWS))
            run = {}
            for call, deco in CALLS:
                got = _call(ctx, call, PAIRS, deco)
                for (a, b), g, w in zip(PAIRS, got, want[(call, deco)]):
                    assert _same(g, w), (call, deco, a, b, len(g), len(w))
                    assert not g["ratio"].any() and not g["dist"].any()
                if call == "fast":
                    assert ctx.last_records() >= sum(len(g) for g in got)      # K9 reports its candidates
                else:
                    assert ctx.last_records() == sum(len(g) for g in got)
                run[(call, deco)] = (got, ctx.last_records(), ctx.last_launches())
            if cap is None:
                for key, n in DEFAULT_LAUNCHES.items():
                    assert run[key][2] == n, (key, run[key][2], n)
                dev_deco = any(_general_position(a) for a, _ in RUN)
                assert run[("positions", True)][2] == 4 + dev_deco
            else:
                # every matched pair alone: 8 batches, one expansion per mixed pair
                assert run[("fast", False)][2] == 8 * 11 + 3 and run[("guided", False)][2] == 8 * 4 + 3
                assert run[("positions", False)][2] == 8 * 4
            results.append(run)
        finally:
            ctx.close()
    for key in results[0]:
        (g0, r0, _), (g1, r1, _) = results[0][key], results[1][key]
        assert r0 == r1 and all(_same(a, b) for a, b in zip(g0, g1)), key


@pytest.mark.gpu
def test_gpu_guided_lists_checks_run_first():
    """A list whose last entry is bad is rejected with its status, and nothing runs: last_launches(), last_records() and
    last_gpu_ms() still hold the previous call's values."""
    from alicevision_b200 import matching
    ctx = matching.Context(0)
    try:
        _upload(ctx, sorted(VIEWS))
        good = PAIRS[:6]
        bad = {"fast": [([(1, 999999)], 1), ([(1, NOPOS)], 1), ([(F64, F64 + 1)], 4)],
               "guided": [([(1, 999999)], 1), ([(1, NOPOS)], 1), ([(F64, F64 + 1)], 4)],
               "positions": [([(1, 999999)], 1), ([(NOPOS, 2)], 1)]}
        for call, cases in bad.items():
            for tail, status in cases:
                _call(ctx, call, good)
                before = (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms())
                with pytest.raises(matching.B200MatchError, match=rf"\(status {status}\)"):
                    _call(ctx, call, good + tail)
                assert (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms()) == before, (call, tail)
        # the fast call checks W and H first for each entry: W < 2 on an entry that also names an unknown view
        _call(ctx, "fast", good)
        before = (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms())
        wh = [(_geo(p)[2], _geo(p)[3]) for p in good] + [(1, 3000)]
        with pytest.raises(matching.B200MatchError, match=r"\(status 1\).*pair 6: the right image must be at least 2 x 2"):
            _call(ctx, "fast", good + [(1, 999999)], wh=wh)
        assert (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms()) == before
        # the decorator needs upload positions; undecorated, geometry positions are enough
        _call(ctx, "positions", good, True)
        before = (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms())
        with pytest.raises(matching.B200MatchError, match=r"\(status 1\).*decorator needs the upload positions"):
            _call(ctx, "positions", good + [(GEOM_ONLY, 2)], True)
        assert (ctx.last_launches(), ctx.last_records(), ctx.last_gpu_ms()) == before
        got = _call(ctx, "positions", good + [(GEOM_ONLY, 2)])
        assert _same(got[-1], _want("positions", GEOM_ONLY, 2)) and len(got[-1]) > 0
        # the position-only call reads no descriptors: 64-component fp32 views are matched
        for deco in (False, True):
            got = _call(ctx, "positions", good + [(F64, F64 + 1)], deco)
            assert _same(got[-1], _want("positions", F64, F64 + 1, deco)) and len(got[-1]) > 0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_guided_lists_empty_cases():
    """A pair with an empty view and no positions gets an empty list without an error, in every call; an empty list of pairs gives
    an empty result."""
    from alicevision_b200 import matching
    ctx = matching.Context(0)
    try:
        _upload(ctx, sorted(VIEWS))
        for call, deco in CALLS:
            got = _call(ctx, call, [(EMPTY, NOPOS), (NOPOS, EMPTY), (EMPTY, EMPTY)], deco)
            assert [len(g) for g in got] == [0, 0, 0], call
            assert ctx.last_records() == 0 and ctx.last_launches() == 0
        z2, z9 = np.zeros((0, 2), np.uint32), np.zeros((0, 9))
        assert ctx.guided_match_fast_pairs(z2, z9, np.zeros((0, 3)), np.zeros((0, 2), np.int32), TH, RATIO) == {}
        assert ctx.guided_match_pairs(z2, z9, np.zeros(0), RATIO) == []
        for deco in (False, True):
            assert ctx.guided_match_positions_pairs(z2, z9, np.zeros(0), matching.MODEL_FUNDAMENTAL, deco) == []
    finally:
        ctx.close()
