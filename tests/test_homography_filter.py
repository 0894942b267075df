"""The `homography_matrix` geometric filter on a putative list: position-only guided matching over a pair list
(b200m_guided_match_positions_pairs: guidedMatching.hpp:37-70, then IndMatchDecorator::getDeduplicated) and the robustModelEstimation stage
around it (matching.robustModelEstimation_H_AC: K10 H, the reference's inlier copy and hasStrongSupport(.., 4), then guided matching of the
kept pairs).  Position-only lists are compared with oracle/guided_positions (the reference loop on double positions) followed by the
oracle's decorator (the compiled reference's IndMatchDecorator when it is built)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from alicevision_b200 import matching, synth
from oracle import acransac_h as acrh
from oracle import guided_fast as gfo
from oracle import guided_positions as gpo

W, H = 4000, 3000
HOM = np.array([[0.96, 0.03, 25.0], [-0.02, 1.02, -14.0], [1.5e-5, -2.0e-5, 1.0]], np.float64)
F_RECT = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)          # x_r^T F x_l = 0 <=> y_r == y_l
DBL_MAX = np.finfo(np.float64).max
Hm, Fm = matching.MODEL_HOMOGRAPHY, matching.MODEL_FUNDAMENTAL


def _np_positions(model, xl, xr, M, th):
    """guidedMatching.hpp:37-70 + IndMatch::getDeduplicated restated with numpy (IEEE double, no contraction)."""
    out = set()
    y0, y1 = xr[:, 0], xr[:, 1]
    with np.errstate(all="ignore"):
        for i, (x0, x1) in enumerate(xl):
            f0 = (M[0, 0] * x0 + M[0, 1] * x1) + M[0, 2] * 1.0
            f1 = (M[1, 0] * x0 + M[1, 1] * x1) + M[1, 2] * 1.0
            f2 = (M[2, 0] * x0 + M[2, 1] * x1) + M[2, 2] * 1.0
            if model == Hm:
                d0, d1 = y0 - f0 / f2, y1 - f1 / f2
                err = d0 * d0 + d1 * d1
            else:
                dot = (f0 * y0 + f1 * y1) + f2 * 1.0
                err = (dot * dot) / (f0 * f0 + f1 * f1)
            ok = (err < th) & (err < DBL_MAX)
            if ok.any():
                out.add((i, int(np.argmin(np.where(ok, err, np.inf)))))       # the first j of the smallest error
            elif DBL_MAX < th:
                out.add((0, 0))                                                # the default IndMatch the reference pushes
    m = np.zeros(len(out), matching.MATCH_DTYPE)
    if out:
        ij = np.array(sorted(out))
        m["i"], m["j"] = ij[:, 0], ij[:, 1]
    return m


def _same_ij(a, b):
    return len(a) == len(b) and np.array_equal(a["i"], b["i"]) and np.array_equal(a["j"], b["j"])


# ---------------------------------------------------------------------------------------------- CPU
def test_oracle_positions_equals_numpy():
    """The oracle's loop against the numpy restatement: exact ties (duplicate right positions: the first j wins), w = 0 rows, threshold 0,
    +inf (a left feature without a finite error contributes (0, 0)), NaN, and an empty side."""
    O = gpo.GuidedPositionsOracle()
    rng = np.random.default_rng(3)
    xl = np.stack([rng.uniform(0, W, 300), rng.uniform(0, H, 300)], 1)
    p = np.c_[xl, np.ones(300)] @ HOM.T
    xr = np.concatenate([p[:, :2] / p[:, 2:] + rng.uniform(-2, 2, (300, 2)), np.stack([rng.uniform(0, W, 200), rng.uniform(0, H, 200)], 1)])
    xr[400:450] = xr[100:150]                                                  # exact ties with earlier right features
    H_W0 = HOM.copy(); H_W0[2] = [1e-3, 0, -1.0]                              # (H x)[2] = 0 on the line x = 1000
    xl_w0 = xl.copy(); xl_w0[:20, 0] = 1000.0
    cases = [(Hm, xl, xr, HOM, 4.0), (Hm, xl, xr, HOM, 0.0), (Hm, xl, xr, HOM, 1e9), (Hm, xl, xr, HOM, np.inf), (Hm, xl_w0, xr, H_W0, np.inf),
             (Hm, xl_w0, xr, H_W0, 1e12), (Hm, xl, xr, np.zeros((3, 3)), np.inf), (Hm, xl, xr, HOM, np.nan), (Fm, xl, xr, F_RECT, 4.0),
             (Fm, xl, xr, F_RECT, np.inf), (Fm, xl, xr, np.zeros((3, 3)), 4.0), (Hm, xl[:0], xr, HOM, np.inf), (Hm, xl, xr[:0], HOM, 4.0)]
    ties = 0
    for k, (model, a, b, M, th) in enumerate(cases):
        got = O.guided_match_positions(a, b, M, th, model)
        assert _same_ij(got, _np_positions(model, a, b, M, th)), k
        ties += int(np.isin(got["j"], np.arange(100, 150)).sum())
    assert ties > 0
    assert _same_ij(O.guided_match_positions(xl, xr, np.zeros((3, 3)), np.inf, Hm), _np_positions(Hm, xl[:1], xr, HOM * 0, np.inf))
    assert len(O.guided_match_positions(xl, xr, HOM, 4.0, Hm)) > 200


def test_strong_support_boundary_homography():
    """hasStrongSupport(.., 4) (Homography4PSolver): 0.14f * 28 = 3.92 fails, 0.14f * 29 passes."""
    def m(n):
        return np.zeros(n, matching.MATCH_DTYPE)
    assert not matching.hasStrongSupport({"sift": m(28)}, 4)
    assert matching.hasStrongSupport({"sift": m(29)}, 4)
    assert not matching.hasStrongSupport({"sift": m(14), "akaze_mldb": m(14)}, 4)
    assert matching.hasStrongSupport({"sift": m(14), "akaze_mldb": m(15)}, 4)


def _reference_src():
    src = oracle.reference_src()
    if src is None:
        pytest.skip("no AliceVision source tree (ALICEVISION_SRC)")
    return src


def test_homography_filter_patch_applies(tmp_path):
    """aliceVision_b200_homographyFilter.patch applies after aliceVision_b200.patch and aliceVision_b200_geometricFilter.patch to copies
    of the reference files they touch."""
    import re
    import shutil
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    patches = [os.path.join(root, "integration", "patches", f"aliceVision_b200{s}.patch") for s in ("", "_geometricFilter", "_homographyFilter")]
    files = sorted({m for p in patches for m in re.findall(r"^\+\+\+ b/(\S+)", open(p).read(), re.M)})
    for f in files:
        dst = tmp_path / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copy(os.path.join(os.path.dirname(src), f), dst)
    for p in patches:
        r = subprocess.run(["patch", "-p1", "-s", "-i", p], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, (p, r.stdout + r.stderr)
    text = (tmp_path / "src" / "software" / "pipeline" / "main_featureMatching.cpp").read_text()
    assert "GeometricFilterMatrix_H_AC_Batch_b200" in text and "robustModelEstimationHOnB200(" in text


def test_homography_filter_adaptor_header_compiles():
    import subprocess
    src = _reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "alicevision_b200", "adaptor", "GeometricFilter_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(root, "oracle", "shim"), "-I", src,
                        "-I", os.path.join(root, "include"), "-I", os.path.join(root, "alicevision_b200", "adaptor"), hdr],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


# ---------------------------------------------------------------------------------------------- GPU: b200m_guided_match_positions_pairs
def _xy(rng, n):
    return np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1).astype(np.float32)


def _positions_case():
    """Views of positions (descriptors are uploaded but never read): left views in general position and with a duplicate x or y, right
    views through HOM +- noise with exact ties, an empty view, a view of another describer type, geometry positions on some views."""
    rng = np.random.default_rng(17)
    n = 1500
    xy = {0: _xy(rng, n)}
    p = np.c_[xy[0].astype(np.float64), np.ones(n)] @ HOM.T
    r = np.concatenate([p[:, :2] / p[:, 2:] + rng.uniform(-1.5, 1.5, (n, 2)), _xy(rng, 400)]).astype(np.float32)
    r[1700:1800] = r[200:300]                                                  # exact ties
    xy[1] = r
    xy[2] = xy[0].copy(); xy[2][10, 0] = xy[2][11, 0]; xy[2][500, 0] = xy[2][900, 0]     # duplicate x: not in general position
    xy[3] = xy[0].copy(); xy[3][20, 1] = xy[3][21, 1]                          # duplicate y
    xy[4] = r.copy(); xy[4][5] = xy[4][6]                                      # a right view with two features at one position
    xy[5] = xy[0][:0]                                                          # empty
    xy[6] = xy[0].copy()                                                       # another describer type (binary)
    views = {}
    for v, x in xy.items():
        if v == 6:
            views[v] = (synth.mldb_images(1, len(x), seed=v)[0][0], x, True)
        else:
            views[v] = (synth.sift_images(1, max(len(x), 1), np.uint8, seed=v, pool_factor=1.0)[0][0][:len(x)], x, False)
    geom = {1: xy[1].astype(np.float64) + rng.uniform(-0.3, 0.3, xy[1].shape), 3: xy[3].astype(np.float64) + rng.uniform(-0.2, 0.2, xy[3].shape)}
    H_INF = HOM.copy(); H_INF[2] = 0                                           # every x / 0: inf or NaN
    items = []
    for th in (0.0, 4.0, 1e9, np.inf):
        items += [(0, 1, HOM, th), (2, 1, HOM, th), (3, 4, HOM, th)]
    items += [(1, 0, np.linalg.inv(HOM), 4.0), (0, 1, HOM, 4.0), (0, 4, HOM, 16.0), (0, 1, H_INF, 4.0), (0, 1, H_INF, np.inf),
              (0, 1, np.full((3, 3), np.nan), np.inf), (0, 5, HOM, 4.0), (5, 1, HOM, np.inf), (6, 1, HOM, 4.0), (0, 1, HOM, np.nan)]
    return views, geom, items


def _upload_views(ctx, views, geom):
    for v, (d, x, binary) in views.items():
        matching._upload_pair(ctx, [v], [matching.Regions(d, x, binary=binary)], [geom.get(v)], [])


def _oracle_positions(O, D, views, geom, l, r, model, M, th, decorate):
    (dl, xl, bl), (dr, xr, br) = views[l], views[r]
    if len(xl) == 0 or len(xr) == 0 or bl != br or dl.dtype != dr.dtype:
        return np.zeros(0, matching.MATCH_DTYPE)
    m = O.guided_match_positions(geom.get(l, xl.astype(np.float64)), geom.get(r, xr.astype(np.float64)), M, th, model)
    return D.decorator_dedup(m, xl, xr) if decorate and len(m) else m


def _check_list(ctx, O, D, views, geom, items, model, decorate):
    got = ctx.guided_match_positions_pairs([it[:2] for it in items], [it[2] for it in items], [it[3] for it in items], model, decorate)
    assert ctx.last_launches() > 0 and ctx.last_records() == sum(len(g) for g in got)
    nonempty = 0
    for (l, r, M, th), g in zip(items, got):
        want = _oracle_positions(O, D, views, geom, l, r, model, M, th, decorate)
        assert _same_ij(g, want), (l, r, th, model, decorate)
        assert not g["ratio"].any() and not g["dist"].any()
        nonempty += len(g) > 0
    assert nonempty >= min(10, len(items) - 1)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("device_finish", ["1", "0"])
def test_gpu_guided_match_positions_pairs(monkeypatch, device_finish):
    """Every list equals the oracle, undecorated (ascending i) and decorated (the reference decorator applied to the oracle's list),
    for both models; with device_finish 0 the decorator runs on the host for every pair.  The same list over several internal batches
    gives the same lists."""
    monkeypatch.setenv("B200M_DEVICE_FINISH", device_finish)
    O, D = gpo.GuidedPositionsOracle(), oracle.best()
    views, geom, items = _positions_case()
    f_items = [(0, 1, F_RECT, 4.0), (2, 1, F_RECT, 1e9), (3, 4, F_RECT, np.inf), (1, 0, F_RECT.T, 4.0), (0, 1, np.zeros((3, 3)), 4.0)]
    results = []
    for cap in (None, "2000"):
        if cap:
            monkeypatch.setenv("B200M_GUIDED_LEFT_CAP", cap)
        ctx = matching.Context(0)
        try:
            _upload_views(ctx, views, geom)
            run = []
            for decorate in (False, True):
                run.append(_check_list(ctx, O, D, views, geom, items, Hm, decorate))
                run.append(_check_list(ctx, O, D, views, geom, f_items, Fm, decorate))
            results.append(run)
            if cap is None:
                # the device decorator is one launch more than the undecorated call, for a left view in general position only
                ctx.guided_match_positions_pairs([(0, 1)], [HOM], [4.0], Hm, False)
                n0 = ctx.last_launches()
                ctx.guided_match_positions_pairs([(0, 1)], [HOM], [4.0], Hm, True)
                assert ctx.last_launches() == n0 + (device_finish == "1")
                ctx.guided_match_positions_pairs([(2, 1)], [HOM], [4.0], Hm, True)
                assert ctx.last_launches() == n0
                assert ctx.guided_match_positions_pairs(np.zeros((0, 2), np.uint32), np.zeros((0, 9)), np.zeros(0)) == []
                with pytest.raises(matching.B200MatchError):
                    ctx.guided_match_positions_pairs([(0, 123456)], [HOM], [4.0])
                # geometry positions only: undecorated works, the decorator needs the upload positions
                d0 = views[0][0]
                matching._check(ctx.lib.b200m_upload_view(ctx._h, C.c_uint32(50), d0.ctypes.data_as(C.c_void_p), C.c_int(len(d0)), C.c_int(128),
                                                           C.c_int(matching.U8), None), "b200m_upload_view")
                ctx.set_view_geometry(50, views[0][1].astype(np.float64))
                g = ctx.guided_match_positions_pairs([(50, 1)], [HOM], [4.0], Hm, False)[0]
                assert _same_ij(g, O.guided_match_positions(views[0][1], geom[1], HOM, 4.0))
                with pytest.raises(matching.B200MatchError):
                    ctx.guided_match_positions_pairs([(50, 1)], [HOM], [4.0], Hm, True)
        finally:
            ctx.close()
    assert all(_same_ij(a, b) for r0, r1 in zip(*results) for a, b in zip(r0, r1))


@pytest.mark.gpu
def test_gpu_guided_match_positions_full_size():
    """One 8192 x 8192 pair among small ones, decorated and not, equal to the oracle whole."""
    O, D = gpo.GuidedPositionsOracle(), oracle.best()
    rng = np.random.default_rng(29)
    xl = _xy(rng, 8192)
    p = np.c_[xl.astype(np.float64), np.ones(8192)] @ HOM.T
    xr = (p[:, :2] / p[:, 2:] + rng.uniform(-2, 2, (8192, 2))).astype(np.float32)[rng.permutation(8192)]
    sl, sr = xl[:700], xr[:900]
    d = synth.sift_images(1, 8192, np.uint8, seed=3, pool_factor=1.0)[0][0]
    ctx = matching.Context(0)
    try:
        for v, x in enumerate((xl, xr, sl, sr)):
            matching._upload_pair(ctx, [v], [matching.Regions(d[:len(x)], x)], [None], [])
        for decorate in (False, True):
            got = ctx.guided_match_positions_pairs([(2, 3), (0, 1), (2, 3)], [HOM] * 3, [9.0] * 3, Hm, decorate)
            assert len(got[1]) > 0.9 * 8192 and _same_ij(got[0], got[2])
            for g, (a, b) in zip(got[:2], ((sl, sr), (xl, xr))):
                w = O.guided_match_positions(a, b, HOM, 9.0)
                assert _same_ij(g, D.decorator_dedup(w, a, b) if decorate else w), decorate
        assert ctx.last_search_kernel_ms() > 0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------- GPU: the filter stage
def _rotation_ring(n_views=6, n_points=900, fresh=300, seed=3):
    """A camera turning about its centre (pure rotations: every pair is related by a homography): SIFT uchar descriptors of the visible
    directions with per-view noise plus fresh features, and an AKAZE-like binary type on every other view."""
    rng = np.random.default_rng(seed)
    P = np.stack([rng.uniform(-1.2, 1.2, n_points), rng.uniform(-0.5, 0.5, n_points), np.ones(n_points)], 1)
    sift = synth.sift_images(1, n_points, np.uint8, seed=seed, pool_factor=1.0)[0][0]
    mldb = synth.mldb_images(1, n_points // 3, seed=seed)[0][0]
    K = np.array([[1500.0, 0, 960], [0, 1500.0, 540], [0, 0, 1]])
    regions, sizes = {}, {}
    for v in range(n_views):
        a = (v - n_views / 2) * 0.05
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        x = (P @ R.T) @ K.T
        xy = x[:, :2] / x[:, 2:] + rng.normal(0, 0.4, (n_points, 2))
        vis = np.flatnonzero((x[:, 2] > 0) & (xy[:, 0] > 0) & (xy[:, 0] < 1920) & (xy[:, 1] > 0) & (xy[:, 1] < 1080))
        d = np.clip(sift[vis].astype(np.int32) + rng.integers(-6, 7, (vis.size, 128)), 0, 255).astype(np.uint8)
        fd = synth.sift_images(1, fresh, np.uint8, seed=seed * 100 + v, pool_factor=1.0)[0][0]
        fxy = np.stack([rng.uniform(0, 1920, fresh), rng.uniform(0, 1080, fresh)], 1)
        perm = rng.permutation(vis.size + fresh)
        regions[v] = {"sift": matching.Regions(np.concatenate([d, fd])[perm], np.concatenate([xy[vis], fxy]).astype(np.float32)[perm])}
        if v % 2 == 0:
            bv = vis[vis < mldb.shape[0]]
            flip = rng.random((bv.size, 64, 8)) < 0.04
            bd = mldb[bv] ^ np.packbits(flip, axis=2, bitorder="little")[:, :, 0]
            regions[v]["akaze_mldb"] = matching.Regions(bd, xy[bv].astype(np.float32), binary=True)
        sizes[v] = (1920, 1080)
    return regions, sizes


def _putatives(regions, pairs, ctx):
    out = {p: {} for p in pairs}
    for t, mt in (("sift", matching.EMatcherType.BRUTE_FORCE_L2_B200), ("akaze_mldb", matching.EMatcherType.BRUTE_FORCE_HAMMING_B200)):
        views = {v: (r[t].descriptors, r[t].positions) for v, r in regions.items() if t in r}
        tp = [p for p in pairs if p[0] in views and p[1] in views]
        if tp:
            m = matching.ImageCollectionMatcherB200(0.8, False, mt, ctx).Match(views, tp)
            for p, lst in m.items():
                if len(lst):
                    out[p][t] = np.asarray(lst).copy()
    return out


def _types(regions, p):
    return [t for t in matching.DESCRIBER_TYPES if t in regions[p[0]] and t in regions[p[1]]]


def _corr(regions, put, p):
    return np.concatenate([np.zeros((0, 4))] + [np.concatenate([regions[p[0]][t].positions[put[p][t]["i"]], regions[p[1]][t].positions[put[p][t]["j"]]], 1)
                                                for t in _types(regions, p) if t in put[p]]).astype(np.float64)


def _guided_want(regions, p, t, Hmat, th, ratio):
    r0, r1 = regions[p[0]][t], regions[p[1]][t]
    if ratio < 0:
        w = gpo.GuidedPositionsOracle().guided_match_positions(r0.positions, r1.positions, Hmat, th)
        return oracle.best().decorator_dedup(w, r0.positions, r1.positions) if len(w) else w
    return gfo.best().guided_match(r0.descriptors, r0.positions.astype(np.float64), r1.descriptors, r1.positions.astype(np.float64), Hmat, th,
                                   ratio * ratio, binary=r0.binary, model=Hm)


@pytest.fixture(scope="module")
def ring():
    regions, sizes = _rotation_ring()
    pairs = [(i, j) for i in range(6) for j in range(i + 1, 6)]
    ctx = matching.Context(0)
    put = _putatives(regions, pairs, ctx)
    yield regions, sizes, pairs, put, ctx
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("guided,ratio", [(False, -1.0), (True, -1.0), (True, 0.6)])
def test_gpu_robust_model_estimation_H_AC(ring, guided, ratio):
    """K10 H per pair against the oracle under the trace protocol of the fundamental-matrix stage, the support rule, and the guided lists
    against the oracle run on the engine's own H and threshold."""
    regions, sizes, pairs, put, ctx = ring
    acr = acrh.AcransacHOracle("ref" if acrh.available("ref") else "port")
    seed, max_it = 42, 400
    out, info = matching.robustModelEstimation_H_AC(put, regions, sizes, seed, max_it, guidedMatching=guided, distanceRatio=ratio, ctx=ctx)
    state = acr.mt_seed(seed)
    kept = compared = 0
    for p in pairs:
        types = _types(regions, p)
        corr = _corr(regions, put, p)
        wh = sizes[p[0]] + sizes[p[1]]
        want = acr.estimate(corr, wh, state, max_it)
        got = ctx.acransac_homography_pairs([corr], [wh], state, max_it)[0]
        assert got["valid"] == info[p]["valid"] and np.array_equal(got["H"], info[p]["H"]), p
        if p in out:
            kept += 1
            if guided:
                assert sorted(out[p]) == sorted(types), p
                for t in types:
                    assert _same_ij(out[p][t], _guided_want(regions, p, t, info[p]["H"], info[p]["error_max"] ** 2, ratio)), (p, t)
        if not (got["n_trace"] == want["n_trace"] and np.array_equal(got["trace"], want["trace"])):
            continue
        compared += 1
        exp_keep = False
        if bool(want["valid"]):
            inl = matching.copyInlierMatches(want["inliers"], put[p], types)
            exp_keep = matching.hasStrongSupport(inl, 4)
        assert (p in out) == exp_keep, p
        if exp_keep and not guided:
            assert list(out[p]) == list(inl) and all(np.array_equal(out[p][t], inl[t]) for t in inl), p
    assert kept >= 5 and compared >= len(pairs) // 2, (kept, compared)


@pytest.mark.gpu
def test_gpu_robust_model_estimation_H_AC_chain(ring):
    """chain=True on a 6-pair list: the K10 results and end states of one generator handed from pair to pair, equal to the engine's own
    one-pair chain and to the oracle's sequential chain (after a rounding-level fork the oracle continues from the engine's state)."""
    regions, sizes, pairs, put, ctx = ring
    sub = {p: put[p] for p in pairs[:6]}
    acr = acrh.AcransacHOracle("ref" if acrh.available("ref") else "port")
    out, info = matching.robustModelEstimation_H_AC(sub, regions, sizes, 7, 300, guidedMatching=True, chain=True, ctx=ctx)
    st_g = st_o = matching.mt19937_state(7)
    agree = 0
    for p in sub:
        corr, wh = _corr(regions, put, p), sizes[p[0]] + sizes[p[1]]
        got = ctx.acransac_homography_pairs([corr], [wh], st_g, 300)[0]
        assert np.array_equal(got["H"], info[p]["H"]) and np.array_equal(got["mt_state_out"], info[p]["mt_state_out"]), p
        want = acr.estimate(corr, wh, st_o, 300)
        same = got["n_trace"] == want["n_trace"] and np.array_equal(got["trace"], want["trace"])
        if same:
            agree += 1
            assert np.array_equal(got["mt_state_out"], want["mt_state_out"]) and got["iterations"] == int(want["iterations"]), p
        assert not np.array_equal(got["mt_state_out"], st_g), p
        st_g = got["mt_state_out"]
        st_o = want["mt_state_out"] if same else got["mt_state_out"]
    assert agree >= 3
    # chain=False: every pair from the caller's state
    out0, info0 = matching.robustModelEstimation_H_AC(sub, regions, sizes, 7, 300, ctx=ctx)
    first = next(iter(sub))
    assert np.array_equal(info0[first]["H"], info[first]["H"])
    assert all(np.array_equal(info0[p]["H"], ctx.acransac_homography_pairs([_corr(regions, put, p)], [sizes[p[0]] + sizes[p[1]]],
                                                                           matching.mt19937_state(7), 300)[0]["H"]) for p in sub)


@pytest.mark.gpu
def test_gpu_robust_model_estimation_H_AC_skip_independent(ring):
    regions, sizes, pairs, put, ctx = ring
    a = matching.robustModelEstimation_H_AC(put, regions, sizes, 11, 300, guidedMatching=True, ctx=ctx)
    ctx.set_acransac_skip(False)
    try:
        b = matching.robustModelEstimation_H_AC(put, regions, sizes, 11, 300, guidedMatching=True, ctx=ctx)
    finally:
        ctx.set_acransac_skip(True)
    assert a[0].keys() == b[0].keys() and len(a[0]) >= 5
    for p in a[0]:
        assert a[0][p].keys() == b[0][p].keys() and all(np.array_equal(a[0][p][t], b[0][p][t]) for t in a[0][p]), p
        assert np.array_equal(a[1][p]["H"], b[1][p]["H"]) and a[1][p]["error_max"] == b[1][p]["error_max"], p


@pytest.mark.gpu
def test_gpu_homography_filter_cpp_adaptor():
    """The C++ batch adaptor (GeometricFilterMatrix_H_AC_Batch_b200) against the "ref" oracles in one executable."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "homography_filter_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "homography_filter adaptor ok" in r.stdout
