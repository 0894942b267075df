"""The fundamental_matrix filter stage on putative lists that mix planar pairs and pairs of two equidistant cameras
(robustModelEstimation_F_AC with `bearings`): which pairs are spherical, the generator contract of chain=False / chain=True against a
host replay of the reference (planar and spherical oracles, the generator handed on by spherical pairs only), and guided matching
with the spherical F on the guided positions (K7 oracle)."""
from __future__ import annotations

import numpy as np
import pytest

import test_geometric_filter as tg
from alicevision_b200 import matching
from oracle import acransac as acr_oracle
from oracle import acransac_s as acrs
from oracle import guided_fast as gfo

FISHEYE = {0, 1, 2, 3, 5}      # views given bearings: pairs among them are spherical


def _lift(xy: np.ndarray, size) -> np.ndarray:
    """A stand-in for toUnitSphere(removeDistortion(ima2cam(x))): the unit vector of ((x - cx) / f, (y - cy) / f, 1)."""
    v = np.c_[(xy[:, 0] - size[0] / 2) / 1500.0, (xy[:, 1] - size[1] / 2) / 1500.0, np.ones(len(xy))]
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _bearings(regions, sizes):
    return {v: {t: _lift(r.positions.astype(np.float64), sizes[v]) for t, r in regions[v].items()} for v in FISHEYE}


def _inputs(regions, put, p, bear):
    types = [t for t in matching.DESCRIBER_TYPES if t in regions[p[0]] and t in regions[p[1]]]
    if bear is not None:
        return types, np.concatenate([np.zeros((0, 6))] + [np.c_[bear[p[0]][t][put[p][t]["i"]], bear[p[1]][t][put[p][t]["j"]]]
                                                           for t in types if t in put[p]])
    return types, np.concatenate([np.zeros((0, 4))] + [np.c_[regions[p[0]][t].positions[put[p][t]["i"]], regions[p[1]][t].positions[put[p][t]["j"]]]
                                                       for t in types if t in put[p]]).astype(np.float64)


def test_spherical_pairs_need_bearings_on_both_views_for_every_type():
    regions, sizes = tg._ring_scene(n_views=4, n_points=200, fresh=20)
    pairs = [(0, 1), (0, 2), (1, 2), (2, 3)]
    common = {p: [t for t in matching.DESCRIBER_TYPES if t in regions[p[0]] and t in regions[p[1]]] for p in pairs}
    put = {p: {t: np.zeros(0, matching.MATCH_DTYPE) for t in common[p]} for p in pairs}
    bear = {v: {t: _lift(r.positions.astype(np.float64), sizes[v]) for t, r in regions[v].items()} for v in (0, 2)}
    assert sorted(matching._spherical_inputs(put, regions, bear, common, pairs)) == [(0, 2)]   # (0, 1), (1, 2), (2, 3): one side only
    partial = {0: bear[0], 2: {"sift": bear[2]["sift"]}}                                      # view 2 lacks akaze_mldb, common with 0
    with pytest.raises(ValueError):
        matching._spherical_inputs(put, regions, partial, common, pairs)
    short = {0: bear[0], 2: {t: b[:-1] for t, b in bear[2].items()}}
    with pytest.raises(ValueError):
        matching._spherical_inputs(put, regions, short, common, pairs)


@pytest.fixture(scope="module")
def stage_scene():
    regions, sizes = tg._ring_scene()
    pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)]
    ctx = matching.Context(0)
    put = tg._putatives(regions, pairs, ctx)
    yield ctx, regions, sizes, pairs, put, _bearings(regions, sizes)
    ctx.close()


def _replay(regions, sizes, pairs, put, bear, seed, max_it, chain):
    """The reference's robustModelEstimation on the host: per pair the planar or spherical oracle, from the caller's state
    (chain=False) or from the state the last spherical pair left (chain=True)."""
    fo, so = acr_oracle.best(), acrs.AcransacSOracle("port")
    st = fo.mt_seed(seed)
    out = {}
    for p in pairs:
        sph = p[0] in FISHEYE and p[1] in FISHEYE
        _, c = _inputs(regions, put, p, bear if sph else None)
        if sph:
            out[p] = so.estimate(c, st, max_it)
            if chain:
                st = out[p]["mt_state_out"]
        else:
            out[p] = fo.estimate(c, sizes[p[0]] + sizes[p[1]], st, max_it)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [False, True])
@pytest.mark.parametrize("guided", [False, True])
def test_gpu_mixed_list(stage_scene, chain, guided):
    ctx, regions, sizes, pairs, put, bear = stage_scene
    seed, max_it = 42, 2000
    out, info = matching.robustModelEstimation_F_AC(put, regions, sizes, seed, max_it, guidedMatching=guided, ctx=ctx, bearings=bear, chain=chain)
    want = _replay(regions, sizes, pairs, put, bear, seed, max_it, chain)
    O = gfo.best()
    st = matching.mt19937_state(seed)
    n_sph = compared = kept = 0
    for p in pairs:
        sph = p[0] in FISHEYE and p[1] in FISHEYE
        assert info[p]["spherical"] == sph, p
        types, c = _inputs(regions, put, p, bear if sph else None)
        if sph:
            n_sph += 1
            assert c.shape[1] == 6 and ("mt_state_out" in info[p])
            got = ctx.acransac_fundamental_spherical_pairs([c], st, max_it)[0]
            assert np.array_equal(got["F"], info[p]["F"]) and got["valid"] == info[p]["valid"], p
            if chain:   # the next spherical pair starts from this one's end state (the engine's, also after a rounding-level fork)
                st = got["mt_state_out"]
        else:
            got = ctx.acransac_fundamental_pairs([c], [sizes[p[0]] + sizes[p[1]]], st, max_it)[0]
            assert np.array_equal(got["F"], info[p]["F"]) and got["valid"] == info[p]["valid"], p
        w = want[p]
        if got["n_trace"] == w["n_trace"] and np.array_equal(got["trace"], w["trace"]):
            compared += 1
            # the same inlier set (the order of the 7 fitted correspondences, at rounding level, follows the model's last bits;
            # copyInlierMatches sorts the indices)
            assert got["valid"] == bool(w["valid"]) and np.array_equal(np.sort(got["inliers"]), np.sort(w["inliers"])), p
            if sph:
                assert np.array_equal(got["mt_state_out"], w["mt_state_out"]), p
            exp_keep = bool(w["valid"]) and matching.hasStrongSupport(matching.copyInlierMatches(w["inliers"], put[p], types))
            assert (p in out) == exp_keep, p
        if p in out:
            kept += 1
            if guided:   # guidedMatching<Mat3Model, FundamentalEpipolarDistanceError> with this pair's F on the guided positions
                assert sorted(out[p]) == sorted(types)
                for t in types:
                    r0, r1 = regions[p[0]][t], regions[p[1]][t]
                    wl = O.guided_match(r0.descriptors, r0.positions.astype(np.float64), r1.descriptors, r1.positions.astype(np.float64),
                                        info[p]["F"], info[p]["error_max"] ** 2, 0.36, binary=r0.binary)
                    assert tg._same_ij(out[p][t], wl), (p, t)
            else:
                inl = matching.copyInlierMatches(got["inliers"], put[p], types)
                assert all(np.array_equal(out[p][t], inl[t]) for t in inl), p
    assert n_sph == 10 and compared >= len(pairs) // 2 and kept >= 5, (n_sph, compared, kept)
    assert any(info[p]["spherical"] and p in out for p in pairs)


@pytest.mark.gpu
def test_gpu_without_spherical_pairs_unchanged(stage_scene):
    """No bearings, bearings on one view only, or chain=True without spherical pairs: the stage's single planar call, unchanged."""
    ctx, regions, sizes, pairs, put, bear = stage_scene
    base = matching.robustModelEstimation_F_AC(put, regions, sizes, 7, 1000, ctx=ctx)
    for kw in ({"bearings": {0: bear[0]}}, {"chain": True}, {"bearings": {0: bear[0]}, "chain": True}):
        out, info = matching.robustModelEstimation_F_AC(put, regions, sizes, 7, 1000, ctx=ctx, **kw)
        assert out.keys() == base[0].keys() and all(not i["spherical"] for i in info.values())
        for p in pairs:
            assert np.array_equal(info[p]["F"], base[1][p]["F"]) and info[p]["error_max"] == base[1][p]["error_max"], (p, kw)


def test_spherical_filter_patch_applies(tmp_path):
    """aliceVision_b200_sphericalFilter.patch applies after aliceVision_b200.patch, _geometricFilter and _homographyFilter to copies of
    the reference files they touch, and replaces the equidistant early return with the lift and addPairSpherical."""
    import os
    import re
    import shutil
    import subprocess
    src = tg._reference_src()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    patches = [os.path.join(root, "integration", "patches", f"aliceVision_b200{s}.patch")
               for s in ("", "_geometricFilter", "_homographyFilter", "_sphericalFilter")]
    files = sorted({m for p in patches for m in re.findall(r"^\+\+\+ b/(\S+)", open(p).read(), re.M)})
    for f in files:
        dst = tmp_path / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copy(os.path.join(os.path.dirname(src), f), dst)
    for p in patches:
        r = subprocess.run(["patch", "-p1", "-s", "-i", p], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, (p, r.stdout + r.stderr)
    text = (tmp_path / "src" / "software" / "pipeline" / "main_featureMatching.cpp").read_text()
    assert "addPairSpherical(" in text and "toUnitSphere(cam->removeDistortion(cam->ima2cam(" in text
    assert "Equidistant*>(camJ))\n            return false;" not in text


@pytest.mark.gpu
def test_gpu_spherical_filter_cpp_adaptor():
    """The C++ batch adaptor on a list of planar and spherical pairs against the "ref" oracles in one executable."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "oracle", "_ref", "spherical_filter_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "spherical_filter adaptor ok" in r.stdout
