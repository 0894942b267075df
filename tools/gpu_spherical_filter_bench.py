"""The `fundamental_matrix` geometric filter on a fisheye rig, with guided matching, on the GPU (matching.robustModelEstimation_F_AC
with `bearings` for every view, guidedMatching=True): K10 with the spherical policy over every putative pair, then one
b200m_guided_match_pairs call over the kept pairs.  Prints one JSON line.

Workload: --views equidistant fisheye cameras (200-degree field of view, so the bearings cover more than a hemisphere) of
--features SIFT uchar features at 4000 x 3000 on a ring around a scene of 3-D points, descriptors per point with per-view noise plus
fresh features, exhaustive pairs, putatives from the engine (ImageCollectionMatcherB200, ratio 0.8), the filter at --max-iteration.
Each feature's bearing is the exact inverse of the equidistant projection of its (noisy) pixel.  Reported: the stage's wall time,
K10's GPU time and its models evaluated / skipped / exact, the guided call's GPU time, and the port oracle's spherical estimation
per pair on one CPU thread for a sample of pairs.

    python tools/gpu_spherical_filter_bench.py [--views 100] [--features 8192] [--max-iteration 50000] [--cpu-sample 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from alicevision_b200 import ImageCollectionMatcherB200, matching, synth  # noqa: E402
from gpu_known_poses_bench import H, W, card  # noqa: E402

FOV = np.radians(200.0)
F_EQ = (min(W, H) / 2) / (FOV / 2)      # equidistant: r = f theta, the 200-degree circle inscribed in the image


def fisheye_ring(n_views: int, m: int, rng):
    """n_views cameras on a circle of radius 4 looking outwards-and-up at points on a surrounding shell (radius 8..14); each view
    keeps 70 % of its features on points it sees within the field of view (observed +- 0.5 px), the rest fresh."""
    n_pts = 6 * m
    d = rng.normal(size=(n_pts, 3))
    P = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(8, 14, (n_pts, 1))
    base = synth.sift_images(1, n_pts, np.uint8, seed=5, pool_factor=1.0)[0][0]
    views, bears = [], []
    for k in range(n_views):
        a = 2 * np.pi * k / n_views
        c = np.array([4 * np.sin(a), 0.1 * np.sin(3 * a), 4 * np.cos(a)])
        R = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        X = (P - c) @ R.T
        b = X / np.linalg.norm(X, axis=1, keepdims=True)
        theta = np.arccos(np.clip(b[:, 2], -1, 1))
        phi = np.arctan2(b[:, 1], b[:, 0])
        x = np.stack([W / 2 + F_EQ * theta * np.cos(phi), H / 2 + F_EQ * theta * np.sin(phi)], 1)
        vis = np.where(theta < FOV / 2)[0]
        vis = rng.permutation(vis)[: int(0.7 * m)]
        r_f = F_EQ * FOV / 2
        u = rng.uniform(0, 2 * np.pi, m - len(vis))
        rr = r_f * np.sqrt(rng.uniform(0, 1, m - len(vis)))
        xy = np.concatenate([x[vis] + rng.uniform(-0.5, 0.5, (len(vis), 2)), np.stack([W / 2 + rr * np.cos(u), H / 2 + rr * np.sin(u)], 1)])
        d = np.concatenate([np.clip(base[vis].astype(np.int32) + rng.integers(-5, 6, (len(vis), 128)), 0, 255).astype(np.uint8),
                            synth.sift_images(1, m - len(vis), np.uint8, seed=100 + k, pool_factor=1.0)[0][0]])
        perm = rng.permutation(m)
        xy = xy[perm].astype(np.float32)
        dx, dy = xy[:, 0].astype(np.float64) - W / 2, xy[:, 1].astype(np.float64) - H / 2
        th, ph = np.hypot(dx, dy) / F_EQ, np.arctan2(dy, dx)
        views.append((d[perm], xy))
        bears.append(np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], 1))
    return views, bears


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--max-iteration", type=int, default=50000)
    ap.add_argument("--cpu-sample", type=int, default=2)
    a = ap.parse_args()
    views, bears = fisheye_ring(a.views, a.features, np.random.default_rng(1))
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, a.views)]
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    put = m.Match({v: views[v] for v in range(a.views)}, pairs)
    m.clear()
    putatives = {p: {"sift": np.asarray(put[p]).copy()} for p in pairs if p in put}
    regions = {v: {"sift": matching.Regions(views[v][0], views[v][1])} for v in range(a.views)}
    sizes = {v: (W, H) for v in range(a.views)}
    bearings = {v: {"sift": bears[v]} for v in range(a.views)}

    t = time.perf_counter()
    out, info = matching.robustModelEstimation_F_AC(putatives, regions, sizes, 42, a.max_iteration, guidedMatching=True, ctx=ctx, bearings=bearings)
    stage_s = time.perf_counter() - t
    guided_ms = ctx.last_gpu_ms()
    k10 = ctx.acransac_last_stats()
    kept = [p for p in out if np.isfinite(info[p]["error_max"])]

    from oracle import acransac_s as acrs
    acrs.build(ref=False) if not acrs.available("port") else None
    O = acrs.AcransacSOracle("port")
    st = O.mt_seed(42)
    cpu = []
    for p in list(putatives)[: a.cpu_sample]:
        b = np.c_[bears[p[0]][putatives[p]["sift"]["i"]], bears[p[1]][putatives[p]["sift"]["j"]]]
        t = time.perf_counter()
        O.estimate(b, st, a.max_iteration)
        cpu.append(time.perf_counter() - t)
    print(json.dumps({
        "bench": "geometric_filter_F_AC_spherical_guided", "gpu": card(), "views": a.views, "features": a.features, "pairs": len(pairs),
        "putative_pairs": len(putatives), "putatives": int(sum(len(v["sift"]) for v in putatives.values())), "max_iteration": a.max_iteration,
        "spherical_pairs": int(sum(info[p]["spherical"] for p in putatives)), "valid_pairs": int(sum(info[p]["valid"] for p in putatives)),
        "kept_pairs": len(out), "guided_pairs": len(kept), "guided_matches": int(sum(len(x) for p in kept for x in out[p].values())),
        "stage_wall_s": round(stage_s, 3), "k10_gpu_ms": round(k10["gpu_ms"], 2), "k10_models_evaluated": k10["models_evaluated"],
        "k10_models_skipped": k10["models_skipped"], "k10_models_exact": k10["models_exact"], "guided_gpu_ms": round(guided_ms, 2),
        "port_oracle_s_per_pair": [round(x, 3) for x in cpu],
    }))
    ctx.close()


if __name__ == "__main__":
    main()
