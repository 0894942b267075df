"""The `homography_matrix` geometric filter with featureMatching's guided matching on the GPU (matching.robustModelEstimation_H_AC with
guidedMatching=True, distanceRatio=-1): K10 H over every putative pair, then one b200m_guided_match_positions_pairs call (position-only
guidedMatching + IndMatchDecorator) over the kept pairs.  Prints one JSON line.

Workload: --views views of --features SIFT uchar features at 4000 x 3000 on a rotation ring (a camera turning about its centre, as in
tools/gpu_acransac_bench.py --model H, so every overlapping pair is related by a homography), descriptors per 3-D direction with
per-view noise plus fresh features, exhaustive pairs, putatives from the engine (ImageCollectionMatcherB200, ratio 0.8), the H filter
at --max-iteration.  Reported: K10 GPU time, the position-guided call's GPU and kernel time, the stage's wall time, the share of
guided left views in general position (decorated on the device), and the port oracle's position-only guided matching per pair on one
CPU thread for a sample of pairs.

    python tools/gpu_homography_filter_bench.py [--views 100] [--features 8192] [--max-iteration 50000] [--cpu-sample 2]
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


def rotation_ring(n_views: int, m: int, rng):
    """n_views yaw angles over a full turn (f = 0.9 W: each view overlaps ~16 neighbours on either side); 70 % of each view's features
    are directions it sees (observed +- 0.5 px), the rest fresh."""
    f = 0.9 * W
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    fov = 2 * np.arctan(W / 2 / f)
    n_pts = int(0.7 * m * 2 * np.pi / fov * 1.3)
    az = rng.uniform(0, 2 * np.pi, n_pts)
    el = rng.uniform(-np.arctan(H / 2 / f), np.arctan(H / 2 / f), n_pts)
    D = np.stack([np.cos(el) * np.sin(az), np.sin(el), np.cos(el) * np.cos(az)], 1)
    base = synth.sift_images(1, n_pts, np.uint8, seed=5, pool_factor=1.0)[0][0]
    views = []
    for k in range(n_views):
        a = 2 * np.pi * k / n_views
        R = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        h = (D @ R.T) @ K.T
        x = h[:, :2] / h[:, 2:]
        vis = np.where((h[:, 2] > 0) & (x[:, 0] >= 0) & (x[:, 0] < W - 1) & (x[:, 1] >= 0) & (x[:, 1] < H - 1))[0]
        vis = rng.permutation(vis)[: int(0.7 * m)]
        xy = np.concatenate([x[vis] + rng.uniform(-0.5, 0.5, (len(vis), 2)),
                             np.stack([rng.uniform(0, W - 1, m - len(vis)), rng.uniform(0, H - 1, m - len(vis))], 1)])
        d = np.concatenate([np.clip(base[vis].astype(np.int32) + rng.integers(-5, 6, (len(vis), 128)), 0, 255).astype(np.uint8),
                            synth.sift_images(1, m - len(vis), np.uint8, seed=100 + k, pool_factor=1.0)[0][0]])
        perm = rng.permutation(m)
        views.append((d[perm], xy[perm].astype(np.float32)))
    return views


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--max-iteration", type=int, default=50000)
    ap.add_argument("--cpu-sample", type=int, default=2)
    a = ap.parse_args()
    views = rotation_ring(a.views, a.features, np.random.default_rng(1))
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, a.views)]
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    put = m.Match({v: views[v] for v in range(a.views)}, pairs)
    m.clear()
    putatives = {p: {"sift": np.asarray(put[p]).copy()} for p in pairs if p in put}
    regions = {v: {"sift": matching.Regions(views[v][0], views[v][1])} for v in range(a.views)}
    sizes = {v: (W, H) for v in range(a.views)}

    t = time.perf_counter()
    out, info = matching.robustModelEstimation_H_AC(putatives, regions, sizes, 42, a.max_iteration, guidedMatching=True, distanceRatio=-1.0, ctx=ctx)
    stage_s = time.perf_counter() - t
    guided_ms, guided_kernel_ms = ctx.last_gpu_ms(), ctx.last_search_kernel_ms()
    k10 = ctx.acransac_last_stats()
    kept = [p for p in out if np.isfinite(info[p]["error_max"])]

    def generic(v):
        xy = views[v][1]
        return len(np.unique(xy[:, 0])) == len(xy) and len(np.unique(xy[:, 1])) == len(xy)
    gen = {v: generic(v) for v in {p[0] for p in kept}}

    from oracle import guided_positions as gpo
    O = gpo.GuidedPositionsOracle()
    cpu = []
    for p in kept[: a.cpu_sample]:
        t = time.perf_counter()
        O.guided_match_positions(views[p[0]][1], views[p[1]][1], info[p]["H"], info[p]["error_max"] ** 2)
        cpu.append(time.perf_counter() - t)
    print(json.dumps({
        "bench": "geometric_filter_H_AC_guided_positions", "gpu": card(), "views": a.views, "features": a.features, "pairs": len(pairs),
        "putative_pairs": len(putatives), "putatives": int(sum(len(v["sift"]) for v in putatives.values())), "max_iteration": a.max_iteration,
        "valid_pairs": int(sum(info[p]["valid"] for p in putatives)), "kept_pairs": len(out), "guided_pairs": len(kept),
        "guided_matches": int(sum(len(x) for p in kept for x in out[p].values())),
        "stage_wall_s": round(stage_s, 3), "k10_gpu_ms": round(k10["gpu_ms"], 2), "guided_positions_gpu_ms": round(guided_ms, 2),
        "guided_positions_kernel_ms": round(guided_kernel_ms, 2),
        "left_views_decorated_on_device": round(sum(gen[p[0]] for p in kept) / max(len(kept), 1), 4),
        "port_oracle_s_per_pair": [round(x, 3) for x in cpu],
    }))
    ctx.close()


if __name__ == "__main__":
    main()
