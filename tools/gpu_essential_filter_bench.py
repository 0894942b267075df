"""The `essential_matrix` geometric filter on the GPU (matching.robustModelEstimation_E_AC, then removePoorlyOverlappingImagePairs):
K10's 5-point policy over every putative pair of a calibrated scene.  Prints one JSON line.

Workload: the scene of tools/gpu_geometric_filter_bench.py (--views views of --features SIFT uchar features at 4000 x 3000 on an arc
around a synthetic point cloud, one shared pinhole K; the undistorted positions of the distorted views are passed as `geometry`),
exhaustive pairs, putatives from the engine (ImageCollectionMatcherB200, ratio 0.8), the E filter at --max-iteration without guided
matching.  Reported: the stage's wall time, K10's GPU time and model counts, valid / kept pairs and the pairs the overlap cut removes;
then the port oracle (one CPU thread) on the first --cpu-sample estimated pairs, and K10 on those same pairs alone.

    python tools/gpu_essential_filter_bench.py [--views 100] [--features 8192] [--max-iteration 50000] [--cpu-sample 2]
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

from alicevision_b200 import ImageCollectionMatcherB200, matching  # noqa: E402
from gpu_known_poses_bench import H, W, camera, card, scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--max-iteration", type=int, default=50000)
    ap.add_argument("--cpu-sample", type=int, default=2)
    a = ap.parse_args()
    gpu = card()
    rng = np.random.default_rng(1)
    _, views = scene(a.views, a.features, rng)
    K = camera(0, a.views, np.random.default_rng(0))[2]   # f = 0.9 W, centred principal point: the same for every view
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, a.views)]
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    put = m.Match({v: (views[v][0], views[v][1]) for v in range(a.views)}, pairs)
    m.clear()
    putatives = {p: {"sift": np.asarray(put[p]).copy()} for p in pairs if p in put}
    regions = {v: {"sift": matching.Regions(views[v][0], views[v][1])} for v in range(a.views)}
    geometry = {v: {"sift": views[v][2]} for v in range(a.views) if views[v][2] is not None}
    sizes = {v: (W, H) for v in range(a.views)}
    intr = {v: K for v in range(a.views)}

    t = time.perf_counter()
    out, info = matching.robustModelEstimation_E_AC(putatives, regions, sizes, intr, 42, a.max_iteration, geometry=geometry, ctx=ctx)
    stage_s = time.perf_counter() - t
    k10 = ctx.acransac_last_stats()
    kept = matching.removePoorlyOverlappingImagePairs(out, putatives)

    from oracle import acransac_e
    P = acransac_e.AcransacEOracle("port")
    st = matching.mt19937_state(42)
    sample = list(putatives)[: a.cpu_sample]
    pos = lambda v: geometry.get(v, {}).get("sift", views[v][1]).astype(np.float64)  # noqa: E731
    corrs = [np.concatenate([pos(p[0])[putatives[p]["sift"]["i"]], pos(p[1])[putatives[p]["sift"]["j"]]], 1) for p in sample]
    cpu = []
    for c in corrs:
        t = time.perf_counter()
        P.estimate(c, (K, K), (W, H), st, a.max_iteration)
        cpu.append(time.perf_counter() - t)
    ctx.acransac_essential_pairs(corrs, [(W, H, W, H)] * len(corrs), [np.concatenate([K.ravel(), K.ravel()])] * len(corrs), st, a.max_iteration)
    sample_k10 = ctx.acransac_last_stats()
    print(json.dumps({
        "bench": "geometric_filter_E_AC", "gpu": gpu, "views": a.views, "features": a.features, "pairs": len(pairs),
        "putative_pairs": len(putatives), "putatives": int(sum(len(v["sift"]) for v in putatives.values())), "max_iteration": a.max_iteration,
        "valid_pairs": int(sum(bool(info[p]["valid"]) for p in putatives)), "kept_pairs": len(out),
        "removed_by_overlap_cut": len(out) - len(kept), "stage_wall_s": round(stage_s, 3), "k10_gpu_ms": round(k10["gpu_ms"], 2),
        "models_evaluated": k10["models_evaluated"], "models_skipped": k10["models_skipped"], "models_exact": k10["models_exact"],
        "cpu_sample_pairs": len(sample), "port_oracle_one_thread_s_per_pair": [round(x, 3) for x in cpu],
        "k10_gpu_ms_cpu_sample_pairs": round(sample_k10["gpu_ms"], 2),
    }))
    ctx.close()


if __name__ == "__main__":
    main()
