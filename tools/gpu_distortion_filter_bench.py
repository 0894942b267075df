"""The `fundamental_with_distortion` geometric filter on the GPU (matching.robustModelEstimation_F_AC with estimateDistortion=True):
K10's 10-point policy over every putative pair.  Prints one JSON line.

Workload: the scene of tools/gpu_essential_filter_bench.py (--views views of --features SIFT uchar features at 4000 x 3000 on an arc
around a synthetic point cloud), with every view's undistorted positions run through a division-model distortion (--lambda, in the
preconditioned units 1 / sqrt(w h)) and passed as the filter's positions; exhaustive pairs, putatives from the engine
(ImageCollectionMatcherB200, ratio 0.8), the filter at --max-iteration without guided matching.  Reported: the card, the stage's
wall time, K10's GPU time and model counts, valid / kept pairs; then the port oracle (one CPU thread) on the first --cpu-sample
estimated pairs, and K10 on those same pairs alone.

    python tools/gpu_distortion_filter_bench.py [--views 100] [--features 8192] [--max-iteration 50000] [--cpu-sample 2]
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
from gpu_known_poses_bench import H, W, card, scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--max-iteration", type=int, default=50000)
    ap.add_argument("--cpu-sample", type=int, default=2)
    ap.add_argument("--lambda", dest="lam", type=float, default=-0.2)
    a = ap.parse_args()
    gpu = card()
    try:   # the card's max SM clock, read in the same call as the measurement
        import subprocess
        gpu["max_sm_clock_mhz"] = float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0])
    except Exception:
        gpu["max_sm_clock_mhz"] = None
    rng = np.random.default_rng(1)
    _, views = scene(a.views, a.features, rng)
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, a.views)]
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    put = m.Match({v: (views[v][0], views[v][1]) for v in range(a.views)}, pairs)
    m.clear()
    putatives = {p: {"sift": np.asarray(put[p]).copy()} for p in pairs if p in put}
    regions = {v: {"sift": matching.Regions(views[v][0], views[v][1])} for v in range(a.views)}
    s, c0 = 1.0 / np.sqrt(W * H), np.array([W / 2, H / 2])

    def distort(u):   # division model: u - c = (d - c) / (1 + lam |s (d - c)|^2)
        du = (np.asarray(u, np.float64) - c0) * s
        d = du.copy()
        for _ in range(100):
            d = du * (1 + a.lam * np.sum(d * d, axis=1, keepdims=True))
        return d / s + c0
    geometry = {v: {"sift": distort(views[v][2] if views[v][2] is not None else views[v][1])} for v in range(a.views)}
    sizes = {v: (W, H) for v in range(a.views)}

    t = time.perf_counter()
    out, info = matching.robustModelEstimation_F_AC(putatives, regions, sizes, 42, a.max_iteration, geometry=geometry, ctx=ctx,
                                                    estimateDistortion=True)
    stage_s = time.perf_counter() - t
    k10 = ctx.acransac_last_stats()

    from oracle import acransac_f10
    P = acransac_f10.AcransacF10Oracle("port")
    st = matching.mt19937_state(42)
    sample = list(putatives)[: a.cpu_sample]
    pos = lambda v: geometry[v]["sift"]  # noqa: E731
    corrs = [np.concatenate([pos(p[0])[putatives[p]["sift"]["i"]], pos(p[1])[putatives[p]["sift"]["j"]]], 1) for p in sample]
    cpu = []
    for c in corrs:
        t = time.perf_counter()
        P.estimate(c, (W, H, W, H), st, a.max_iteration)
        cpu.append(time.perf_counter() - t)
    ctx.acransac_fundamental_distortion_pairs(corrs, [(W, H, W, H)] * len(corrs), st, a.max_iteration)
    sample_k10 = ctx.acransac_last_stats()
    print(json.dumps({
        "bench": "geometric_filter_F10_AC", "gpu": gpu, "lambda": a.lam, "views": a.views, "features": a.features, "pairs": len(pairs),
        "putative_pairs": len(putatives), "putatives": int(sum(len(v["sift"]) for v in putatives.values())), "max_iteration": a.max_iteration,
        "valid_pairs": int(sum(bool(info[p]["valid"]) for p in putatives)), "kept_pairs": len(out), "stage_wall_s": round(stage_s, 3), "k10_gpu_ms": round(k10["gpu_ms"], 2),
        "models_evaluated": k10["models_evaluated"], "models_skipped": k10["models_skipped"], "models_exact": k10["models_exact"],
        "cpu_sample_pairs": len(sample), "port_oracle_one_thread_s_per_pair": [round(x, 3) for x in cpu],
        "k10_gpu_ms_cpu_sample_pairs": round(sample_k10["gpu_ms"], 2),
    }))
    ctx.close()


if __name__ == "__main__":
    main()
