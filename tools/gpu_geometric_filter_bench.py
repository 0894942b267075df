"""The `fundamental_matrix` geometric filter with guided matching on the GPU (matching.robustModelEstimation_F_AC): K10 over every
putative pair, then b200m_guided_match_pairs over the kept pairs.  Prints one JSON line.

Workload: --views views of --features SIFT uchar features at 4000 x 3000 on an arc around a synthetic point cloud (the scene of
tools/gpu_known_poses_bench.py), exhaustive pairs, putatives from the engine (ImageCollectionMatcherB200, ratio 0.8), the F filter
at --max-iteration with guided matching (distRatio 0.6^2, errorTh = error_max^2 per pair).  Reported: K10 GPU time, the batched
guided call's GPU time and the stage's wall time; then, on resident views, the same kept pairs through one batched call and through
a loop of one-pair b200m_guided_match calls (what a per-pair caller does), and the port oracle's guided matching on a sample of pairs.

    python tools/gpu_geometric_filter_bench.py [--views 100] [--features 8192] [--max-iteration 50000] [--steps 3] [--cpu-sample 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
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
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=2)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    _, views = scene(a.views, a.features, rng)
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, a.views)]
    ctx = matching.Context(0)
    m = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    put = m.Match({v: (views[v][0], views[v][1]) for v in range(a.views)}, pairs)
    m.clear()
    putatives = {p: {"sift": np.asarray(put[p]).copy()} for p in pairs if p in put}
    regions = {v: {"sift": matching.Regions(views[v][0], views[v][1])} for v in range(a.views)}
    sizes = {v: (W, H) for v in range(a.views)}

    t = time.perf_counter()
    out, info = matching.robustModelEstimation_F_AC(putatives, regions, sizes, 42, a.max_iteration, guidedMatching=True, ctx=ctx)
    stage_s = time.perf_counter() - t
    guided_ms, guided_kernel_ms = ctx.last_gpu_ms(), ctx.last_search_kernel_ms()
    k10 = ctx.acransac_last_stats()
    kept = [p for p in out if np.isfinite(info[p]["error_max"])]

    # the kept pairs on resident views: one batched call against a loop of one-pair calls
    for v in range(a.views):
        matching._upload_pair(ctx, [v], [regions[v]["sift"]], [None], [])
    Fs = [info[p]["F"] for p in kept]
    ths = [info[p]["error_max"] ** 2 for p in kept]
    ratio = 0.6 ** 2
    batched = ctx.guided_match_pairs(kept, Fs, ths, ratio)                 # warm-up
    t_batch, t_loop = [], []
    for _ in range(a.steps):
        t = time.perf_counter()
        batched = ctx.guided_match_pairs(kept, Fs, ths, ratio)
        t_batch.append(time.perf_counter() - t)
        t = time.perf_counter()
        loop = []
        for p, F, th in zip(kept, Fs, ths):
            res = C.c_void_p()
            matching._check(ctx.lib.b200m_guided_match(ctx._h, C.c_uint32(p[0]), C.c_uint32(p[1]), np.ascontiguousarray(F).ctypes.data_as(C.c_void_p),
                                                       C.c_double(th), C.c_double(ratio), C.byref(res)), "b200m_guided_match")
            off = C.c_void_p()
            matching._check(ctx.lib.b200m_result_get(res, None, C.byref(off), None), "b200m_result_get")
            loop.append(C.cast(off, C.POINTER(C.c_int64))[1])
            ctx.lib.b200m_result_free(res)
        t_loop.append(time.perf_counter() - t)
    assert loop == [len(b) for b in batched]

    from oracle import guided_fast as gfo
    P = gfo.GuidedFastOracle("port")
    cpu = []
    for p, F, th in list(zip(kept, Fs, ths))[: a.cpu_sample]:
        t = time.perf_counter()
        P.guided_match(views[p[0]][0], views[p[0]][1].astype(np.float64), views[p[1]][0], views[p[1]][1].astype(np.float64), F, th, ratio)
        cpu.append(time.perf_counter() - t)
    print(json.dumps({
        "bench": "geometric_filter_F_AC_guided", "gpu": card(), "views": a.views, "features": a.features, "pairs": len(pairs),
        "putative_pairs": len(putatives), "putatives": int(sum(len(v["sift"]) for v in putatives.values())), "max_iteration": a.max_iteration,
        "kept_pairs": len(out), "guided_pairs": len(kept), "guided_matches": int(sum(len(b) for b in batched)),
        "stage_wall_s": round(stage_s, 3), "k10_gpu_ms": round(k10["gpu_ms"], 2), "guided_gpu_ms": round(guided_ms, 2),
        "guided_kernel_ms": round(guided_kernel_ms, 2),
        "resident_batched_call_ms": [round(1e3 * x, 2) for x in t_batch], "resident_one_pair_loop_ms": [round(1e3 * x, 2) for x in t_loop],
        "port_oracle_s_per_pair": [round(x, 3) for x in cpu],
    }))
    ctx.close()


if __name__ == "__main__":
    main()
