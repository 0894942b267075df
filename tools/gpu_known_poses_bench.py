"""Guided matching from known poses on the GPU: b200m_guided_match_fast_pairs (guidedMatchingFundamentalFast for a pair list over
resident views) against the port oracle's CPU time per pair.  Prints one JSON line.

Workload: --views views of --features SIFT uchar features at 4000 x 3000 on an arc around a synthetic point cloud (known poses,
every second camera with radial distortion and its undistorted positions set as geometry), a frustum-like pair list of the
views within --reach of each other along the arc (about 1000 pairs for 60 views), errorTh = 4^2, distRatio = 0.8^2 as
StructureEstimationFromKnownPoses passes them.  The views are uploaded once; the timed calls run the whole list.

    python tools/gpu_known_poses_bench.py [--views 60] [--features 8192] [--reach 20] [--steps 5] [--warmup 1] [--cpu-sample 8]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from alicevision_b200 import ImageCollectionMatcherB200, matching, synth  # noqa: E402

W, H = 4000, 3000


def card() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")[:2]]
        return {"name": name, "power_limit_w": float(plim)}
    except Exception:
        return {"name": None, "power_limit_w": None}


def camera(k, n_views, rng):
    """Camera k on an arc of radius 12 around the cloud, looking at its centre: (P, centre, K, k1)."""
    a = -0.9 + 1.8 * k / max(n_views - 1, 1)
    C = np.array([12 * np.sin(a), rng.uniform(-0.5, 0.5), 10 - 12 * np.cos(a)])
    z = np.array([0, 0, 10.0]) - C; z /= np.linalg.norm(z)
    x = np.cross([0, 1, 0], z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    f = 0.9 * W
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    return K @ np.concatenate([R, -(R @ C)[:, None]], 1), C, K, -0.05 * (k % 2)


def fundamental(PL, CL, PR):
    """F_from_P (numeric/projection.cpp:115-143) and epipole_from_P (StructureEstimationFromKnownPoses.cpp:29-35)."""
    rows = lambda P: [P[[1, 2]], P[[2, 0]], P[[0, 1]]]
    X, Y = rows(PL), rows(PR)
    F = np.array([[np.linalg.det(np.concatenate([X[c], Y[r]])) for c in range(3)] for r in range(3)])
    return F, PR @ np.append(CL, 1.0)


def scene(n_views, m, rng):
    n_pts = 6 * m
    X = np.stack([rng.uniform(-5, 5, n_pts), rng.uniform(-3.5, 3.5, n_pts), rng.uniform(7, 13, n_pts)], 1)
    base = synth.sift_images(1, n_pts, np.uint8, seed=5, pool_factor=1.0)[0][0]
    cams, views = [], []
    for k in range(n_views):
        P, C, K, k1 = camera(k, n_views, rng)
        h = np.concatenate([X, np.ones((n_pts, 1))], 1) @ P.T
        x = h[:, :2] / h[:, 2:]
        vis = np.where((h[:, 2] > 0) & (x[:, 0] >= 0) & (x[:, 0] < W - 1) & (x[:, 1] >= 0) & (x[:, 1] < H - 1))[0]
        vis = rng.permutation(vis)[: int(0.7 * m)]
        und = np.concatenate([x[vis] + rng.uniform(-0.7, 0.7, (len(vis), 2)),
                              np.stack([rng.uniform(0, W - 1, m - len(vis)), rng.uniform(0, H - 1, m - len(vis))], 1)])
        d = np.concatenate([np.clip(base[vis].astype(np.int32) + rng.integers(-5, 6, (len(vis), 128)), 0, 255).astype(np.uint8),
                            synth.sift_images(1, m - len(vis), np.uint8, seed=100 + k, pool_factor=1.0)[0][0]])
        c = K[:2, 2]; dn = (und - c) / K[0, 0]
        obs = c + dn * (1 + k1 * (dn * dn).sum(1, keepdims=True)) * K[0, 0]
        cams.append((P, C)); views.append((d, obs.astype(np.float32), und if k1 else None))
    return cams, views


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=60)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--reach", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cpu-sample", type=int, default=8)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    cams, views = scene(a.views, a.features, rng)
    pairs = [(i, j) for i in range(a.views) for j in range(i + 1, min(a.views, i + a.reach + 1))]
    Fs, eps = zip(*[fundamental(cams[i][0], cams[i][1], cams[j][0]) for i, j in pairs])
    wh = [(W, H)] * len(pairs)
    th, ratio = 4.0 ** 2, 0.8 ** 2

    ctx = matching.Context(0)
    up = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    t0 = time.perf_counter()
    up.upload({v: (views[v][0], views[v][1]) for v in range(a.views)})
    for v in range(a.views):
        if views[v][2] is not None:
            ctx.set_view_geometry(v, views[v][2])
    up.wait_uploads()
    t_upload = time.perf_counter() - t0

    for _ in range(a.warmup):
        ctx.guided_match_fast_pairs(pairs, Fs, eps, wh, th, ratio)
    times, gpu_ms = [], []
    for _ in range(a.steps):
        t = time.perf_counter()
        res = ctx.guided_match_fast_pairs(pairs, Fs, eps, wh, th, ratio)     # synchronous: returns with the results on the host
        times.append(time.perf_counter() - t)
        gpu_ms.append(ctx.last_gpu_ms())
    cands, kernel_ms, launches = ctx.last_records(), ctx.last_search_kernel_ms(), ctx.last_launches()
    n_matches = sum(len(v) for v in res.values())

    # CPU: the port oracle (guidedMatchingFundamentalFast restated, one thread) on a sample of the same pairs
    from oracle import guided_fast as gfo
    P = gfo.GuidedFastOracle("port")
    sample = [pairs[k] for k in np.linspace(0, len(pairs) - 1, a.cpu_sample).astype(int)]
    pos = lambda v: views[v][2] if views[v][2] is not None else views[v][1].astype(np.float64)
    t = time.perf_counter()
    for (i, j) in sample:
        k = pairs.index((i, j))
        P.guided_fast(views[i][0], pos(i), views[j][0], pos(j), Fs[k], eps[k], W, H, th, ratio)
    cpu_s_per_pair = (time.perf_counter() - t) / len(sample)

    med = float(np.median(times))
    print(json.dumps({
        "workload": {"views": a.views, "features": a.features, "image": [W, H], "pairs": len(pairs), "errorTh": th, "distRatio": ratio,
                     "geometry_views": sum(1 for v in views if v[2] is not None)},
        "gpu": {"pairs_per_s": len(pairs) / med, "call_s_median": med, "call_s": times, "gpu_ms": gpu_ms, "candidate_kernel_ms": kernel_ms,
                "launches": launches, "upload_s": t_upload},
        "candidates": int(cands), "matches": int(n_matches),
        "cpu_port_oracle": {"s_per_pair": cpu_s_per_pair, "threads": 1, "sample_pairs": len(sample)},
        "speedup_vs_one_cpu_thread": cpu_s_per_pair * len(pairs) / med,
        "card": card(),
    }))
    ctx.close()


if __name__ == "__main__":
    main()
