"""A-contrario RANSAC estimation (K10) on an exhaustive synthetic scene: ~100 views, every pair at maxIteration = 50000, next to
the oracle's host time on a sample of pairs (the oracle runs the reference loop around a restated kernel, so its time is indicative
only).  --model F (default): the fundamental matrix; --model H: the homography, on a rotation ring (a camera turning about its
centre, so overlapping views are related by a homography).  Prints one JSON line; --out also writes it to a file.

Putative-list sizes: views on a ring, each overlapping its 3 neighbours on either side (300-2000 putatives, 30-80 % inliers);
every other pair has 20-200 putatives and no inliers, as the ratio test leaves them in an exhaustive list.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import alicevision_b200 as av  # noqa: E402
from alicevision_b200 import matching  # noqa: E402
from oracle import acransac as acr_oracle  # noqa: E402
from oracle import acransac_h as acrh_oracle  # noqa: E402
from test_acransac import WH, two_view_scene  # noqa: E402
from test_acransac_h import h_scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--max-iteration", type=int, default=50000)
    ap.add_argument("--oracle-pairs", type=int, default=3)
    ap.add_argument("--model", choices=("F", "H"), default="F")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    H = a.model == "H"
    r = np.random.default_rng(7)
    corrs, overlap = [], []
    for i in range(a.views):
        for j in range(i + 1, a.views):
            d = min(j - i, a.views - (j - i))
            ov = d <= 3
            n = int(r.integers(300, 2000)) if ov else int(r.integers(20, 200))
            ratio = float(r.uniform(0.3, 0.8)) if ov else 0.0
            corrs.append(h_scene(n, ratio, len(corrs), kind="rotation") if H else two_view_scene(n, ratio, len(corrs)))
            overlap.append(ov)
    ctx = av.Context(0)
    st = matching.mt19937_state(5489)
    run = ctx.acransac_homography_pairs if H else ctx.acransac_fundamental_pairs
    run(corrs[:8], [WH] * 8, st, 1000)   # module load
    t0 = time.perf_counter()
    res = run(corrs, [WH] * len(corrs), st, a.max_iteration)
    wall = time.perf_counter() - t0
    s = ctx.acransac_last_stats()
    port = acrh_oracle.AcransacHOracle("port") if H else acr_oracle.AcransacOracle("port")
    host = []
    for k in [i for i, o in enumerate(overlap) if o][:1] + [i for i, o in enumerate(overlap) if not o][:max(a.oracle_pairs - 1, 0)]:
        t = time.perf_counter()
        port.estimate(corrs[k], WH, st, a.max_iteration)
        host.append(time.perf_counter() - t)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    line = {"workload": f"acransac_{a.model} exhaustive{' rotation ring' if H else ''} {a.views} views, {len(corrs)} pairs, maxIteration {a.max_iteration}",
            "gpu": gpu, "pairs": len(corrs), "putatives": int(sum(len(c) for c in corrs)), "valid_pairs": int(sum(x["valid"] for x in res)),
            "gpu_ms": round(s["gpu_ms"], 2), "wall_s": round(wall, 3), "pairs_per_s": round(len(corrs) / (s["gpu_ms"] / 1e3), 1),
            "models_evaluated": s["models_evaluated"], "models_per_s": round(s["models_evaluated"] / (s["gpu_ms"] / 1e3)),
            "skip_rate": round(s["models_skipped"] / max(s["models_evaluated"], 1), 4), "models_exact": s["models_exact"],
            "launches": s["launches"], "iterations": int(sum(x["iterations"] for x in res)),
            "oracle_host_s_per_pair_sample": [round(x, 3) for x in host]}
    print(json.dumps(line))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
