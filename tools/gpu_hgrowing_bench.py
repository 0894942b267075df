"""Measure the homography-growing filter (K12) on engine putatives, and the oracle's single-threaded port on the CPU.

Workload: a multi-plane ring (synth.planar_views(ring=True)): 100 views x up to 8192 SIFT uchar features (about 6200 ring points each, seeing
a 12 % arc of the ring, plus unrelated ones), 3 planes, exhaustive pairs matched by ImageCollectionMatcherB200 (BRUTE_FORCE_L2, ratio
0.8), each list sorted by Lowe ratio as featureMatching does, then robustModelEstimation_HGrowing over the whole list.  Writes one JSON
line (to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--points", type=int, default=52000)
    ap.add_argument("--port-sample", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(_ROOT, "profiles", "h100_hgrowing_filter_bench.json"))
    a = ap.parse_args()
    from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth
    from alicevision_b200.matches_filtering import sortMatches_byDistanceRatio
    from oracle import hgrowing

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    descs, feats = synth.planar_views(a.views, a.points, planes=3, seed=41, visible=0.12, fresh=0.3, ring=True)
    descs = [d[:8192] for d in descs]
    feats = [f[:8192] for f in feats]
    pairs = synth.exhaustive_pairs(a.views)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200)
    got = m.Match({i: (descs[i], np.ascontiguousarray(feats[i][:, :2])) for i in range(a.views)}, pairs)
    putatives = {p: {"sift": sortMatches_byDistanceRatio(mm)} for p, mm in got.items() if len(mm)}
    views = {v: {"sift": feats[v]} for v in range(a.views)}
    ctx = matching.default_context()
    ctx.hgrowing_pairs([hgrowing.putative_features(feats[0], feats[1], putatives[(0, 1)]["sift"])])   # warm-up
    t0 = time.perf_counter()
    out, hs = matching.robustModelEstimation_HGrowing(putatives, views, ctx=ctx)
    wall = time.perf_counter() - t0
    st = ctx.hgrowing_last_stats()
    n_put = [len(p["sift"]) for p in putatives.values()]
    big = sorted(putatives, key=lambda p: -len(putatives[p]["sift"]))[:a.port_sample]
    ora = hgrowing.HGrowingOracle()
    port_s = []
    for p in big:
        f = hgrowing.putative_features(feats[p[0]], feats[p[1]], putatives[p]["sift"])
        t0 = time.perf_counter()
        w = ora.filter(f)
        port_s.append(time.perf_counter() - t0)
        assert np.array_equal(putatives[p]["sift"][w["inliers"]], out[p]["sift"])
    line = {"bench": "hgrowing_filter", "card": card, "views": a.views, "features_per_view": [min(len(f) for f in feats), max(len(f) for f in feats)], "pairs": len(pairs),
            "pairs_with_putatives": len(putatives), "putatives": int(sum(n_put)), "max_putatives": int(max(n_put)),
            "stage_wall_s": round(wall, 3), "gpu_ms": round(st["gpu_ms"], 1), "seeds_grown": st["seeds_grown"],
            "seeds_skipped": st["seeds_skipped"], "rounds": st["rounds"],
            "homographies": int(sum(len(v) for h in hs.values() for v in h.values())),
            "geometric_matches": int(sum(len(v) for o in out.values() for v in o.values())),
            "port_sample_putatives": [len(putatives[p]["sift"]) for p in big], "port_s_per_pair": [round(s, 3) for s in port_s]}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        fh.write(json.dumps(line) + "\n")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
