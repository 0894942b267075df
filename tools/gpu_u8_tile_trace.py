"""Per-tile pipeline trace of the u8 search kernels (l2_tc.cuh, U8 and its norm-GEMM form NG) on the GPU: where one tile's cycles go.

Builds the library if needed, matches 20 x 8192 uchar SIFT images (190 pairs, every pair on the norm-GEMM kernel, or on the u8 kernel
under B200M_U8_NORM_GEMM=0) with
`Context.debug_trace` on, and prints one JSON line: the medians, in SM cycles, of what CTA 0 stamped per database tile t.
Each warpgroup runs the tiles of a work item as a pipeline: it issues the MMAs of tile t + 1, then waits for tile t's and runs
tile t's epilogue while tile t + 1's MMAs run.  The columns are
  period         start of tile t's step to the start of tile t + 1's
  wait           waiting for tile t + 1's operands to land (db_full; none on the last tile of an item)
  mma            tile t + 1's MMAs issued, then blocked until tile t's have completed (wgmma.wait_group 1)
  epilogue       tile t's MMAs complete -> its chunk minima folded (under tile t + 1's MMAs)
  producer_wait  the TMA producer waiting for a free ring slot
for each of the two consumer warpgroups, over the traced tiles after the first two work items, and the card's name and power limit
read in the same call.  There is no fallback: without a GPU the script fails.

  python tools/gpu_u8_tile_trace.py [--images 20] [--features 8192]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SKIP_TILES = 128      # the first two 64-tile work items: the ring fills, the clocks ramp


def gpu_info(index: int) -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True)
    name, plim, smax = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}


def medians(trace):
    import numpy as np
    out = {}
    for wg in (0, 1):
        s = trace[1 + wg]
        n = int(np.count_nonzero(s[:, 3]))              # tiles this warpgroup stamped
        if n <= SKIP_TILES + 1:
            raise SystemExit(f"only {n} traced tiles: the u8 kernel did not run or the workload is too small")
        t = s[SKIP_TILES:n]
        out[f"wg{wg}"] = {"tiles": n - SKIP_TILES - 1,
                          "period": float(np.median(t[1:, 0] - t[:-1, 0])), "wait": float(np.median(t[:-1, 1] - t[:-1, 0])),
                          "mma": float(np.median(t[:-1, 2] - t[:-1, 1])), "epilogue": float(np.median(t[:-1, 3] - t[:-1, 2]))}
    p = trace[0]
    n = int(np.count_nonzero(p[:, 1]))
    out["producer_wait"] = float(np.median(p[SKIP_TILES + 1:n, 0] - p[SKIP_TILES:n - 1, 1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=20)
    ap.add_argument("--features", type=int, default=8192)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: the tile trace is SM clock stamps and cannot be taken without one")
    from alicevision_b200 import build
    build.build_native()
    from alicevision_b200 import EMatcherType, ImageCollectionMatcherB200, matching, synth

    descs, xys = synth.sift_images(args.images, args.features, np.uint8, seed=synth.SEED_DATA, pool_factor=1.0)
    pairs = synth.exhaustive_pairs(args.images)
    ctx = matching.Context(args.device)
    m = ImageCollectionMatcherB200(0.8, False, EMatcherType.BRUTE_FORCE_L2_B200, ctx)
    m.upload({i: (descs[i], xys[i]) for i in range(args.images)})
    m.wait_uploads()
    for _ in range(3):                                   # warm: module load, clocks
        m.match_uploaded(pairs, matching.STAGE_FULL)
    ctx.debug_trace(True)
    m.match_uploaded(pairs, matching.STAGE_FULL)
    trace = ctx.debug_trace(True, read=True)
    ctx.debug_trace(False)
    if ctx.last_u8_tc_pairs() != len(pairs) or ctx.exactness_errors() != 0:
        raise SystemExit(f"u8 pairs {ctx.last_u8_tc_pairs()} of {len(pairs)}, exactness errors {ctx.exactness_errors()}")
    kernel = "l2_top2_tc_u8ng_kernel" if ctx.last_u8_norm_gemm_pairs() == len(pairs) else "l2_top2_tc_u8_kernel"
    out = {"workload": f"{args.images} x {args.features} uchar SIFT, {len(pairs)} pairs, CTA 0 of {kernel}", "unit": "SM cycles (median per tile)",
           "search_kernel_ms": ctx.last_search_kernel_ms(), "gpu": gpu_info(args.device)}
    out.update(medians(trace))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
