#!/usr/bin/env python
"""Device time of the parity path's tiled GEMM (lane_gemm_tiled_kernel) at every multi-row shape of the bark-small bench clip, on an H100.

usage: python tools/gemm_bench.py [--reps R]
Shapes (E = 768): the fine model's 1024-row passes (QKV 768 -> 2304, c_proj 768 -> 768, fc 768 -> 3072, proj 3072 -> 768, lm_head
768 -> 1056) and the per-layer mat-muls of the semantic prefill (513 rows) and the coarse-window prefills (257 rows, then 60-91; 91 here).
Each shape goes through bark_b200_parity_gemm (f16 operands, STORE epilogue) 2 times to warm up, then R times with the CUDA-event
profiler on: the GEMM kernel's device time per call, for the block tile the library picks ("auto") and for each variant forced (all must give the same bits).  Also
printed: the FMA-pipe floor 2 M N K / (SMs x 128 lanes x 2 x the maximum SM clock) and the share of it reached.  Writes
$BARK_TOOLS_OUT/gemm_bench.json with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get("BARK_TOOLS_OUT", os.path.join(tempfile.gettempdir(), "bark_tools"))   # results stay out of the tree
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402
from attn_bench import card, sm_count  # noqa: E402

E = 768
LAYER = [("qkv", 3 * E, E), ("c_proj", E, E), ("fc", 4 * E, E), ("proj", E, 4 * E)]      # name, N, K
SHAPES = [("fine", 1024, n, N, K) for n, N, K in LAYER + [("lm_head", 1056, E)]] + \
         [(pre, M, n, N, K) for pre, M in (("semantic_prefill", 513), ("coarse_prefill", 257), ("coarse_window", 91)) for n, N, K in LAYER]
VARIANTS = (0, 1, 2)     # 0 = as the library picks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    pkg = graft.load_package()
    name, power, clock_mhz = card()
    n_sm = sm_count()
    fma_rate = n_sm * 128 * 2 * clock_mhz * 1e6                   # flop/s of the FP32 FMA pipe at the maximum SM clock
    rng = np.random.default_rng(0)
    rows = []
    for stage, M, label, N, K in SHAPES:
        A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
        W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
        flop = 2.0 * M * N * K
        floor_us = flop / fma_rate * 1e6
        ref = None
        for variant in VARIANTS:
            for _ in range(2):
                out, ran = pkg.parity_gemm(A, W, variant=variant, return_variant=True)
            if ref is None:
                ref = out
            assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), f"{stage} {label}: variant {variant} gives other bits"
            pkg.profile_enable(True)
            for _ in range(args.reps):
                pkg.parity_gemm(A, W, variant=variant)
            rep = pkg.profile_report()
            pkg.profile_enable(False)
            gemm = {k: r for k, r in rep.items() if "lane_gemm_tiled_kernel" in k}
            assert len(gemm) == 1 and all(r["launches"] == args.reps for r in gemm.values()), rep
            us = sum(r["ms"] for r in gemm.values()) * 1e3 / args.reps
            rows.append(dict(stage=stage, matrix=label, M=M, N=N, K=K, variant="auto" if variant == 0 else variant, ran=ran, us_per_call=us,
                             tflops=flop / us / 1e6, fma_floor_us=floor_us, share_of_floor=floor_us / us))
            print(f"{stage:16s} {label:7s} {M:4d} x {N:4d} x {K:4d}  variant {'auto' if variant == 0 else variant:>4} (ran {ran})  {us:8.1f} us/call"
                  f"  {flop / us / 1e6:5.1f} TFLOP/s  FMA-pipe floor {floor_us:6.1f} us ({100 * floor_us / us:4.1f} %)")
    print(f"card: {name}, power limit {power} W, max SM clock {clock_mhz:.0f} MHz, {n_sm} SMs")
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "gemm_bench.json"), "w") as f:
        json.dump(dict(card=name, power_limit_w=power, max_sm_clock_mhz=clock_mhz, n_sm=n_sm, reps=args.reps, shapes=rows), f, indent=1)


if __name__ == "__main__":
    main()
