#!/usr/bin/env python
"""Device time of the parity path's multi-row attention kernel at the shapes bark-small runs, on an H100.

usage: python tools/attn_bench.py [--reps R]
Shapes (12 heads of 64): the fine model's non-causal pass (1024 queries x 1024 keys), the semantic prefill (257 causal rows) and a
coarse window prefill (90 causal rows after 710 cached positions).  Each shape goes through bark_b200_parity_attention 3 times to
warm up, then R times with the CUDA-event profiler on: the attention kernels' summed device time per call, for the path the library
picks ("auto") and for each path forced (the three-kernel path only where its score buffer allows the row count).  Also printed: the FP32 lane operations
the shape needs (2 N n_kv E FMAs for QK^T and P.V, 31 adds per score for the lane trees, ~20 per score for soft_max) over the FMA
pipe's rate (SMs x 128 lanes x the maximum SM clock), as a floor, and the share of it reached.  Writes
$BARK_TOOLS_OUT/attn_bench.json with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get("BARK_TOOLS_OUT", os.path.join(tempfile.gettempdir(), "bark_tools"))   # results stay out of the tree
sys.path.insert(0, ROOT)
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402

SHAPES = [   # name, N, n_kv, n_past, causal
    ("fine", 1024, 1024, 0, False),
    ("semantic_prefill", 257, 257, 0, True),
    ("coarse_window", 90, 800, 710, True),
]
E, H = 768, 12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise SystemExit("nvidia-smi failed: this tool measures on the GPU and has no CPU mode")
    name, power, clock = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return name, power, float(clock)


def sm_count():
    rt = ctypes.CDLL("libcudart.so.12")
    n = ctypes.c_int(0)
    if rt.cudaDeviceGetAttribute(ctypes.byref(n), 16, 0) != 0:      # cudaDevAttrMultiProcessorCount
        raise SystemExit("no CUDA device")
    return n.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    pkg = graft.load_package()
    name, power, clock_mhz = card()
    n_sm = sm_count()
    lane_rate = n_sm * 128 * clock_mhz * 1e6
    rng = np.random.default_rng(0)
    rows = []
    for label, N, n_kv, n_past, causal in SHAPES:
        q = rng.standard_normal((N, E), np.float32)
        k = rng.standard_normal((n_kv, E), np.float32)
        v = rng.standard_normal((n_kv, E), np.float32)
        scores = H * N * n_kv
        ops = 2.0 * N * n_kv * E + 31.0 * scores + 20.0 * scores
        floor_us = ops / lane_rate * 1e6
        tiled_ok = N <= 32 * (-(-n_sm // H) - 1)                # the three-kernel path's score buffer limit (include/bark_b200.h)
        for path in ("auto", "fused", "tiled") if tiled_ok else ("auto", "fused"):
            for _ in range(3):
                pkg.parity_attention(q, k, v, H, n_past=n_past, causal=causal, path=path)
            pkg.profile_enable(True)
            for _ in range(args.reps):
                pkg.parity_attention(q, k, v, H, n_past=n_past, causal=causal, path=path)
            rep = pkg.profile_report()
            pkg.profile_enable(False)
            attn = {k_: r for k_, r in rep.items() if "attn_" in k_}
            assert attn and all(r["launches"] == args.reps for r in attn.values()), rep
            us = sum(r["ms"] for r in attn.values()) * 1e3 / args.reps
            rows.append(dict(shape=label, path=path, N=N, n_kv=n_kv, n_past=n_past, causal=causal, kernels=sorted(attn), us_per_call=us,
                             lane_ops=ops, fma_floor_us=floor_us, share_of_floor=floor_us / us))
            print(f"{label:17s} {path:5s} N {N:4d} n_kv {n_kv:4d} {'causal' if causal else 'full  '}  {us:8.1f} us/call   FMA-pipe floor"
                  f" {floor_us:6.1f} us ({100 * floor_us / us:4.1f} %)  {'+'.join(sorted(attn))}")
    print(f"card: {name}, power limit {power} W, max SM clock {clock_mhz:.0f} MHz, {n_sm} SMs")
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "attn_bench.json"), "w") as f:
        json.dump(dict(card=name, power_limit_w=power, max_sm_clock_mhz=clock_mhz, n_sm=n_sm, reps=args.reps, shapes=rows), f, indent=1)


if __name__ == "__main__":
    main()
