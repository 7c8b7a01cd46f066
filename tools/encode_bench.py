#!/usr/bin/env python
"""EnCodec encoding (bark_b200_encodec_encode) on an H100.

usage: python tools/encode_bench.py [--reps R] [--ref-threads N]
Codec of the synthetic tiny f16 file (every synthetic file carries the full-size 24 kHz codec), seeded noise of 1, 10 and 30 s:
  * wall time of one encode call (host clock around the call, which ends in a device synchronise), median / min / max of R calls after
    one warm-up call per length; audio seconds per wall second;
  * in a separate run with the CUDA-event profiler on: device time per kernel of one call and their sum, with the algorithmic FLOPs
    of the encoder computed from the layer shapes (the profiler's own work column counts the same shapes per launch);
  * where oracle/_ref/libbark_ref.so exists: the reference's CPU encodec_compress_audio on the 1 and 10 s clips (its graph unrolls the
    LSTM and is capped at 80 000 nodes, about 13 s of audio), with --ref-threads threads.
Prints a table and writes $BARK_TOOLS_OUT/encode_bench.json with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get("BARK_TOOLS_OUT", os.path.join(tempfile.gettempdir(), "bark_tools"))   # results stay out of the tree
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402

SR = 24000
SECONDS = (1, 10, 30)
RATIOS = (2, 4, 5, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def encoder_flops(n: int) -> dict:
    """2 * outputs * contraction for every conv, the LSTM's 2 layers x (input + recurrent) mat-vecs, the RVQ's 8 x 1024 dots."""
    f = {"conv": 2.0 * n * 32 * 7, "lstm": 0.0, "rvq": 0.0}
    L, C = n, 32
    for r in RATIOS:
        f["conv"] += 2.0 * L * (C * C + (C // 2) * 3 * C + C * (C // 2))   # shortcut k1, conv_1 k3, conv_2 k1
        L = (L + r - 1) // r
        f["conv"] += 2.0 * L * (2 * C) * (C * 2 * r)                         # down-sampling k 2r, stride r
        C *= 2
    T = L
    f["lstm"] = 2 * 2 * (2.0 * T * 4 * 512 * 512)
    f["conv"] += 2.0 * T * 128 * 512 * 7
    f["rvq"] = 2.0 * T * 8 * 1024 * 128
    f["total"] = sum(f.values())
    f["T"] = T
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ref-threads", type=int, default=min(16, os.cpu_count() or 1))
    a = ap.parse_args()
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    os.makedirs(OUT, exist_ok=True)
    res = dict(card=card(), reps=a.reps, lengths=[])
    with tempfile.TemporaryDirectory() as d:
        path = weights.write_weights(os.path.join(d, "tiny_f16.bin"), weights.tiny(), 1234)
        clips = {s: np.random.Generator(np.random.PCG64(s)).uniform(-1, 1, s * SR).astype(np.float32) for s in SECONDS}
        with pkg.Bark(path, seed=0) as b:
            for s in SECONDS:
                b.encodec_encode(clips[s])                                   # warm-up: module load, scratch growth
            for s in SECONDS:
                x = clips[s]
                walls = []
                for _ in range(a.reps):
                    t0 = time.perf_counter(); b.encodec_encode(x); walls.append(time.perf_counter() - t0)
                pkg.profile_enable(True)
                b.encodec_encode(x)
                prof = pkg.profile_report()
                pkg.profile_enable(False)
                fl = encoder_flops(x.size)
                dev_ms = sum(v["ms"] for v in prof.values())
                res["lengths"].append(dict(
                    seconds=s, samples=int(x.size), frames=fl["T"], wall_ms_median=1e3 * float(np.median(walls)), wall_ms_min=1e3 * min(walls),
                    wall_ms_max=1e3 * max(walls), audio_s_per_s=s / float(np.median(walls)), device_ms=dev_ms, flops=fl,
                    achieved_tflops=fl["total"] / (dev_ms * 1e-3) / 1e12, kernels=prof))
        orc = graft.load_oracle_bindings()
        if orc.have_ref():
            from make_golden_encoder import RefCodec
            ref = RefCodec(path)
            res["reference"] = dict(threads=a.ref_threads, lengths=[])
            for s in (1, 10):
                ref.compress(clips[s][:SR], a.ref_threads)
                t0 = time.perf_counter(); ref.compress(clips[s], a.ref_threads); dt = time.perf_counter() - t0
                res["reference"]["lengths"].append(dict(seconds=s, wall_ms=1e3 * dt, audio_s_per_s=s / dt))
    print(f"card: {res['card']}")
    print(f"{'clip':>6} {'frames':>7} {'wall ms (med/min/max)':>24} {'audio s/s':>10} {'device ms':>10} {'GFLOP':>7} {'TFLOP/s':>8}")
    for r in res["lengths"]:
        print(f"{r['seconds']:>5}s {r['frames']:>7} {r['wall_ms_median']:>9.2f} /{r['wall_ms_min']:>6.2f} /{r['wall_ms_max']:>6.2f} "
              f"{r['audio_s_per_s']:>10.0f} {r['device_ms']:>10.2f} {r['flops']['total'] / 1e9:>7.2f} {r['achieved_tflops']:>8.2f}")
        top = sorted(r["kernels"].items(), key=lambda kv: -kv[1]["ms"])[:6]
        print("        " + ", ".join(f"{k} {v['ms']:.2f} ms ({v['launches']})" for k, v in top))
    for r in res.get("reference", {}).get("lengths", []):
        print(f"reference encodec_compress_audio ({res['reference']['threads']} threads) {r['seconds']} s: {r['wall_ms']:.0f} ms, {r['audio_s_per_s']:.1f} audio s/s")
    with open(os.path.join(OUT, "encode_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(OUT, "encode_bench.json"))


if __name__ == "__main__":
    main()
