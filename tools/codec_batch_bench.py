#!/usr/bin/env python
"""Batched EnCodec (bark_b200_encodec_*_batch, bark_cpp_b200.Encodec.*_batch) against single calls on an H100.

usage: python tools/codec_batch_bench.py [--reps R] [--bandwidth KBPS]
Codec of the synthetic tiny f16 file (every synthetic file carries the full-size 24 kHz codec), seeded noise:
  * workloads: B = 1, 8 and 32 clips of 1 s and of 10 s, and B = 8 and 32 clips of a seeded mix of 2 to 15 s;
  * compress and decompress (of the compress's codes): the batch call and the B single calls on the same context, alternated R times
    after one warm-up of each; wall time (host clock around work that ends in a device synchronise), median / min / max; audio
    seconds per wall second; every batch item is checked bit for bit against its single call;
  * in a separate run with the CUDA-event profiler on: device time of lstm_recur_kernel (and of all kernels) for one batch call and for
    the B single calls.
Prints a table and writes $BARK_TOOLS_OUT/codec_batch_bench.json with the card's name, power limit and maximum SM clock.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def workloads():
    rng = np.random.Generator(np.random.PCG64(2024))
    mix = [int(s * SR) for s in rng.uniform(2.0, 15.0, 32)]
    out = []
    for s in (1, 10):
        for B in (1, 8, 32):
            out.append((f"{B} x {s} s", [s * SR] * B))
    for B in (8, 32):
        out.append((f"{B} x 2-15 s", mix[:B]))
    return out


def stats(walls, seconds):
    med = float(np.median(walls))
    return dict(wall_ms_median=1e3 * med, wall_ms_min=1e3 * min(walls), wall_ms_max=1e3 * max(walls), audio_s_per_s=seconds / med)


def profiled(pkg, fn):
    pkg.profile_enable(True)
    fn()
    prof = pkg.profile_report()
    pkg.profile_enable(False)
    return dict(device_ms=sum(v["ms"] for v in prof.values()), lstm_recur_ms=prof.get("lstm_recur_kernel", {}).get("ms", 0.0),
                lstm_recur_launches=prof.get("lstm_recur_kernel", {}).get("launches", 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bandwidth", type=int, default=6)
    a = ap.parse_args()
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    from make_golden_encoder import codec_offset
    os.makedirs(OUT, exist_ok=True)
    res = dict(card=card(), reps=a.reps, bandwidth=a.bandwidth, runs=[])
    with tempfile.TemporaryDirectory() as d:
        path = weights.write_weights(os.path.join(d, "tiny_f16.bin"), weights.tiny(), 1234)
        with pkg.Encodec(path, codec_offset(path)) as e:
            e.bandwidth = a.bandwidth
            for k, (name, lens) in enumerate(workloads()):
                xs = [np.random.Generator(np.random.PCG64(1000 * k + i)).uniform(-1, 1, n).astype(np.float32) for i, n in enumerate(lens)]
                seconds = sum(lens) / SR
                codes = [e.compress(x) for x in xs]
                ops = {
                    "compress": (lambda: e.compress_batch(xs), lambda: [e.compress(x) for x in xs]),
                    "decompress": (lambda: e.decompress_batch(codes), lambda: [e.decompress(c) for c in codes]),
                }
                row = dict(workload=name, items=len(xs), audio_s=seconds)
                for op, (batch, single) in ops.items():
                    got, ref = batch(), single()                                  # warm-up of both, and the bit-for-bit check
                    same = all(np.array_equal(np.asarray(g).view(np.uint32), np.asarray(r).view(np.uint32)) for g, r in zip(got, ref))
                    wb, ws = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter(); batch(); wb.append(time.perf_counter() - t0)
                        t0 = time.perf_counter(); single(); ws.append(time.perf_counter() - t0)
                    row[op] = dict(bit_identical=bool(same), batch=stats(wb, seconds), single=stats(ws, seconds),
                                   speedup=float(np.median(ws) / np.median(wb)), batch_profile=profiled(pkg, batch),
                                   single_profile=profiled(pkg, single))
                res["runs"].append(row)
    print(f"card: {res['card']}   bandwidth {a.bandwidth} kbps, {a.reps} alternated reps")
    print(f"{'workload':>12} {'op':>10} | {'batch ms (med/min/max)':>24} {'s/s':>6} | {'singles ms (med/min/max)':>26} {'s/s':>6} | "
          f"{'x':>5} | {'lstm_recur ms batch / singles':>30} | same")
    for r in res["runs"]:
        for op in ("compress", "decompress"):
            o = r[op]
            b, s = o["batch"], o["single"]
            print(f"{r['workload']:>12} {op:>10} | {b['wall_ms_median']:>8.2f} /{b['wall_ms_min']:>7.2f} /{b['wall_ms_max']:>7.2f} {b['audio_s_per_s']:>6.0f} | "
                  f"{s['wall_ms_median']:>10.2f} /{s['wall_ms_min']:>7.2f} /{s['wall_ms_max']:>7.2f} {s['audio_s_per_s']:>6.0f} | {o['speedup']:>5.2f} | "
                  f"{o['batch_profile']['lstm_recur_ms']:>13.2f} / {o['single_profile']['lstm_recur_ms']:>13.2f} | {o['bit_identical']}")
    with open(os.path.join(OUT, "codec_batch_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(OUT, "codec_batch_bench.json"))


if __name__ == "__main__":
    main()
