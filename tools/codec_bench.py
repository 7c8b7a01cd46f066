#!/usr/bin/env python
"""encodec.cpp's API (include/encodec.h, bark_cpp_b200.Encodec) on an H100, per bandwidth.

usage: python tools/codec_bench.py [--reps R] [--ref-threads N]
Codec of the synthetic tiny f16 file (every synthetic file carries the full-size 24 kHz codec with 32 codebooks), seeded noise of 1, 10
and 30 s, at 2, 3, 6, 12 and 24 kbps (2, 4, 8, 16 and 32 codebooks):
  * wall time of compress, decompress (of the compress's codes) and reconstruct: host clock around the call, which ends in a device
    synchronise; median / min / max of R calls after one warm-up call per shape; audio seconds per wall second;
  * in a separate run with the CUDA-event profiler on: device time per kernel of one call, and the RVQ encode kernel's share;
  * where oracle/_ref/libbark_ref.so exists: the reference's CPU encodec_compress_audio and encodec_decompress_audio on the 1 and 10 s
    clips (its graph is capped at 80 000 nodes, about 13 s of audio), with --ref-threads threads.
Prints a table and writes $BARK_TOOLS_OUT/codec_bench.json with the card's name and power limit.
"""
import argparse
import ctypes as C
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
BANDWIDTHS = (2, 3, 6, 12, 24)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def timed(fn, reps):
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); walls.append(time.perf_counter() - t0)
    return walls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ref-threads", type=int, default=min(16, os.cpu_count() or 1))
    a = ap.parse_args()
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    from make_golden_encoder import codec_offset
    os.makedirs(OUT, exist_ok=True)
    res = dict(card=card(), reps=a.reps, runs=[])
    with tempfile.TemporaryDirectory() as d:
        path = weights.write_weights(os.path.join(d, "tiny_f16.bin"), weights.tiny(), 1234)
        off = codec_offset(path)
        clips = {s: np.random.Generator(np.random.PCG64(s)).uniform(-1, 1, s * SR).astype(np.float32) for s in SECONDS}
        with pkg.Encodec(path, off) as e:
            for bw in BANDWIDTHS:
                e.bandwidth = bw
                for s in SECONDS:
                    x = clips[s]
                    codes = e.compress(x); e.decompress(codes); e.reconstruct(x)          # warm-up: module load, scratch growth
                    row = dict(bandwidth=bw, n_q=int(codes.shape[0]), seconds=s)
                    for op, fn in (("compress", lambda: e.compress(x)), ("decompress", lambda: e.decompress(codes)),
                                   ("reconstruct", lambda: e.reconstruct(x))):
                        w = timed(fn, a.reps)
                        pkg.profile_enable(True)
                        fn()
                        prof = pkg.profile_report()
                        pkg.profile_enable(False)
                        row[op] = dict(wall_ms_median=1e3 * float(np.median(w)), wall_ms_min=1e3 * min(w), wall_ms_max=1e3 * max(w),
                                       audio_s_per_s=s / float(np.median(w)), device_ms=sum(v["ms"] for v in prof.values()),
                                       rvq_encode_ms=prof.get("rvq_encode_kernel", {}).get("ms", 0.0), kernels=prof)
                    res["runs"].append(row)
        orc = graft.load_oracle_bindings()
        if orc.have_ref():
            from make_golden_encoder import RefCodec
            ref = RefCodec(path)
            ref.L.encodec_decompress_audio.restype = C.c_bool
            ref.L.encodec_decompress_audio.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
            res["reference"] = dict(threads=a.ref_threads, runs=[])
            for bw in BANDWIDTHS:
                ref.L.encodec_set_target_bandwidth(ref.ctx, bw)
                for s in (1, 10):
                    x = np.ascontiguousarray(clips[s])
                    t0 = time.perf_counter(); assert ref.L.encodec_compress_audio(ref.ctx, x.ctypes.data, x.size, a.ref_threads)
                    tc = time.perf_counter() - t0
                    n = ref.L.encodec_get_codes_size(ref.ctx)
                    codes = np.ctypeslib.as_array(ref.L.encodec_get_codes(ref.ctx), shape=(n,)).copy()
                    t0 = time.perf_counter(); assert ref.L.encodec_decompress_audio(ref.ctx, codes.ctypes.data, codes.size, a.ref_threads)
                    td = time.perf_counter() - t0
                    res["reference"]["runs"].append(dict(bandwidth=bw, seconds=s, compress_ms=1e3 * tc, decompress_ms=1e3 * td))
    print(f"card: {res['card']}")
    print(f"{'kbps':>4} {'n_q':>3} {'clip':>5} | {'compress ms (med/min/max)':>26} {'s/s':>6} {'rvq ms':>7} | {'decompress ms':>14} {'s/s':>6} | "
          f"{'reconstruct ms':>15} {'s/s':>6}")
    for r in res["runs"]:
        c, dd, rc = r["compress"], r["decompress"], r["reconstruct"]
        print(f"{r['bandwidth']:>4} {r['n_q']:>3} {r['seconds']:>4}s | {c['wall_ms_median']:>8.2f} /{c['wall_ms_min']:>7.2f} /{c['wall_ms_max']:>7.2f} "
              f"{c['audio_s_per_s']:>6.0f} {c['rvq_encode_ms']:>7.3f} | {dd['wall_ms_median']:>14.2f} {dd['audio_s_per_s']:>6.0f} | "
              f"{rc['wall_ms_median']:>15.2f} {rc['audio_s_per_s']:>6.0f}")
    for r in res.get("reference", {}).get("runs", []):
        print(f"reference ({res['reference']['threads']} threads) {r['bandwidth']} kbps {r['seconds']} s: compress {r['compress_ms']:.0f} ms, "
              f"decompress {r['decompress_ms']:.0f} ms")
    with open(os.path.join(OUT, "codec_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(OUT, "codec_bench.json"))


if __name__ == "__main__":
    main()
