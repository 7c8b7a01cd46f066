#!/usr/bin/env python
"""Streaming EnCodec (bark_b200_encodec_stream_*, bark_cpp_b200.Encodec.stream) on an H100: the cost of one push.

usage: python tools/codec_stream_bench.py [--pushes P] [--bandwidth KBPS] [--frames F ...] [--streams S ...]
                                          [--sample-rate HZ ...] [--channels C ...]
Codec of the synthetic tiny f16 file (every synthetic file carries the full-size 24 kHz codec), seeded noise and seeded codes:
  * cases: pushes of 1, 4 and 16 frames (320 samples a frame at 24 kHz), encode and decode, one stream and 32 streams in one push_batch;
  * formats (DESIGN.md §20): --sample-rate and --channels (paired lists, default 24000 and 1) give the streams' formats: an encode pushes
    a frame's worth of interleaved source frames (640 at 48 kHz, 588 at 44.1 kHz), a decode returns samples at the rate (mono).  Within
    each case the formats alternate, so they are measured side by side;
  * each case opens its streams, pushes 8 frames to each (past the 7 frames a stream waits for), then times P pushes;
  * per push: wall time (host clock around the call, which ends in a device synchronise), median / min / max; kernel launches; audio
    seconds per wall second (all streams); then, in a separate run of P pushes with the CUDA-event profiler on, the device time of the
    kernels per push;
  * every stream's output is checked bit for bit against the whole-clip call on its input.
Prints a table and writes $BARK_TOOLS_OUT/codec_stream_bench.json with the card's name, power limit and maximum SM clock.
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

SR, HOP, FRAME_MS = 24000, 320, 1e3 * 320 / 24000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def run_case(pkg, e, direction, frames, count, pushes, sr=SR, ch=1):
    """Times `pushes` pushes of `frames` frames to each of `count` streams at sr Hz and ch channels; returns the row and whether every
    stream's output equals the whole-clip call."""
    rng = np.random.Generator(np.random.PCG64(frames * 100 + count))
    total = 8 + 2 * pushes                               # frames: the lead-in, the timed pushes and the profiled ones
    plain = (sr, ch) == (SR, 1)
    streams = [e.stream(direction) if plain else e.stream(direction, sample_rate=sr, channels=ch if direction == "encode" else None) for _ in range(count)]
    n_q = streams[0].n_q
    if direction == "encode":
        F = HOP * sr // SR                               # source frames of one code frame
        shape = lambda n: (n,) if ch == 1 else (n, ch)   # noqa: E731
        inputs = [rng.uniform(-1, 1, shape(total * frames * F + 8 * F)).astype(np.float32) for _ in range(count)]
        chunk = lambda x, i: x[i * frames * F:(i + 1) * frames * F]
        lead = lambda x: x[:8 * F]
        rest = lambda x, i: x[i * frames * F:]
    else:
        inputs = [rng.integers(0, 1024, (n_q, total * frames + 8)).astype(np.int32) for _ in range(count)]
        chunk = lambda x, i: x[:, i * frames:(i + 1) * frames]
        lead = lambda x: x[:, :8]
        rest = lambda x, i: x[:, i * frames:]
    timed = [x[8 * F:] if direction == "encode" else x[:, 8:] for x in inputs]
    outs = [[] for _ in range(count)]

    def push(i):
        if count == 1:
            return [streams[0].push(chunk(timed[0], i))]
        return pkg.encodec_stream_push_batch(streams, [chunk(x, i) for x in timed])

    for s, x, o in zip(streams, inputs, outs):
        o.append(s.push(lead(x)))
    walls, launches = [], []
    for i in range(pushes):
        l0 = pkg.kernel_launches()
        t0 = time.perf_counter()
        got = push(i)
        walls.append(time.perf_counter() - t0)
        launches.append(pkg.kernel_launches() - l0)
        for o, g in zip(outs, got):
            o.append(g)
    pkg.profile_enable(True)
    for i in range(pushes, 2 * pushes):
        for o, g in zip(outs, push(i)):
            o.append(g)
    prof = pkg.profile_report()
    pkg.profile_enable(False)
    same = True
    for s, x, o in zip(streams, timed, outs):
        o.append(s.push(rest(x, 2 * pushes)))
        o.append(s.finish())
        s.close()
    for x, o in zip(inputs, outs):
        if direction == "encode":
            want = e.compress(x) if plain else e.compress(x if x.ndim == 1 else np.ascontiguousarray(x.T), sample_rate=sr)
            same &= bool(np.array_equal(np.concatenate(o, axis=1), want))
        else:
            want = e.decompress(x) if sr == SR else pkg.resample(e.decompress(x), SR, sr)
            same &= bool(np.array_equal(np.concatenate(o).view(np.uint32), want.view(np.uint32)))
    med = float(np.median(walls))
    return dict(direction=direction, sample_rate=sr, channels=ch if direction == "encode" else 1, frames_per_push=frames, streams=count, pushes=pushes,
                wall_ms_median=1e3 * med, wall_ms_min=1e3 * min(walls),
                wall_ms_max=1e3 * max(walls), device_ms_per_push=sum(v["ms"] for v in prof.values()) / pushes,
                launches_per_push=float(np.median(launches)), audio_s_per_s=count * frames * HOP / SR / med,
                frame_budget_ms=frames * FRAME_MS, bit_identical=same,
                top_kernels={k: v["ms"] / pushes for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[:6]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=60)
    ap.add_argument("--bandwidth", type=int, default=6)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4, 16], help="frames per push")
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 32], help="streams per push")
    ap.add_argument("--sample-rate", type=int, nargs="+", default=[SR], help="the streams' sample rates, alternated within each case")
    ap.add_argument("--channels", type=int, nargs="+", default=None, help="an encode's channels, one per sample rate (default 1)")
    a = ap.parse_args()
    chans = a.channels or [1] * len(a.sample_rate)
    if len(chans) != len(a.sample_rate):
        ap.error("--channels takes one count per --sample-rate")
    fmts = list(zip(a.sample_rate, chans))
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    from make_golden_encoder import codec_offset
    os.makedirs(OUT, exist_ok=True)
    res = dict(card=card(), pushes=a.pushes, bandwidth=a.bandwidth, runs=[])
    with tempfile.TemporaryDirectory() as d:
        path = weights.write_weights(os.path.join(d, "tiny_f16.bin"), weights.tiny(), 1234)
        with pkg.Encodec(path, codec_offset(path)) as e:
            e.bandwidth = a.bandwidth
            for sr, ch in fmts:                          # warm-up: modules loaded, scratch grown
                run_case(pkg, e, "encode", 1, 1, 5, sr, ch)
                run_case(pkg, e, "decode", 1, 32, 5, sr, ch)
            for direction in ("encode", "decode"):
                for count in a.streams:
                    for frames in a.frames:
                        for sr, ch in fmts:
                            res["runs"].append(run_case(pkg, e, direction, frames, count, a.pushes, sr, ch))
    print(f"card: {res['card']}   bandwidth {a.bandwidth} kbps, {a.pushes} timed pushes per case")
    print(f"{'dir':>6} {'format':>10} {'streams':>7} {'frames':>6} | {'wall ms med/min/max':>22} {'budget ms':>9} | {'device ms':>9} | {'launches':>8} | {'audio s/s':>9} | same")
    for r in res["runs"]:
        fmt = f"{r['sample_rate']}x{r['channels']}"
        print(f"{r['direction']:>6} {fmt:>10} {r['streams']:>7} {r['frames_per_push']:>6} | {r['wall_ms_median']:>6.2f} /{r['wall_ms_min']:>6.2f} /{r['wall_ms_max']:>6.2f} "
              f"{r['frame_budget_ms']:>9.1f} | {r['device_ms_per_push']:>9.2f} | {r['launches_per_push']:>8.0f} | {r['audio_s_per_s']:>9.1f} | {r['bit_identical']}")
    with open(os.path.join(OUT, "codec_stream_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(OUT, "codec_stream_bench.json"))


if __name__ == "__main__":
    main()
