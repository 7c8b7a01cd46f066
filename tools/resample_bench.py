#!/usr/bin/env python
"""GPU resampling (bark_b200_resample, Encodec.compress_batch(..., sample_rate=...)) on an H100.

usage: python tools/resample_bench.py [--reps R] [--bandwidth KBPS]
  * kernel: device time of resample_kernel per audio second (CUDA-event profiler, one call per format after a warm-up) for 60 s of
    seeded noise at 16 kHz mono, 44.1 and 48 kHz stereo -> 24 kHz, and 24 kHz mono -> 48 kHz;
  * end to end: 32 x 10 s of 44.1 kHz stereo through compress_batch with sample_rate=44100, against a host conversion (torchaudio's
    convert order: channel mean, then torchaudio.functional.resample on the CPU) followed by compress_batch, alternated R times after a
    warm-up of each; wall time (host clock around work that ends in a device synchronise), median / min / max.  The host leg is
    skipped when torchaudio cannot be imported.
Codec of the synthetic tiny f16 file (every synthetic file carries the full-size 24 kHz codec).  Prints a table and writes
$BARK_TOOLS_OUT/resample_bench.json with the card's name, power limit and maximum SM clock.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def noise(seed, channels, n):
    return np.random.Generator(np.random.PCG64(seed)).uniform(-1, 1, (channels, n)).astype(np.float32)


def kernel_times(pkg):
    rows = []
    for sr, ch, nsr in ((16000, 1, 24000), (44100, 2, 24000), (48000, 2, 24000), (24000, 1, 48000)):
        x = noise(sr + ch, ch, 60 * sr)
        pkg.resample(x, sr, nsr)                                   # warm-up
        pkg.profile_enable(True)
        pkg.resample(x, sr, nsr)
        prof = pkg.profile_report()
        pkg.profile_enable(False)
        ms = prof["resample_kernel"]["ms"]
        rows.append(dict(fmt=f"{sr} Hz x {ch} -> {nsr} Hz", audio_s=60.0, kernel_ms=ms, us_per_audio_s=1e3 * ms / 60.0))
    return rows


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
    res = dict(card=card(), reps=a.reps, bandwidth=a.bandwidth, kernel=kernel_times(pkg))
    try:
        import torch
        import torchaudio.functional as taf
    except ImportError:
        taf = None
    clips = [noise(i, 2, 441000) for i in range(32)]
    with tempfile.TemporaryDirectory() as d:
        path = weights.write_weights(os.path.join(d, "tiny_f16.bin"), weights.tiny(), 1234)
        with pkg.Encodec(path, codec_offset(path)) as e:
            e.bandwidth = a.bandwidth
            gpu = lambda: e.compress_batch(clips, sample_rate=44100)                          # noqa: E731
            host = (lambda: e.compress_batch([taf.resample(torch.from_numpy(x).mean(dim=0), 44100, 24000).numpy() for x in clips])) if taf else None  # noqa: E731
            gpu()
            if host:
                host()
            wg, wh = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); gpu(); wg.append(time.perf_counter() - t0)
                if host:
                    t0 = time.perf_counter(); host(); wh.append(time.perf_counter() - t0)
    st = lambda w: dict(wall_ms_median=1e3 * float(np.median(w)), wall_ms_min=1e3 * min(w), wall_ms_max=1e3 * max(w), audio_s_per_s=320.0 / float(np.median(w)))  # noqa: E731
    res["batch_32x10s_44k1_stereo"] = dict(gpu_resample=st(wg), host_torchaudio=st(wh) if wh else "not measured: torchaudio is not importable")
    print(f"card: {res['card']}")
    for r in res["kernel"]:
        print(f"  resample_kernel {r['fmt']:>28}: {r['kernel_ms']:8.3f} ms for 60 s, {r['us_per_audio_s']:7.2f} us per audio second")
    b = res["batch_32x10s_44k1_stereo"]
    print(f"  32 x 10 s 44.1 kHz stereo, compress_batch at {a.bandwidth} kbps: GPU resample {b['gpu_resample']['wall_ms_median']:.1f} ms "
          f"(min {b['gpu_resample']['wall_ms_min']:.1f}, max {b['gpu_resample']['wall_ms_max']:.1f})", end="")
    print(f", host torchaudio then compress_batch {b['host_torchaudio']['wall_ms_median']:.1f} ms (min {b['host_torchaudio']['wall_ms_min']:.1f}, "
          f"max {b['host_torchaudio']['wall_ms_max']:.1f})" if wh else f", {b['host_torchaudio']}")
    with open(os.path.join(OUT, "resample_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(OUT, "resample_bench.json"))


if __name__ == "__main__":
    main()
