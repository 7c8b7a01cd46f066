#!/usr/bin/env python
"""What the top-k / top-p filter (DESIGN.md §14) costs, on an H100.

usage: python tools/sampling_bench.py [--reps R] [--launches L]
1. The bench clip: bark-small f16 weights of the bench (bench.weights_path), "hello world", seed 0, n_steps_text_encoder = 138 (the
   synthetic weights never emit EOS, so every setting runs 138 semantic steps).  Filters off, top_k 50, top_p 0.9 and both, on the
   semantic and coarse stages, alternated R times after one warm-up of each: e2e audio s/s and per-stage ms (min / median / max).
2. In a separate pass with the CUDA-event profiler on: device time per launch of filter_rows_kernel through
   bark_b200_sample_filtered_given_u, L launches per shape, at n = 10048 (a semantic row) and 1024 (a coarse window), one row with 1024
   threads and B = 8 rows with 256 threads (a batched step), for each setting.  The rows are seeded N(0, 3^2) logits.
Prints a table and writes $BARK_TOOLS_OUT/sampling_bench.json with the card's name and power limit read in the same call.
"""
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
os.environ.setdefault("BARK_B200_QUIET", "1")
import bench  # noqa: E402
import __graft_entry__ as graft  # noqa: E402

TEXT, SEED, N_STEPS, SR = "hello world", 0, 138, 24000
SETTINGS = {"off": (None, None), "top_k 50": (50, None), "top_p 0.9": (None, 0.9), "both": (50, 0.9)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def stats(rs, keys):
    out = {}
    for k in keys:
        v = sorted(r[k] for r in rs)
        out[k] = dict(min=v[0], median=float(np.median(v)), max=v[-1])
    return out


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    launches = int(sys.argv[sys.argv.index("--launches") + 1]) if "--launches" in sys.argv else 200
    pkg = graft.load_package()
    path = bench.weights_path("small")
    res = dict(card=card(), weights="bark-small f16 (bench weights)", n_steps_text_encoder=N_STEPS, text=TEXT, seed=SEED, reps=reps)
    print(f"card: {res['card']}", flush=True)
    with pkg.Bark(path, seed=SEED, n_steps_text_encoder=N_STEPS) as b:
        def one(k, p):
            for stage in ("semantic", "coarse"):
                b.set_sampling(stage, top_k=k, top_p=p)
            b.reseed(SEED)
            t0 = time.perf_counter()
            a = b.generate(TEXT)
            wall = time.perf_counter() - t0
            s, _ = b.stats()
            return dict(audio_s_per_s=a.size / SR / wall, audio_s=a.size / SR, eval_ms=s.t_eval_us / 1e3, semantic_ms=s.t_semantic_us / 1e3,
                        coarse_ms=s.t_coarse_us / 1e3, fine_ms=s.t_fine_us / 1e3, n_semantic=int(b.tokens(0).size))
        for kp in SETTINGS.values():
            one(*kp)                                                           # warm-up: every shape of the timed calls
        runs = {name: [] for name in SETTINGS}
        for _ in range(reps):                                                  # alternated, so drifts of a shared host hit all alike
            for name, kp in SETTINGS.items():
                runs[name].append(one(*kp))
    res["e2e"] = {}
    for name, rs in runs.items():
        out = stats(rs, ("audio_s_per_s", "eval_ms", "semantic_ms", "coarse_ms", "fine_ms"))
        out["audio_s"], out["n_semantic"] = rs[0]["audio_s"], rs[0]["n_semantic"]
        res["e2e"][name] = out
        print(f"{name:>10}: {out['audio_s']:.2f} s of audio ({out['n_semantic']} semantic ids), e2e {out['audio_s_per_s']['median']:.2f} "
              f"[{out['audio_s_per_s']['min']:.2f}, {out['audio_s_per_s']['max']:.2f}] audio s/s; median ms: semantic "
              f"{out['semantic_ms']['median']:.1f}, coarse {out['coarse_ms']['median']:.1f}, fine {out['fine_ms']['median']:.1f}, "
              f"eval {out['eval_ms']['median']:.1f}", flush=True)

    rng = np.random.default_rng(0)
    res["kernel_us"] = {}
    for n in (10048, 1024):
        for rows, threads in ((1, 1024), (8, 256)):
            x = (rng.standard_normal((rows, n)) * 3).astype(np.float32)
            u = rng.random(rows)
            for name, (k, p) in SETTINGS.items():
                if name == "off":
                    continue
                pkg.sample_filtered_given_u(x, 0.7, u, top_k=k, top_p=p, threads=threads)          # warm-up
                pkg.profile_enable(True)
                for _ in range(launches):
                    pkg.sample_filtered_given_u(x, 0.7, u, top_k=k, top_p=p, threads=threads)
                rep = pkg.profile_report()
                pkg.profile_enable(False)
                kname = f"filter_rows_kernel<{threads}>"
                e = rep[kname]
                s = rep[f"sample_rows_kernel<{threads}>"]
                us, us_s = 1e3 * e["ms"] / e["launches"], 1e3 * s["ms"] / s["launches"]
                res["kernel_us"][f"n={n} rows={rows} {name}"] = dict(filter_us=us, sampler_us=us_s, launches=e["launches"])
                print(f"filter_rows_kernel n={n:5d} rows={rows} threads={threads:4d} {name:>9}: {us:7.1f} us per launch "
                      f"(sample_rows_kernel {us_s:6.1f} us)", flush=True)
    os.makedirs(OUT, exist_ok=True)
    json.dump(res, open(os.path.join(OUT, "sampling_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
