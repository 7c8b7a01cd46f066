#!/usr/bin/env python
"""Batched generation against sequential generation on one context, on an H100.

usage: python tools/batch_bench.py [--reps R]
bark-small f16 weights of the bench (bench.weights_path), n_steps_text_encoder = 138, distinct prompts and seeds.  For B in 1, 2, 4, 8:
  * one bark_b200_generate_batch of B prompts, and B sequential generate calls (reseeded per prompt) on the same context, alternated
    R times after one warm-up of each: aggregate audio seconds per wall second (min / median / max over the R runs), the factor of the
    medians and its range over the R pairs, and the stage wall times of the median run;
  * the batched decode step on its own (bark_b200_gpt_step_batch, coarse model, B rows at n_kv ~ 640): us per step and launches per
    step, and the per-kernel device times of one step from the CUDA-event profiler in a separate run;
and B = 8 again with BARK_B200_MODE=fast.  Prints a table and writes $BARK_TOOLS_OUT/batch_bench.json with the card's name and power limit.
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

TEXTS = ["hello world", "the quick brown fox", "hello the world", "brown fox world", "world hello", "the fox", "quick hello fox", "the brown world"]
SEEDS = [0, 1, 2, 3, 4, 5, 6, 7]
N_STEPS = 138
SR = 24000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def generation(pkg, b, B, reps):
    def batch():
        a = b.generate_batch(TEXTS[:B], SEEDS[:B]); s, _ = b.stats()
        return sum(x.size for x in a), dict(semantic_ms=s.t_semantic_us / 1e3, coarse_ms=s.t_coarse_us / 1e3, fine_ms=s.t_fine_us / 1e3, eval_ms=s.t_eval_us / 1e3)

    def seq():
        n, st = 0, dict(semantic_ms=0.0, coarse_ms=0.0, fine_ms=0.0, eval_ms=0.0)
        for i in range(B):
            b.reseed(SEEDS[i]); n += b.generate(TEXTS[i]).size; s, _ = b.stats()
            for k, v in (("semantic_ms", s.t_semantic_us), ("coarse_ms", s.t_coarse_us), ("fine_ms", s.t_fine_us), ("eval_ms", s.t_eval_us)):
                st[k] += v / 1e3
        return n, st
    batch(); seq()                                                        # warm-up: every shape of the timed calls
    runs = {"batch": [], "seq": []}
    for _ in range(reps):                                                 # alternated, so drifts of a shared host hit both alike
        for name, f in (("batch", batch), ("seq", seq)):
            t0 = time.perf_counter(); n, st = f(); runs[name].append((n / SR / (time.perf_counter() - t0), st))
    out = dict(B=B, reps=reps)
    for name in ("batch", "seq"):
        rates = sorted(r for r, _ in runs[name])
        out[name] = dict(audio_s_per_s_min=rates[0], audio_s_per_s_median=float(np.median(rates)), audio_s_per_s_max=rates[-1],
                         stages=sorted(runs[name], key=lambda x: x[0])[len(rates) // 2][1])
    pairs = [b[0] / q[0] for b, q in zip(runs["batch"], runs["seq"])]
    out["speedup_median"] = out["batch"]["audio_s_per_s_median"] / out["seq"]["audio_s_per_s_median"]
    out["speedup_pairs_min"], out["speedup_pairs_max"] = min(pairs), max(pairs)
    return out


def show(label, g):
    b, q = g["batch"], g["seq"]
    print(f"{label}: batch {b['audio_s_per_s_median']:.2f} [{b['audio_s_per_s_min']:.2f}, {b['audio_s_per_s_max']:.2f}] audio s/s, sequential "
          f"{q['audio_s_per_s_median']:.2f} [{q['audio_s_per_s_min']:.2f}, {q['audio_s_per_s_max']:.2f}] -> x{g['speedup_median']:.3f} "
          f"(pairs {g['speedup_pairs_min']:.3f}..{g['speedup_pairs_max']:.3f}, {g['reps']} runs each)  "
          f"batch stages {json.dumps({k: round(v, 1) for k, v in b['stages'].items()})}  seq stages {json.dumps({k: round(v, 1) for k, v in q['stages'].items()})}",
          flush=True)


def step(pkg, b, B):
    rng = np.random.default_rng(B)
    slots, n_past = list(range(B)), []
    for sl in slots:
        prompt = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 360 + 3 * sl)]).astype(np.int32)
        n_past.append(b.gpt_eval_slot(1, sl, prompt, 0, False)[1])
    toks = [10001] * B
    for _ in range(5):
        _, n_past = b.gpt_step_batch(1, slots, toks, n_past)
    l0 = pkg.kernel_launches(); t0 = time.perf_counter(); n = 40
    for _ in range(n):
        _, n_past = b.gpt_step_batch(1, slots, toks, n_past)
    us = (time.perf_counter() - t0) / n * 1e6
    launches = (pkg.kernel_launches() - l0) / n
    pkg.profile_enable(True)
    for _ in range(10):
        _, n_past = b.gpt_step_batch(1, slots, toks, n_past)
    rep = pkg.profile_report(); pkg.profile_enable(False)
    kern = {k: round(v["ms"] * 1e3 / 10, 2) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}
    return dict(B=B, n_kv_mean=float(np.mean(n_past)), us_per_step=us, us_per_token=us / B, launches_per_step=launches, kernel_us_per_step=kern)


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    pkg = graft.load_package()
    path = bench.weights_path("small")
    res = dict(card=card(), weights="bark-small f16 (bench weights)", n_steps_text_encoder=N_STEPS, gen=[], step=[])
    print(f"card: {res['card']}", flush=True)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS) as b:
        for B in (1, 2, 4, 8):
            g = generation(pkg, b, B, reps); res["gen"].append(g)
            show(f"B={B}", g)
        for B in (1, 2, 4, 8):
            st = step(pkg, b, B); res["step"].append(st)
            top = ", ".join(f"{k} {v}" for k, v in list(st["kernel_us_per_step"].items())[:8])
            print(f"step B={B} n_kv~{st['n_kv_mean']:.0f}: {st['us_per_step']:.1f} us/step ({st['us_per_token']:.1f} us/token), "
                  f"{st['launches_per_step']:.0f} launches; profiled us/step: {top}", flush=True)
    os.environ["BARK_B200_MODE"] = "fast"
    with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS) as b:
        assert b.fast_mode
        g = generation(pkg, b, 8, reps); g["mode"] = "fast"; res["fast"] = g
        show("fast B=8", g)
    os.makedirs(OUT, exist_ok=True)
    json.dump(res, open(os.path.join(OUT, "batch_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
