#!/usr/bin/env python
"""What a speaker history prompt costs, on an H100.

usage: python tools/prompt_bench.py [--reps R]
bark-small f16 weights of the bench (bench.weights_path), n_steps_text_encoder = 138.  The prompt is the ids of a 138-step
generation of another text (Bark.last_generation_prompt).  "hello world" with seed 0, unprompted and prompted, alternated R times
after one warm-up of each: per-stage ms and end-to-end audio seconds per wall second (min / median / max over the R runs).  Prints
a table and writes $BARK_TOOLS_OUT/prompt_bench.json with the card's name and power limit read in the same call.
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

TEXT, SEED, PROMPT_TEXT, PROMPT_SEED = "hello world", 0, "the quick brown fox jumps over the lazy dog", 1
N_STEPS = 138
SR = 24000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    pkg = graft.load_package()
    path = bench.weights_path("small")
    res = dict(card=card(), weights="bark-small f16 (bench weights)", n_steps_text_encoder=N_STEPS, text=TEXT, seed=SEED, reps=reps)
    print(f"card: {res['card']}", flush=True)
    with pkg.Bark(path, seed=PROMPT_SEED, n_steps_text_encoder=N_STEPS) as b:
        b.generate(PROMPT_TEXT)
        prompt = b.last_generation_prompt()
    res["prompt"] = dict(n_semantic=int(prompt["semantic_prompt"].size), n_coarse_frames=int(prompt["coarse_prompt"].shape[1]),
                         n_fine_frames=int(prompt["fine_prompt"].shape[1]))
    print(f"prompt: {res['prompt']}", flush=True)
    with pkg.Bark(path, seed=SEED, n_steps_text_encoder=N_STEPS) as b:
        def one(p):
            b.reseed(SEED)
            t0 = time.perf_counter()
            a = b.generate(TEXT, history_prompt=p)
            wall = time.perf_counter() - t0
            s, _ = b.stats()
            return dict(audio_s_per_s=a.size / SR / wall, audio_s=a.size / SR, eval_ms=s.t_eval_us / 1e3, semantic_ms=s.t_semantic_us / 1e3,
                        coarse_ms=s.t_coarse_us / 1e3, fine_ms=s.t_fine_us / 1e3, n_semantic=int(b.tokens(0).size))
        one(None); one(prompt)                                                 # warm-up: every shape of the timed calls
        runs = {"unprompted": [], "prompted": []}
        for _ in range(reps):                                                  # alternated, so drifts of a shared host hit both alike
            for name, p in (("unprompted", None), ("prompted", prompt)):
                runs[name].append(one(p))
    for name, rs in runs.items():
        out = {}
        for k in ("audio_s_per_s", "eval_ms", "semantic_ms", "coarse_ms", "fine_ms"):
            v = sorted(r[k] for r in rs)
            out[k] = dict(min=v[0], median=float(np.median(v)), max=v[-1])
        out["audio_s"], out["n_semantic"] = rs[0]["audio_s"], rs[0]["n_semantic"]
        res[name] = out
        print(f"{name:>10}: {out['audio_s']:.2f} s of audio ({out['n_semantic']} semantic ids), e2e {out['audio_s_per_s']['median']:.2f} "
              f"[{out['audio_s_per_s']['min']:.2f}, {out['audio_s_per_s']['max']:.2f}] audio s/s; median ms: semantic "
              f"{out['semantic_ms']['median']:.1f}, coarse {out['coarse_ms']['median']:.1f}, fine {out['fine_ms']['median']:.1f}, "
              f"eval {out['eval_ms']['median']:.1f}", flush=True)
    os.makedirs(OUT, exist_ok=True)
    json.dump(res, open(os.path.join(OUT, "prompt_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
