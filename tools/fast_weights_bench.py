#!/usr/bin/env python
"""Fast mode on f32 and quantised files, on an H100: what the fine model's load-time f16 conversion buys.

usage: python tools/fast_weights_bench.py [--reps R] [--types f16,f32,q4_0,q8_0]
bark-small-sized synthetic files (bark.cpp_b200/weights.py, seed 1234): f16 and f32 as written, q4_0 and q8_0 made from the f16 file
by bark_model_quantize.  Per type, one context in the parity path and one with BARK_B200_MODE=fast, both loaded before timing; "hello
world" with seed 0 and n_steps_text_encoder = 138 (the bench clip), parity and fast alternated R times after one warm-up of each:
fine-stage ms (bark_statistics t_fine_us) and end-to-end audio seconds per wall second, min / median / max over the R runs, plus
the load time of each context and the bytes of the fine model's f16 copy computed from its shapes.  Prints a table and writes
$BARK_TOOLS_OUT/fast_weights_bench.json with the card's name and power limit read in the same call.
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
QUANT_FTYPE = {"q4_0": 2, "q4_1": 3, "q8_0": 7, "q5_0": 8, "q5_1": 9}       # enum ggml_ftype


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def weight_file(pkg, weights, t):
    """bark-small-sized file of type t in the bench's fixture directory (outside the tree and the results directory)"""
    os.makedirs(bench.FIXTURE_DIR, exist_ok=True)
    src = os.path.join(bench.FIXTURE_DIR, f"small_{'f32' if t == 'f32' else 'f16'}_1234.bin")
    if not os.path.exists(src):
        weights.write_weights(src + ".tmp", weights.small(weights.F32 if t == "f32" else weights.F16), 1234)
        os.replace(src + ".tmp", src)
    if t in ("f16", "f32"):
        return src
    path = os.path.join(bench.FIXTURE_DIR, f"small_{t}_1234.bin")
    if not os.path.exists(path):
        if not pkg.lib().bark_model_quantize(src.encode(), (path + ".tmp").encode(), QUANT_FTYPE[t]):
            raise RuntimeError("bark_model_quantize failed")
        os.replace(path + ".tmp", path)
    return path


def f16_copy_bytes(cfg):
    E, L, V = cfg.fine.n_embd, cfg.fine.n_layer, cfg.fine_vocab
    return 2 * (L * 12 * E * E + 7 * V * E)


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3
    types = sys.argv[sys.argv.index("--types") + 1].split(",") if "--types" in sys.argv else ["f16", "f32", "q4_0", "q8_0"]
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    res = dict(card=card(), weights="bark-small dims, synthetic (seed 1234)", n_steps_text_encoder=N_STEPS, text=TEXT, seed=SEED, reps=reps,
               f16_copy_mb=dict(small=f16_copy_bytes(weights.small()) / 1e6, large=f16_copy_bytes(weights.large()) / 1e6), types={})
    print(f"card: {res['card']}", flush=True)
    for t in types:
        path = weight_file(pkg, weights, t)
        ctxs = {}
        for mode in ("parity", "fast"):
            os.environ["BARK_B200_MODE"] = mode
            t0 = time.perf_counter()
            ctxs[mode] = pkg.Bark(path, seed=SEED, n_steps_text_encoder=N_STEPS)
            load_s = time.perf_counter() - t0
            if ctxs[mode].fast_mode != (mode == "fast"):
                raise RuntimeError(f"{t}: {mode} context has fast_mode {ctxs[mode].fast_mode}")
            ctxs[mode].load_s = load_s
        os.environ.pop("BARK_B200_MODE", None)

        def one(b):
            b.reseed(SEED)
            t0 = time.perf_counter()
            a = b.generate(TEXT)
            wall = time.perf_counter() - t0
            s, _ = b.stats()
            return dict(audio_s_per_s=a.size / SR / wall, audio_s=a.size / SR, fine_ms=s.t_fine_us / 1e3, eval_ms=s.t_eval_us / 1e3)

        for b in ctxs.values():
            one(b)                                                     # warm-up: every shape of the timed calls
        runs = {m: [] for m in ctxs}
        for _ in range(reps):                                          # alternated, so drifts of a shared host hit both alike
            for m, b in ctxs.items():
                runs[m].append(one(b))
        out = {}
        for m, rs in runs.items():
            o = dict(load_s=ctxs[m].load_s, audio_s=rs[0]["audio_s"])
            for k in ("audio_s_per_s", "fine_ms", "eval_ms"):
                v = sorted(r[k] for r in rs)
                o[k] = dict(min=v[0], median=float(np.median(v)), max=v[-1])
            out[m] = o
            ctxs[m].close()
        out["fine_speedup_median"] = out["parity"]["fine_ms"]["median"] / out["fast"]["fine_ms"]["median"]
        out["e2e_speedup_median"] = out["fast"]["audio_s_per_s"]["median"] / out["parity"]["audio_s_per_s"]["median"]
        res["types"][t] = out
        for m in ("parity", "fast"):
            o = out[m]
            print(f"{t:>5} {m:>6}: fine {o['fine_ms']['median']:.1f} ms [{o['fine_ms']['min']:.1f}, {o['fine_ms']['max']:.1f}], e2e "
                  f"{o['audio_s_per_s']['median']:.2f} [{o['audio_s_per_s']['min']:.2f}, {o['audio_s_per_s']['max']:.2f}] audio s/s "
                  f"({o['audio_s']:.2f} s of audio), load {o['load_s']:.1f} s", flush=True)
        print(f"{t:>5}: fine stage x{out['fine_speedup_median']:.2f}, e2e x{out['e2e_speedup_median']:.2f} (medians)", flush=True)
    os.makedirs(OUT, exist_ok=True)
    json.dump(res, open(os.path.join(OUT, "fast_weights_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
