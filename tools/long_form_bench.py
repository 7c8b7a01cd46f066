#!/usr/bin/env python
"""What long-form generation (DESIGN.md §18) costs against the loop a caller would write in Python.

usage: python tools/long_form_bench.py [--reps R] [--n-steps N]
1. A paragraph of 7 sentences on bark-small f16 weights (weights.py, seed 1234): bark_generate_audio with long form on (chain voice,
   defaults) against the Python loop it stands for (split_text, then per chunk set_history_prompt of the previous chunk's ids and
   generate, the waveforms joined with the same gap), alternated R times after one warm-up of each.  Every round checks that both give
   the same waveform bit for bit.  Wall time (min / median / max), audio s/s of the generated audio (gaps excluded), and the difference
   of the medians with the spread of each arm.
2. The splitter on the host: bark_b200_split_text on a 10 KB text (the paragraph repeated), minus the same call on a one-word text (the
   hook builds its vocabulary map per call), median of R rounds of 20 calls.
Prints a table and writes $BARK_TOOLS_OUT/long_form_bench.json with the card's name and power limit, read in the same run.
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
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402

PARAGRAPH = ("The old lighthouse stood at the edge of the cliff. Every night its lamp swept across the dark water! Sailors trusted it "
             "more than their charts. One winter the keeper fell ill and the light went out. Three ships ran aground before dawn. "
             "Nobody in the village ever forgot that night. Is the lamp still burning today?")


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unknown ({e})"


def spread(v):
    return dict(min=float(np.min(v)), median=float(np.median(v)), max=float(np.max(v)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-steps", type=int, default=138, help="n_steps_text_encoder (138: the bench clip's)")
    args = ap.parse_args()
    pkg = graft.load_package()
    import importlib
    weights = importlib.import_module("bark_cpp_b200.weights")
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(tempfile.gettempdir(), f"bark_b200_fixtures_{os.getuid()}", "small_f16_1234.bin")
    if not os.path.exists(path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        weights.write_weights(path + ".tmp", weights.CONFIGS["small"](weights.F16), 1234)
        os.replace(path + ".tmp", path)
    vocab = weights.synth_vocab(weights.CONFIGS["small"](weights.F16))
    chunks = pkg.split_text(vocab, PARAGRAPH)
    gap = 6000

    def library(b):
        b.set_long_form("chain")
        t = time.perf_counter()
        a = b.generate(PARAGRAPH)
        return time.perf_counter() - t, a

    def loop(b):
        b.set_long_form(None)
        t = time.perf_counter()
        out = []
        for k, c in enumerate(chunks):
            if k:
                try:
                    b.set_history_prompt(b.last_generation_prompt())
                except ValueError:
                    pass
                out.append(np.zeros(gap, np.float32))
            out.append(b.generate(c))
        a = np.concatenate(out)
        dt = time.perf_counter() - t
        b.set_history_prompt(None)
        return dt, a

    res = {"library": [], "loop": []}
    n_audio = None
    with pkg.Bark(path, seed=0, n_steps_text_encoder=args.n_steps) as b1, pkg.Bark(path, seed=0, n_steps_text_encoder=args.n_steps) as b2:
        library(b1); loop(b2)                                                      # warm-up: same RNG position on both afterwards
        for r in range(args.reps):
            dl, al = library(b1)
            dp, ap_ = loop(b2)
            assert np.array_equal(al.view(np.uint32), ap_.view(np.uint32)), f"round {r}: long form and the loop differ"
            res["library"].append(dl); res["loop"].append(dp)
            n_audio = al.size - gap * (len(chunks) - 1)
    secs = n_audio / 24000
    summary = {k: dict(wall_s=spread(v), audio_s_per_s=spread([secs / x for x in v])) for k, v in res.items()}
    diff = float(np.median(res["library"]) - np.median(res["loop"]))

    text10k = " ".join([PARAGRAPH] * (10240 // len(PARAGRAPH) + 1))[:10240].rsplit(" ", 1)[0]
    split = {}
    for name, t in (("10KB", text10k), ("one_word", "lighthouse")):
        per = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            for _ in range(20):
                n = len(pkg.split_text(vocab, t))
            per.append((time.perf_counter() - t0) / 20)
        split[name] = dict(seconds=float(np.median(per)), chunks=n)
    split_ms = (split["10KB"]["seconds"] - split["one_word"]["seconds"]) * 1e3

    result = dict(card=card(), n_steps=args.n_steps, reps=args.reps, chunks=len(chunks), audio_s=secs, gap_samples=gap, arms=summary,
                  median_difference_s=diff, raw=res, splitter=split, splitter_10kb_ms=split_ms, bytes_10kb=len(text10k.encode()))
    with open(os.path.join(OUT, "long_form_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(f"card: {result['card']}")
    print(f"{len(chunks)} chunks, {secs:.2f} s of audio, n_steps {args.n_steps}, {args.reps} rounds")
    for k, v in summary.items():
        w, a = v["wall_s"], v["audio_s_per_s"]
        print(f"  {k:8s} wall {w['min']:.3f} / {w['median']:.3f} / {w['max']:.3f} s   audio s/s {a['min']:.2f} / {a['median']:.2f} / {a['max']:.2f}")
    print(f"  median difference (library - loop): {diff * 1e3:+.1f} ms")
    print(f"splitter: {split_ms:.3f} ms for {len(text10k.encode())} bytes ({split['10KB']['chunks']} chunks)")


if __name__ == "__main__":
    main()
