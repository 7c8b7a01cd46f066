#!/usr/bin/env python
"""What upstream Bark's text tokenizer (DESIGN.md §17) costs per prompt, on the host.

usage: python tools/tokenize_bench.py [--reps R] [--calls N]
1. No device needed: bark_b200_bert_tokenize on a 256-piece text over a synthetic vocabulary of the real size (119,547 entries,
   bert-base-multilingual-cased's count): the five specials, the ASCII pieces of weights.synth_vocab, and seeded pieces of 1 to 6
   characters from Latin-1, Latin Extended, Greek, Cyrillic, Devanagari, Hangul and kana, whole and "##", and single CJK characters.
   The text is words of a first piece and 0 to 2 continuations, and CJK characters: 256 pieces.  The hook builds its std::map of the
   vocabulary on every call (about 0.1 s, which buries one text's tokenization), so it is timed on the empty text and on K = 256 copies
   of the text joined by spaces: the tokenization of one 256-piece text is the difference of the medians over K.  Per call: min /
   median / max over R rounds of N calls.
2. Where a device exists: bark_b200_text_ids on a context (tiny f16 weights written with that vocabulary), the BERT and the reference
   tokenizer on the same text, the way a generation pays for it (the map is built once at load).
Prints a table and writes $BARK_TOOLS_OUT/tokenize_bench.json with the host's CPU model (and the card's name and power limit when a
device ran).
"""
import argparse
import dataclasses
import json
import os
import platform
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

N_VOCAB = 119547
BLOCKS = [(0xC0, 0x24F), (0x391, 0x3C9), (0x410, 0x44F), (0x905, 0x939), (0xAC00, 0xD7A3), (0x3041, 0x30FA), (0x4E00, 0x9FFF)]


def vocabulary(weights, seed=0):
    """extra_words of a weights.Config whose synth_vocab has N_VOCAB entries, mostly multilingual pieces, all distinct.  CJK entries
    are single characters without "##", as in the real vocabulary (each CJK character is a word of its own)."""
    rng = np.random.default_rng(seed)
    base = weights.synth_vocab(dataclasses.replace(weights.tiny(), extra_words=[]))
    seen, extra = set(base), []
    while len(base) + len(extra) < N_VOCAB:
        lo, hi = BLOCKS[int(rng.integers(len(BLOCKS)))]
        if lo == 0x4E00:
            w = chr(int(rng.integers(lo, hi + 1)))
        else:
            w = ("##" if rng.random() < 0.5 else "") + "".join(chr(int(c)) for c in rng.integers(lo, hi + 1, int(rng.integers(1, 7))))
        if w not in seen:
            seen.add(w)
            extra.append(w)
    return extra, weights.synth_vocab(dataclasses.replace(weights.tiny(), extra_words=extra))    # the order a weights file holds


def text_of(vocab, seed=1):
    """Words of a whole piece and 0 to 2 continuation pieces glued to it, or a CJK character, up to 256 pieces in all."""
    rng = np.random.default_rng(seed)
    heads = [v for v in vocab if not v.startswith("##") and not v.startswith("[") and len(v) > 1]
    tails = [v[2:] for v in vocab if v.startswith("##") and len(v) > 3]
    cjk = [v for v in vocab if len(v) == 1 and 0x4E00 <= ord(v) <= 0x9FFF]
    words, n = [], 0
    while n < 256:
        if rng.random() < 0.15:
            words.append(cjk[int(rng.integers(len(cjk)))])
            n += 1
            continue
        w = heads[int(rng.integers(len(heads)))]
        for _ in range(min(int(rng.integers(0, 3)), 255 - n)):
            w += tails[int(rng.integers(len(tails)))]
            n += 1
        words.append(w)
        n += 1
    return " ".join(words)


def timed(fn, reps, calls):
    per = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        per.append((time.perf_counter() - t0) / calls * 1e6)
    return {"min_us": min(per), "median_us": float(np.median(per)), "max_us": max(per)}


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    pkg = graft.load_package()
    weights = graft.importlib.import_module("bark_cpp_b200.weights")
    extra, vocab = vocabulary(weights)
    text = text_of(vocab)
    ids = pkg.bert_tokenize(vocab, text)
    res = {"vocab_entries": len(vocab), "text_bytes": len(text.encode()), "pieces": int(ids.size), "unk": int((ids == 1).sum()),
           "cpu": cpu_model()}
    L = pkg.lib()
    import ctypes as C
    arr = (C.c_char_p * len(vocab))(*[v.encode() for v in vocab])
    K = 256
    out = np.zeros(256 * K, np.int32)
    tb, tk = text.encode(), " ".join([text] * K).encode()
    hook = lambda t: L.bark_b200_bert_tokenize(arr, len(vocab), t, out.ctypes.data_as(C.c_void_p), out.size)  # noqa: E731
    assert hook(tk) == K * ids.size
    res["hook_text"] = timed(lambda: hook(tb), a.reps, a.calls)
    res["hook_empty_text"] = timed(lambda: hook(b""), a.reps, a.calls)
    res[f"hook_{K}_copies"] = timed(lambda: hook(tk), a.reps, a.calls)
    res["tokenize_one_text_us"] = (res[f"hook_{K}_copies"]["median_us"] - res["hook_empty_text"]["median_us"]) / K
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except ImportError:
        have_gpu = False
    if have_gpu:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "tiny_big_vocab.bin")
            weights.write_weights(path, dataclasses.replace(weights.tiny(), extra_words=extra), seed=1234)
            with pkg.Bark(path) as b:
                assert np.array_equal(b.text_ids(text, "bert"), ids)
                for kind in ("bert", "reference"):
                    k = pkg.TOKENIZERS[kind]
                    ctx_call = lambda: L.bark_b200_text_ids(b.ctx, k, tb, out.ctypes.data_as(C.c_void_p), out.size)  # noqa: E731
                    ctx_call()
                    res[f"text_ids_{kind}"] = timed(ctx_call, a.reps, a.calls * 5)
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        res["card"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print(f"{res['vocab_entries']} vocabulary entries, text of {res['text_bytes']} bytes -> {res['pieces']} pieces ({res['unk']} [UNK]); "
          f"{res['cpu']}")
    for k, v in res.items():
        if isinstance(v, dict):
            print(f"  {k:24s} min {v['min_us']:10.1f} us   median {v['median_us']:10.1f} us   max {v['max_us']:10.1f} us")
    print(f"  tokenization of one 256-piece text (hook, from {K} copies): {res['tokenize_one_text_us']:.1f} us")
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "tokenize_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
