"""Synthetic `ggml_weights.bin` writer (test / bench fixture generator).

No Bark checkpoint can be fetched offline, and the reference loader takes every dimension from the
file header (bark.cpp:700-709, encodec.cpp/encodec.cpp:156-165), so parity and throughput are
measured on files of the exact reference format filled with seeded random weights.  The byte
layout follows the reference writer (convert.py:293-350) and readers (bark.cpp:664-690,
692-1078, 1080-1163; encodec.cpp/encodec.cpp:141-502); see DESIGN.md "File format".

Distributions (SURVEY.md §8d): GPT matrices N(0, 0.02^2), LayerNorm gains 1 + N(0, 0.02^2), fine
LayerNorm biases N(0, 0.02^2), lm_head N(0, 0.2^2), codec conv / LSTM weights N(0, 1/fan_in)
stored F16, codec biases N(0, 0.02^2), codebooks N(0, 1).

The numpy PCG64 stream is platform independent, so the same (config, seed) gives the same bytes in
every machine.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

MAGIC = 0x67676D6C  # 'ggml'
F32, F16, Q4_0 = 0, 1, 2


@dataclass
class GPTDims:
    n_layer: int
    n_head: int
    n_embd: int
    block_size: int = 1024


@dataclass
class Config:
    name: str
    semantic: GPTDims
    coarse: GPTDims
    fine: GPTDims
    gpt_ftype: int = F16      # 0 = f32, 1 = f16 (q4_0 files are made from these, see quantize_q4_0)
    codec_ftype: int = F16    # must stay F16: an f32 codec aborts in the reference (ggml.c:14899)
    lm_head_std: float = 0.2
    # vocabulary sizes are pinned by constants in the reference (bark.cpp:2215-2226)
    sem_in: int = 129600
    sem_out: int = 10048
    coarse_vocab: int = 12096
    fine_vocab: int = 1056
    extra_words: list = field(default_factory=lambda: ["hello", "world", "the", "quick", "brown", "fox"])


def small(ftype=F16):
    d = GPTDims(12, 12, 768)
    return Config("bark-small", d, d, d, gpt_ftype=ftype)


def large(ftype=F16):
    d = GPTDims(24, 16, 1024)
    return Config("bark-large", d, d, d, gpt_ftype=ftype)


def tiny(ftype=F16):
    """2 layers, E=128, head 64 — seconds on the CPU oracle; exercises the K%32==0 paths."""
    d = GPTDims(2, 2, 128)
    return Config("tiny", d, d, d, gpt_ftype=ftype)


def mini(ftype=F16):
    """3 layers, E=256, 4 heads of 64; different depth per stage to catch index mix-ups."""
    return Config("mini", GPTDims(3, 4, 256), GPTDims(2, 4, 256), GPTDims(2, 4, 256), gpt_ftype=ftype)


def wide(ftype=F16):
    """bark-large widths (E=1024, 16 heads of 64, K=4096 MLP rows) at 2 layers: the shapes of BASELINE configs[2] at a depth the
    CPU oracle finishes in seconds."""
    d = GPTDims(2, 16, 1024)
    return Config("wide", d, d, d, gpt_ftype=ftype)


CONFIGS = {"tiny": tiny, "mini": mini, "small": small, "large": large, "wide": wide}


def synth_vocab(cfg: Config):
    """A WordPiece vocabulary small enough to write quickly but rich enough to tokenize ASCII text:
    specials, every printable ASCII char as a word start and as a '##' continuation, a few words."""
    toks = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    chars = [chr(c) for c in range(33, 127)]
    toks += chars
    toks += ["##" + c for c in chars]
    toks += cfg.extra_words
    toks += ["##" + w for w in ("ing", "ed", "ly", "er", "s")]
    return toks


class _Writer:
    def __init__(self, f, rng, overrides=None):
        self.f, self.rng = f, rng
        self.overrides = dict(overrides or {})
        self.scope = ""                          # "semantic/", "coarse/", "fine/" while a GPT is written, "" for the codec

    def i32(self, *v):
        self.f.write(struct.pack("<%di" % len(v), *v))

    def tensor(self, name: str, arr: np.ndarray, ttype: int):
        new = self.overrides.pop(self.scope + name, None)
        if new is not None:                      # the seeded values are still drawn, so every other tensor keeps its bytes
            assert np.shape(new) == arr.shape, (self.scope + name, np.shape(new), arr.shape)
            arr = np.asarray(new)
        arr = np.ascontiguousarray(arr.astype(np.float16 if ttype == F16 else np.float32))
        nb = name.encode()
        self.i32(arr.ndim, len(nb), ttype)
        for d in reversed(arr.shape):          # ggml order = reversed numpy shape (convert.py:286-287)
            self.i32(d)
        self.f.write(nb)
        self.f.write(arr.tobytes())

    def normal(self, shape, std, mean=0.0):
        n = int(np.prod(shape))
        out = np.empty(n, dtype=np.float32)
        step = 1 << 24                           # bounded temporaries for the 130k x 768 tables
        for s in range(0, n, step):
            e = min(n, s + step)
            out[s:e] = self.rng.standard_normal(e - s, dtype=np.float32)
        out *= np.float32(std)
        if mean:
            out += np.float32(mean)
        return out.reshape(shape)


def _write_gpt(w: _Writer, d: GPTDims, n_in, n_out, n_lm_heads, n_wtes, bias, ftype, lm_std):
    E, L = d.n_embd, d.n_layer
    w.i32(L, d.n_head, E, d.block_size, bias, n_in, n_out, n_lm_heads, n_wtes, ftype)
    n_tensors = n_wtes + 1 + n_lm_heads + (2 if bias else 1) + L * (4 + (4 if bias else 2))
    w.i32(n_tensors)
    wt = F16 if ftype == F16 else F32
    for i in range(n_wtes):
        w.tensor(f"model/wte/{i}", w.normal((n_in, E), 0.02), wt)
    w.tensor("model/wpe", w.normal((d.block_size, E), 0.02), F32)
    for l in range(L):
        w.tensor(f"model/h{l}/ln_1/g", w.normal((E,), 0.02, 1.0), F32)
        if bias:
            w.tensor(f"model/h{l}/ln_1/b", w.normal((E,), 0.02), F32)
        w.tensor(f"model/h{l}/attn/c_attn/w", w.normal((3 * E, E), 0.02), wt)
        w.tensor(f"model/h{l}/attn/c_proj/w", w.normal((E, E), 0.02), wt)
        w.tensor(f"model/h{l}/ln_2/g", w.normal((E,), 0.02, 1.0), F32)
        if bias:
            w.tensor(f"model/h{l}/ln_2/b", w.normal((E,), 0.02), F32)
        w.tensor(f"model/h{l}/mlp/c_fc/w", w.normal((4 * E, E), 0.02), wt)
        w.tensor(f"model/h{l}/mlp/c_proj/w", w.normal((E, 4 * E), 0.02), wt)
    w.tensor("model/ln_f/g", w.normal((E,), 0.02, 1.0), F32)
    if bias:
        w.tensor("model/ln_f/b", w.normal((E,), 0.02), F32)
    for i in range(n_lm_heads):
        w.tensor(f"model/lm_head/{i}", w.normal((n_out, E), lm_std), wt)


def _write_codec(w: _Writer, ftype: int, with_encoder: bool):
    hidden, nf, k, rk, n_bins = 128, 32, 7, 3, 1024
    ratios = [8, 5, 4, 2]
    w.i32(1, hidden, nf, k, rk, n_bins, 24, 24000, ftype)   # bandwidth 24 like convert.py:69
    wt = F16 if ftype == F16 else F32

    def conv(name, cout, cin, ks):                           # torch shape [Cout, Cin, k]
        w.tensor(name + ".weight", w.normal((cout, cin, ks), (1.0 / (cin * ks)) ** 0.5), wt)
        w.tensor(name + ".bias", w.normal((cout,), 0.02), F32)

    def convtr(name, cin, cout, ks):                         # torch shape [Cin, Cout, k]
        w.tensor(name + ".weight", w.normal((cin, cout, ks), (1.0 / (cin * ks)) ** 0.5), wt)
        w.tensor(name + ".bias", w.normal((cout,), 0.02), F32)

    def lstm(prefix, h):
        for l in range(2):
            w.tensor(f"{prefix}.weight_ih_l{l}", w.normal((4 * h, h), (1.0 / h) ** 0.5), wt)
            w.tensor(f"{prefix}.weight_hh_l{l}", w.normal((4 * h, h), (1.0 / h) ** 0.5), wt)
            w.tensor(f"{prefix}.bias_ih_l{l}", w.normal((4 * h,), 0.02), F32)
            w.tensor(f"{prefix}.bias_hh_l{l}", w.normal((4 * h,), 0.02), F32)

    if with_encoder:  # present in real files; the decoder path never reads them
        mult = 1
        conv("encoder.model.0.conv.conv", nf, 1, k)
        for i in range(4):
            conv(f"encoder.model.{3*i+1}.block.1.conv.conv", mult * nf // 2, mult * nf, rk)
            conv(f"encoder.model.{3*i+1}.block.3.conv.conv", mult * nf, mult * nf // 2, 1)
            conv(f"encoder.model.{3*i+1}.shortcut.conv.conv", mult * nf, mult * nf, 1)
            conv(f"encoder.model.{3*(i+1)}.conv.conv", mult * nf * 2, mult * nf, 2 * ratios[3 - i])
            mult *= 2
        lstm("encoder.model.13.lstm", mult * nf)
        conv("encoder.model.15.conv.conv", hidden, mult * nf, k)

    mult = 16
    conv("decoder.model.0.conv.conv", mult * nf, hidden, k)
    lstm("decoder.model.1.lstm", mult * nf)
    for i in range(4):
        c = mult * nf
        convtr(f"decoder.model.{3*(i+1)}.convtr.convtr", c, c // 2, 2 * ratios[i])
        conv(f"decoder.model.{3*(i+1)+1}.block.1.conv.conv", c // 4, c // 2, rk)
        conv(f"decoder.model.{3*(i+1)+1}.block.3.conv.conv", c // 2, c // 4, 1)
        conv(f"decoder.model.{3*(i+1)+1}.shortcut.conv.conv", c // 2, c // 2, 1)
        mult //= 2
    conv("decoder.model.15.conv.conv", 1, nf, k)
    for q in range(32):
        w.tensor(f"quantizer.vq.layers.{q}._codebook.embed", w.normal((n_bins, hidden), 1.0), F32)


def write_weights(path: str, cfg: Config, seed: int = 1234, with_encoder: bool = True, overrides: dict | None = None) -> str:
    """overrides: tensor name -> array written instead of the seeded values (same shape); the names of the three GPTs' tensors
    are prefixed with "semantic/", "coarse/" or "fine/" (e.g. "coarse/model/wpe"), the codec's are as in the file."""
    rng = np.random.Generator(np.random.PCG64(seed))
    with open(path, "wb") as f:
        w = _Writer(f, rng, overrides)
        f.write(struct.pack("<I", MAGIC))
        vocab = synth_vocab(cfg)
        w.i32(len(vocab))
        for t in vocab:
            b = t.encode()
            f.write(struct.pack("<I", len(b)))
            f.write(b)
        w.scope = "semantic/"
        _write_gpt(w, cfg.semantic, cfg.sem_in, cfg.sem_out, 1, 1, 0, cfg.gpt_ftype, cfg.lm_head_std)
        w.scope = "coarse/"
        _write_gpt(w, cfg.coarse, cfg.coarse_vocab, cfg.coarse_vocab, 1, 1, 0, cfg.gpt_ftype, cfg.lm_head_std)
        w.scope = "fine/"
        _write_gpt(w, cfg.fine, cfg.fine_vocab, cfg.fine_vocab, 7, 8, 1, cfg.gpt_ftype, cfg.lm_head_std)
        f.write(struct.pack("<I", MAGIC))
        w.scope = ""
        _write_codec(w, cfg.codec_ftype, with_encoder)
        if w.overrides:
            raise KeyError(f"no tensor named {sorted(w.overrides)}")
    return path


if __name__ == "__main__":
    import argparse, time
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="tiny", choices=sorted(CONFIGS))
    ap.add_argument("--ftype", default="f16", choices=["f32", "f16"])
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    t0 = time.time()
    write_weights(a.out, CONFIGS[a.config](F16 if a.ftype == "f16" else F32), a.seed)
    print(f"wrote {a.out} in {time.time()-t0:.1f}s")
