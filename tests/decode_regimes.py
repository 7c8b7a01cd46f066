"""The persistent decode step's branch regimes, restated on the CPU (bark.cpp_b200/csrc/decode_kernels.cu, gpt_decode_step_kernel).

Which branch a warp of the decode step takes depends on the model's widths, its weight type, the CTA count and n_kv:
  * split or unsplit grid (`score_cta0`): with at least H * (D / 16) + 64 CTAs the soft_max CTAs take no score tasks and the score
    CTAs prefetch their K rows; with fewer every CTA takes score tasks and no K row is prefetched;
  * score tasks beyond the staged K rows (`p2_scores`, the loop after `done`): a warp's key tail (`key_tail`) holds `cap` tasks,
    the rest come straight from global memory;
  * V rows from global memory in P.V (`p3_attention`, `vs_ok == false`): the V tile does not fit behind the warp's c_proj rows;
  * the soft_max and P.V leftovers of n_kv % 8 and n_kv % 32.
This module restates `warp_rows`, `staged_bytes_of`, `q4_staged`, `key_tail`, the `vs_ok` test, `score_cta0`, the balanced row split
of the kernel's phase table and the CTA count bark_load_model picks.  The constants are read from the sources, so a retuned staging
slot moves the thresholds here too.  BANDS lists the decode steps tests/test_long_context_gpu.py compares with the oracle;
tests/test_decode_regimes.py checks that they reach every regime.
"""
from __future__ import annotations

import functools
import os
import re
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bark.cpp_b200", "csrc")


def _grab(file: str, name: str, pattern: str) -> str:
    with open(os.path.join(CSRC, file)) as f:
        m = re.search(pattern, f.read())
    if not m:
        raise RuntimeError(f"{name}: pattern {pattern!r} not found in {file}; the restatement in tests/decode_regimes.py is out of date")
    return m.group(1)


def _int_expr(file: str, name: str) -> int:
    e = _grab(file, name, rf"constexpr int {name}\s*=\s*([0-9 *+]+);")
    return int(eval(e, {"__builtins__": {}}))         # digits, spaces, * and + only (the pattern admits nothing else)


K_THREADS = _int_expr("decode_kernels.cu", "kThreads")
K_WARPS = K_THREADS // 32
K_WARP_SLOT_BYTES = _int_expr("decode_kernels.cu", "kWarpSlotBytes")
K_HALF_SLOT_BYTES = K_WARP_SLOT_BYTES // 2
K_MAX_TASKS = _int_expr("decode_kernels.cu", "kMaxTasks")
CAP_TASKS = int(_grab("decode_kernels.cu", "key_tail cap", r"cap = min\((\d+) \* kMaxTasks,")) * K_MAX_TASKS
SPLIT_SCORE_CTAS = int(_grab("decode_kernels.cu", "score_cta0", r"gridDim\.x >= \(unsigned\)\(H \* parts \+ (\d+)\)"))
SM_CLAMP_FROM = int(_grab("bark_api.cu", "decode CTA clamp", r"if \(ctx->n_sm >= (\d+)\) ctx->n_sm = \d+;"))
SM_CLAMP_TO = int(_grab("bark_api.cu", "decode CTA clamp", r"if \(ctx->n_sm >= \d+\) ctx->n_sm = (\d+);"))
KNOB_MIN = int(_grab("bark_api.cu", "BARK_B200_DECODE_CTAS", r"BARK_B200_DECODE_CTAS\"\); if \(e && atoi\(e\) >= (\d+)"))
BLOCK_SIZE = 1024                                      # every Bark GPT's context (weights.GPTDims.block_size)


def launch_ctas(n_sms: int, knob: int | None = None) -> int:
    """CTAs of the decode step on a device with n_sms SMs, BARK_B200_DECODE_CTAS = knob (None: unset)."""
    n = SM_CLAMP_TO if n_sms >= SM_CLAMP_FROM else n_sms
    return knob if knob is not None and KNOB_MIN <= knob <= n else n


@dataclass(frozen=True)
class Model:
    E: int
    H: int
    wtype: str                                         # "f16", "f32" or "q4_0"

    @property
    def D(self) -> int:
        return self.E // self.H

    def phase(self, i: int) -> tuple[int, int]:
        """(n_out, K) of phase i of a layer: c_attn, c_proj, mlp c_fc, mlp c_proj"""
        E = self.E
        return ((3 * E, E), (E, E), (4 * E, E), (E, 4 * E))[i]

    def row_bytes(self, K: int) -> int:
        if self.wtype == "q4_0":
            return K // 2                              # 16-byte nibble words per 32-element block; the f16 scales are a second array
        es = 2 if self.wtype == "f16" else 4
        q = 32 * (16 // es)                            # li_padded_k (common.cuh)
        return (K + q - 1) // q * q * es


def _cta_rows(n: int, G: int):
    """the kernel's balanced split: CTA c owns rows [r0[c], r1[c]) of an n-row phase"""
    c = np.arange(G)
    base, rem = divmod(n, G)
    r0 = c * base + np.minimum(c, rem)
    return r0, r0 + base + (c < rem)


def staged_bytes(m: Model, phase: int, G: int) -> np.ndarray:
    """[G][16] bytes of each warp's staging half that the phase occupies (staged_bytes_of)"""
    n_out, K = m.phase(phase)
    r0, r1 = _cta_rows(n_out, G)
    n = (r1 - r0)[:, None]
    w = np.arange(K_WARPS)[None, :]
    a = r0[:, None] + ((w * n) >> 4)
    b = r0[:, None] + (((w + 1) * n) >> 4)
    qbytes = (b - a) * m.row_bytes(K)
    if m.wtype != "q4_0":
        return np.where(qbytes <= K_HALF_SLOT_BYTES, qbytes, 0)
    sbytes = (b - a) * (K >> 5) * 2
    # q4_staged; the scale array starts on a cudaMalloc boundary, so the row's address is 16-byte aligned iff its offset is
    ok = (qbytes != 0) & (qbytes + sbytes <= K_HALF_SLOT_BYTES) & (sbytes % 16 == 0) & ((a * (K >> 5) * 2) % 16 == 0)
    return np.where(ok, qbytes + sbytes, 0)


@dataclass(frozen=True)
class Layout:
    """What every warp of one (model, CTA count) grid holds; independent of n_kv."""
    model: Model
    G: int
    split: bool
    score_cta0: int
    cap: np.ndarray                                    # [score CTAs][16]: tasks the warp's key tail holds (0 when unsplit)
    gw: np.ndarray                                     # [score CTAs][16]: the warp's first task
    nw: int                                            # score warps of the grid (task stride)
    voff: np.ndarray                                   # [soft_max CTAs][16]: where the warp's V tile starts in its staging half

    def beyond_cap(self, n_kv: int) -> np.ndarray:
        """[score CTAs][16]: the warp has score tasks that read K from global memory (t = gw + cap * nw < H * n_past)"""
        return self.gw + self.cap * self.nw < self.model.H * (n_kv - 1)

    def vs_ok(self, n_kv: int) -> np.ndarray:
        """[soft_max CTAs][16]: the warp's V rows fit its staging half"""
        nstep_all = (n_kv + 31) // 32
        return self.voff + nstep_all * 128 <= K_HALF_SLOT_BYTES

    def first(self, pred) -> int | None:
        """the first n_kv in 2 .. 1024 at which pred(n_kv) holds"""
        return next((n for n in range(2, BLOCK_SIZE + 1) if pred(n)), None)


@functools.lru_cache(maxsize=None)
def layout(m: Model, G: int) -> Layout:
    parts = m.D // 16
    n_pv = m.H * parts
    if n_pv > G:
        raise ValueError(f"{m}: {n_pv} soft_max tiles need more than {G} CTAs (the model decodes through the per-op kernels)")
    split = G >= n_pv + SPLIT_SCORE_CTAS
    cta0 = n_pv if split else 0
    sc = slice(cta0, G)
    if split:
        off = (np.maximum(staged_bytes(m, 0, G), staged_bytes(m, 2, G))[sc] + 127) & ~127
        cap = np.minimum(CAP_TASKS, (K_HALF_SLOT_BYTES - np.minimum(off, K_HALF_SLOT_BYTES)) // (m.D * 4))
    else:
        cap = np.zeros((G, K_WARPS), np.int64)
    gw = (np.arange(G - cta0)[:, None] * K_WARPS + np.arange(K_WARPS)[None, :])
    voff = (staged_bytes(m, 1, G)[:n_pv] + 127) & ~127
    return Layout(m, G, split, cta0, cap, gw, (G - cta0) * K_WARPS, voff)


def regimes(m: Model, G: int, n_kv: int) -> frozenset:
    """the branches one decode step at n_kv (n_past = n_kv - 1) takes, as labels"""
    lay = layout(m, G)
    out = {"split" if lay.split else "unsplit"}
    if not lay.split:
        out.add("K from global only")
    elif lay.beyond_cap(n_kv).any():
        out.add("K staged + beyond cap")
    else:
        out.add("K staged only")
    out.add("V staged" if lay.vs_ok(n_kv).all() else "V from global")
    out.add("n_kv % 8 tail" if n_kv % 8 else "n_kv % 32 tail" if n_kv % 32 else "no tail")
    if n_kv == BLOCK_SIZE:
        out.add("last position")
    return frozenset(out)


# ---- the GPU bands ----------------------------------------------------------------------------------------------------------------
# Models of tests/test_long_context_gpu.py: the regimes depend on the widths and the weight type only.  "small2" is bark-small's width
# (E 768, 12 heads) at 2 layers.
MODELS = {
    "tiny_f16": Model(128, 2, "f16"), "mini_f32": Model(256, 4, "f32"), "mini_f16": Model(256, 4, "f16"),
    "wide_f16": Model(1024, 16, "f16"), "wide_f32": Model(1024, 16, "f32"), "small2_f32": Model(768, 12, "f32"),
    "tiny_q4_0": Model(128, 2, "q4_0"), "wide_q4_0": Model(1024, 16, "q4_0"),
}
BAND_STEPS = 12                                        # single-token steps per band: n_kv = start .. start + 11
# model -> (CTA counts, first n_kv of each band).  Bands straddle n_kv 513/514 (bark-large f16 keys beyond the tail, f32 V from
# global), 768/769 (bark-small f32 V from global) and end at 1024 (the last position).  CTA counts: 128 (an H100 SXM), the split
# boundary of the model (tiny 72 / 71, wide 128 / 127), 64 (every CTA a soft_max tile at 16 heads) and 97 (rows split with remainders).
BANDS = {
    "tiny_f16": ((128, 97, 72, 71, 64), (505, 761, 1013)),
    "mini_f32": ((128, 64), (505, 1013)),
    "mini_f16": ((128, 64), (505, 1013)),
    "wide_f16": ((128, 127, 97, 64), (505, 761, 1013)),
    "wide_f32": ((128, 127), (505, 761, 1013)),
    "small2_f32": ((128,), (761, 1013)),
    "tiny_q4_0": ((128, 71), (505, 1013)),
    "wide_q4_0": ((128, 127), (505, 1013)),
}
# the per-op path (BARK_B200_DECODE=multi) replays these models' bands once, at the default CTA count
PER_OP_MODELS = ("tiny_f16", "wide_f16")


def band_kvs(start: int) -> range:
    return range(start, start + BAND_STEPS)


def reached(models=None) -> dict:
    """weight type -> the regimes the bands reach"""
    out: dict = {}
    for name, (ctas, starts) in BANDS.items():
        if models is not None and name not in models:
            continue
        m = MODELS[name]
        for G in ctas:
            for s in starts:
                for n_kv in band_kvs(s):
                    out.setdefault(m.wtype, set()).update(regimes(m, G, n_kv))
    return out


def reachable() -> dict:
    """weight type -> every regime the bands' models can take, over every CTA count the library launches (64 .. 128) and n_kv 2 .. 1024"""
    out: dict = {}
    for m in {MODELS[n] for n in BANDS}:
        for G in range(KNOB_MIN, SM_CLAMP_TO + 1):
            if m.H * (m.D // 16) > G:
                continue
            for n_kv in range(2, BLOCK_SIZE + 1):
                out.setdefault(m.wtype, set()).update(regimes(m, G, n_kv))
    return out
