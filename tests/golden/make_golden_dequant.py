"""Regenerates tests/golden/ref_pairs/dequant.npz: the unmodified reference's dequantize_row_{q4_0,q4_1,q5_0,q5_1,q8_0}
(oracle/_ref/libbark_ref.so, AVX2 build) on the weight edge blocks of quant_dots.npz and on random rows.  The inputs of
tests/test_fast_weights.py (the numpy restatement, CPU) and tests/test_fast_weights_gpu.py (bark_b200_fast_convert, fast mode's
load-time conversion to f16).

  edge_<t> [B][bytes], edge_<t>_names   quant_dots.npz's w_<t> (d = +-0, f16-subnormal, +-65504; codes all 0 / all 15; q5 high bits;
                                        q4_1 / q5_1 m negative, zero, large; q8_0 codes +-127, -128), then d = +-inf and NaN blocks
  edge_deq_<t> [B][32] f32              dequantize_row_<t> of each block (k = 32)
  rows_<t>_<K> [n][K/32 * bytes]        random rows (n odd) at K = 768 and 4096: d f16 of N(0, 0.02) magnitude, a few blocks with
                                        d = +-65504, m of N(0, 0.5)
  rows_deq_<t>_<K> [n][K] f32           dequantize_row_<t> of each row

Run once where the reference library exists:

    python tests/golden/make_golden_dequant.py
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import __graft_entry__ as graft  # noqa: E402
from make_golden_quant_dots import TYPES, weight_block  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "dequant.npz")
DOTS = os.path.join(HERE, "ref_pairs", "quant_dots.npz")
BYTES = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}
ROWS = {768: 5, 4096: 3}                                # K: rows (odd)


def codes(t, rng, n=32):
    hi = 127 if t == "q8_0" else 31 if t.startswith("q5") else 15
    return rng.integers(-128 if t == "q8_0" else 0, hi + 1, n)


def special_blocks(t, rng):
    """d = +inf, -inf, NaN: every element of the block is inf or NaN in the reference (0 * inf = NaN)"""
    return [(name, weight_block(t, d, codes(t, rng), 0x3c00)) for name, d in (("d_inf", 0x7c00), ("d_neg_inf", 0xfc00), ("d_nan", 0x7e00))]


def random_row(t, rng, K):
    blocks = []
    for b in range(K // 32):
        d = np.float16(rng.standard_normal() * 0.02).view(np.uint16)
        if rng.random() < 0.02:
            d = 0x7bff if rng.random() < 0.5 else 0xfbff
        blocks.append(weight_block(t, int(d), codes(t, rng), int(np.float16(rng.standard_normal() * 0.5).view(np.uint16))))
    return np.concatenate(blocks)


class RefDequant:
    def __init__(self, path):
        L = self.L = C.CDLL(path)

        class InitParams(C.Structure):
            _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]
        L.ggml_init.restype = C.c_void_p
        L.ggml_init.argtypes = [InitParams]
        L.ggml_free.argtypes = [C.c_void_p]
        L.ggml_free(L.ggml_init(InitParams(1 << 16, None, False)))      # fills ggml's f16 -> f32 table, which GGML_FP16_TO_FP32 reads
        for t in TYPES:
            getattr(L, f"dequantize_row_{t}").argtypes = [C.c_void_p, C.c_void_p, C.c_int64]

    def rows(self, t, W, K):
        """[n][K] f32: dequantize_row_<t> of each row of W [n][K/32 * bytes]"""
        W = np.ascontiguousarray(W, np.uint8)
        out = np.zeros((W.shape[0], K), np.float32)
        for r in range(W.shape[0]):
            getattr(self.L, f"dequantize_row_{t}")(W[r].ctypes.data, out[r].ctypes.data, K)
        return out


def main():
    orc = graft.load_oracle_bindings()
    if not orc.have_ref():
        sys.exit(f"{orc.REF_SO} is missing: run __graft_entry__.build() where the reference tree exists")
    ref = RefDequant(orc.REF_SO)
    dots = np.load(DOTS)
    rng = np.random.default_rng(20261017)
    res = {}
    for t in TYPES:
        extra = special_blocks(t, rng)
        edge = np.concatenate([dots[f"w_{t}"], np.stack([b for _, b in extra])])
        res[f"edge_{t}"] = edge
        res[f"edge_{t}_names"] = np.concatenate([dots[f"w_{t}_names"], np.array([n for n, _ in extra])])
        with np.errstate(invalid="ignore"):
            res[f"edge_deq_{t}"] = ref.rows(t, edge, 32)
        for K, n in ROWS.items():
            W = np.stack([random_row(t, rng, K) for _ in range(n)])
            res[f"rows_{t}_{K}"] = W
            res[f"rows_deq_{t}_{K}"] = ref.rows(t, W, K)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **res)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
