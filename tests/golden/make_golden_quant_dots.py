"""Regenerates tests/golden/ref_pairs/quant_dots.npz: the unmodified reference's activation quantisers and quantised block dot
products (oracle/_ref/libbark_ref.so: quantize_row_q8_0, quantize_row_q8_1 and ggml_vec_dot_{q4_0,q5_0,q8_0}_q8_0 /
ggml_vec_dot_{q4_1,q5_1}_q8_1 with nrc = 1, AVX2 build) on edge blocks.  The inputs of tests/test_quant_dots.py (oracle, CPU) and
tests/test_quant_matmul_gpu.py (kernels).

  act [A][32] f32, act_names       activation blocks: zeros, +-0, one non-zero, round-half ties at every k (amax 127), d on an f16
                                   rounding tie, d f16-subnormal, d past the f16 range, 0 < amax < 127 / FLT_MAX, +-inf, random
  q8_0_qs / q8_0_d                 quantize_row_q8_0 of each block (int8 [A][32], f16 bits [A])
  q8_1_qs / q8_1_d / q8_1_s        quantize_row_q8_1 of each block
  w_<t> [W][bytes], w_<t>_names    weight blocks of type t: d = +-0, f16-subnormal, +-65504; codes all 0 / all 15; q5 qh = 0, all
                                   ones, alternating and each single bit; q4_1 / q5_1 m negative, zero, large; q8_0 codes +-127, -128
  dot1_<t> [W][A] f32              the dot of weight block w against activation block a (n = 32)
  rows_act [R][256] f32            activation rows of 8 blocks: random with edge blocks substituted, the last block included
  rows_w_<t> [N][8 * bytes]        weight rows of 8 blocks drawn from w_<t>
  rows_dot_<t> [N][R] f32          row dots (n = 256)
  int_act [I][1024] f32            integer activations with amax 127 in every block (d_a = 1, q = x) and |block sum| <= 2048
  int_w_<t> [J][32 * bytes]        weight rows with d = 1 and small integer m
  int_dot_<t> [J][I] f32           their dots: exactly sum(q_w q_a) (+ m s) (tests/test_quant_dots.py checks that too)

NaN activations are out of scope (DESIGN.md §5).  Run once where the reference library exists:

    python tests/golden/make_golden_quant_dots.py
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "quant_dots.npz")
TYPES = ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0")
F32_MAX = np.finfo(np.float32).max


def f16(x):
    return np.uint16(np.float16(x).view(np.uint16))


def act_blocks(rng):
    """(name, 32 floats) edge blocks"""
    z = np.zeros(32, np.float32)
    out = [("zeros", z.copy())]
    sz = z.copy(); sz[1::2] = -0.0; out.append(("signed_zeros", sz))
    b = z.copy(); b[13] = -2.75; out.append(("one_nonzero", b))
    b = z.copy(); b[31] = 1e-30; out.append(("one_nonzero_small", b))
    ks = np.arange(-127, 127) + 0.5                     # x * 127 / 127 = x exactly: every round-half tie, -126.5 .. 126.5
    for i in range(0, ks.size, 31):
        b = z.copy(); b[0] = 127.0 if (i // 31) % 2 == 0 else -127.0; b[1:1 + ks[i:i + 31].size] = ks[i:i + 31]
        out.append((f"ties_{i // 31}", b))
    for name, d in (("d_tie_even_down", 1 + 2.0 ** -11), ("d_tie_even_up", 1 + 3 * 2.0 ** -11), ("d_tie_subnormal", 1.5 * 2.0 ** -24),
                    ("d_tie_to_zero", 2.0 ** -25), ("d_subnormal", 1e-6), ("d_max_f16", 65504.0), ("d_overflow_tie", 65520.0),
                    ("d_overflow", 1e7 / 127)):
        amax = np.float32(np.float64(d) * 127)
        assert name == "d_overflow" or np.float32(amax / np.float32(127)) == np.float32(d), name
        b = (rng.uniform(-1, 1, 32) * amax).astype(np.float32); b[int(rng.integers(32))] = -amax if name.endswith("up") else amax
        out.append((name, b))
    tiny = np.float32(127 / F32_MAX)                    # 127 / amax overflows to inf below this
    b = (rng.uniform(-1, 1, 32) * tiny * 0.5).astype(np.float32); b[4] = 0.0; b[9] = -0.0; out.append(("amax_below_127_over_fltmax", b))
    b = z.copy(); b[5] = np.float32(1e-45); b[6] = -0.0; out.append(("amax_denormal", b))
    b = z.copy(); b[0] = -tiny * np.float32(0.75); out.append(("amax_tiny_single", b))
    b = rng.standard_normal(32).astype(np.float32); b[7] = np.inf; out.append(("pos_inf", b))
    b = rng.standard_normal(32).astype(np.float32); b[31] = -np.inf; out.append(("neg_inf", b))
    b = rng.standard_normal(32).astype(np.float32); b[3] = np.inf; b[20] = -np.inf; out.append(("two_inf", b))
    b = z.copy(); b[0] = np.inf; out.append(("inf_among_zeros", b))
    for i in range(6):
        out.append((f"random_{i}", (rng.standard_normal(32) * (10.0 ** (i - 2))).astype(np.float32)))
    return out


def pack_nibbles(codes):
    """32 codes 0..15 -> 16 bytes: element j in the low nibble of byte j, element j + 16 in the high one"""
    c = np.asarray(codes, np.uint8)
    return (c[:16] & 15) | ((c[16:] & 15) << 4)


def weight_block(t, d, codes, m=0, qh=None):
    """one block of type t as the file stores it; codes: 32 values (q4: 0..15, q5: 0..31 (the fifth bit goes to qh), q8: -128..127)"""
    c = np.asarray(codes)
    parts = [np.array([d], "<u2").view(np.uint8)]
    if t in ("q4_1", "q5_1"):
        parts.append(np.array([m], "<u2").view(np.uint8))
    if t in ("q5_0", "q5_1"):
        if qh is None:
            qh = int(sum(((int(c[j]) >> 4) & 1) << j for j in range(32)))
        parts.append(np.array([qh], "<u4").view(np.uint8))
    parts.append(c.astype(np.int8).view(np.uint8) if t == "q8_0" else pack_nibbles(c & 15))
    return np.concatenate(parts)


def weight_blocks(t, rng):
    hi = 127 if t == "q8_0" else 31 if t.startswith("q5") else 15
    lo = -128 if t == "q8_0" else 0

    def rcodes():
        return rng.integers(lo, hi + 1, 32)

    rd = lambda: f16(rng.uniform(0.001, 0.05) * rng.choice([-1, 1]))       # noqa: E731
    rm = lambda: f16(rng.uniform(-0.5, 0.5))                               # noqa: E731
    out = []
    for name, d in (("d_zero", 0x0000), ("d_neg_zero", 0x8000), ("d_min_subnormal", 0x0001), ("d_max_subnormal", 0x03ff),
                    ("d_max", 0x7bff), ("d_neg_max", 0xfbff), ("d_one", 0x3c00)):
        out.append((name, weight_block(t, d, rcodes(), rm())))
    if t != "q8_0":
        out.append(("codes_all_0", weight_block(t, rd(), np.zeros(32, int), rm(), 0 if t.startswith("q5") else None)))
        out.append(("codes_all_15", weight_block(t, rd(), np.full(32, 15), rm(), 0 if t.startswith("q5") else None)))
    else:
        for name, v in (("codes_all_127", 127), ("codes_all_neg127", -127), ("codes_all_neg128", -128)):
            out.append((name, weight_block(t, rd(), np.full(32, v))))
        out.append(("codes_alt_127_neg128", weight_block(t, rd(), np.tile([127, -128], 16))))
    if t.startswith("q5"):
        for name, qh in (("qh_zero", 0), ("qh_ones", 0xffffffff), ("qh_0x55555555", 0x55555555), ("qh_0xaaaaaaaa", 0xaaaaaaaa)):
            out.append((name, weight_block(t, rd(), rcodes() & 15, rm(), qh)))
        for i in range(32):
            out.append((f"qh_bit_{i}", weight_block(t, rd(), np.full(32, 15 if i % 2 else 0), rm(), 1 << i)))
    if t in ("q4_1", "q5_1"):
        for name, m in (("m_negative", f16(-3.25)), ("m_zero", 0x0000), ("m_neg_zero", 0x8000), ("m_large", 0x7bff), ("m_neg_large", 0xfbff)):
            out.append((name, weight_block(t, rd(), rcodes(), m)))
    for i in range(8):
        out.append((f"random_{i}", weight_block(t, rd(), rcodes(), rm())))
    return out


def int_rows(rng, n, K):
    """integer rows: amax exactly 127 in every block, |block sum| <= 2048 (f16-exact s)"""
    a = np.zeros((n, K), np.float32)
    for r in range(n):
        for b in range(K // 32):
            while True:
                x = rng.integers(-127, 128, 32); x[int(rng.integers(32))] = 127 * rng.choice([-1, 1])
                if abs(int(x.sum())) <= 2048:
                    break
            a[r, b * 32:(b + 1) * 32] = x
    return a


def int_weights(t, rng, n, K):
    hi = 127 if t == "q8_0" else 31 if t.startswith("q5") else 15
    lo = -128 if t == "q8_0" else 0
    return np.stack([np.concatenate([weight_block(t, 0x3c00, rng.integers(lo, hi + 1, 32), f16(int(rng.integers(-8, 9))))
                                     for _ in range(K // 32)]) for _ in range(n)])


class RefQ:
    def __init__(self, path):
        L = self.L = C.CDLL(path)

        class InitParams(C.Structure):
            _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]
        L.ggml_init.restype = C.c_void_p
        L.ggml_init.argtypes = [InitParams]
        L.ggml_free.argtypes = [C.c_void_p]
        L.ggml_free(L.ggml_init(InitParams(1 << 16, None, False)))      # fills ggml's f16 -> f32 table, which GGML_FP16_TO_FP32 reads
        for k in ("q8_0", "q8_1"):
            getattr(L, f"quantize_row_{k}").argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        for t in TYPES:
            getattr(L, self.dot_name(t)).argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]

    @staticmethod
    def dot_name(t):
        return f"ggml_vec_dot_{t}_{'q8_1' if t in ('q4_1', 'q5_1') else 'q8_0'}"

    def quantize(self, x, kind, orc):
        x = np.ascontiguousarray(x, np.float32)
        y = np.zeros(x.shape[:-1] + (x.shape[-1] // 32,), orc.Q8_DTYPES[kind])
        getattr(self.L, f"quantize_row_{kind}")(x.ctypes.data, y.ctypes.data, x.size)
        return y

    def dots(self, t, W, A, orc):
        """[N][M]: weight row n against activation row m"""
        Q = self.quantize(A, orc.vec_dot_type(t), orc)
        K = A.shape[1]
        f = getattr(self.L, self.dot_name(t))
        out = np.zeros((W.shape[0], A.shape[0]), np.float32)
        s = C.c_float(0)
        for n in range(W.shape[0]):
            w = np.ascontiguousarray(W[n])
            for m in range(A.shape[0]):
                f(K, C.byref(s), 0, w.ctypes.data, 0, Q[m].ctypes.data, 0, 1)
                out[n, m] = s.value
        return out


def main():
    orc = graft.load_oracle_bindings()
    if not orc.have_ref():
        sys.exit(f"{orc.REF_SO} is missing: run __graft_entry__.build() where the reference tree exists")
    ref = RefQ(orc.REF_SO)
    rng = np.random.default_rng(20261016)
    ab = act_blocks(rng)
    act = np.stack([b for _, b in ab])
    res = {"act": act, "act_names": np.array([n for n, _ in ab])}
    for kind in ("q8_0", "q8_1"):
        y = ref.quantize(act, kind, orc)
        res[f"{kind}_qs"] = y["qs"].reshape(len(ab), 32); res[f"{kind}_d"] = y["d"].reshape(len(ab))
        if kind == "q8_1":
            res["q8_1_s"] = y["s"].reshape(len(ab))
    R, nbr = 12, 8
    rows = rng.standard_normal((R, nbr * 32)).astype(np.float32)
    finite = [i for i, (n, _) in enumerate(ab) if "inf" not in n]
    for r in range(R):                                  # edge blocks in the middle and in the last block of a row
        for b in (int(rng.integers(nbr - 1)), nbr - 1):
            rows[r, b * 32:(b + 1) * 32] = act[finite[int(rng.integers(len(finite)))]]
    res["rows_act"] = rows
    res["int_act"] = int_rows(rng, 6, 1024)
    for t in TYPES:
        wb = weight_blocks(t, rng)
        W = np.stack([b for _, b in wb])
        res[f"w_{t}"] = W; res[f"w_{t}_names"] = np.array([n for n, _ in wb])
        res[f"dot1_{t}"] = ref.dots(t, W, act, orc)
        rw = np.stack([np.concatenate([W[int(i)] for i in rng.integers(len(wb), size=nbr)]) for _ in range(24)])
        res[f"rows_w_{t}"] = rw; res[f"rows_dot_{t}"] = ref.dots(t, rw, rows, orc)
        iw = int_weights(t, rng, 5, 1024)
        res[f"int_w_{t}"] = iw; res[f"int_dot_{t}"] = ref.dots(t, iw, res["int_act"], orc)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **res)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
