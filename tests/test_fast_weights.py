"""Fast mode for f32 and quantised files: the fine model's matrices are converted once at load to f16 for the tensor cores
(bark_b200_fast_convert, csrc/fast_kernels.cu convert_f16_kernel).  The rule for every element: the f16 is the round to nearest even of
the f32 that the reference's dequantize_row_<type> computes (for f32 files, of the weight itself).

Here, on the CPU:
  * a numpy restatement of the rule (dequant, to_f16) against the unmodified reference's dequantize_row_* on edge blocks and random
    rows (tests/golden/ref_pairs/dequant.npz, tests/golden/make_golden_dequant.py), bit for bit, with the non-finite count;
  * the construction behind the exact end-to-end tests of tests/test_fast_weights_gpu.py: files whose fine matrices quantise without
    loss (bark_model_quantize) to values that are f16-exact, and the splice of one file's fine section into another file.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR

DEQ = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "dequant.npz"))
QTYPES = ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0")
BLOCK_BYTES = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}
GGML_TYPE = {"f32": 0, "f16": 1, "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}
GGML_FTYPE = {"q4_0": 2, "q4_1": 3, "q8_0": 7, "q5_0": 8, "q5_1": 9}        # enum ggml_ftype, what bark_model_quantize takes


# ---------------------------------------------------------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------------------------------------------------------
def dequant(t, W, K, fused=True):
    """dequantize_row_<t> of each row of W [n][K/32 * bytes] (the file's blocks) -> float32 [n][K].  q4_1 / q5_1: x*d + m as one
    fused multiply-add (fused=True, the pinned build's vfmadd132ps) or as a product and a sum rounded separately."""
    W = np.ascontiguousarray(W, np.uint8)
    n = W.shape[0]
    b = W.reshape(n * (K // 32), BLOCK_BYTES[t])
    d = b[:, 0:2].copy().view("<f2").astype(np.float32)                   # [B][1]
    has_m, q5 = t in ("q4_1", "q5_1"), t in ("q5_0", "q5_1")
    m = b[:, 2:4].copy().view("<f2").astype(np.float32) if has_m else None
    if t == "q8_0":
        q = b[:, 2:].view(np.int8).astype(np.float32)
        with np.errstate(invalid="ignore"):
            return (q * d).reshape(n, K)
    qs = b[:, 2 + 2 * has_m + 4 * q5:]
    q = np.concatenate([qs & 0x0F, qs >> 4], axis=1).astype(np.int64)      # element j < 16: low nibble of byte j; j >= 16: high of j - 16
    if q5:
        qh = b[:, 2 + 2 * has_m:6 + 2 * has_m].copy().view("<u4").astype(np.int64)
        q |= ((qh >> np.arange(32)) & 1) << 4
    with np.errstate(invalid="ignore", over="ignore"):
        if not has_m:
            return ((q - (16 if q5 else 8)).astype(np.float32) * d).reshape(n, K)
        if fused:                                                           # q d + m exactly in float64 (< 2^22, a multiple of 2^-48), one rounding to f32
            return (q.astype(np.float64) * d.astype(np.float64) + m.astype(np.float64)).astype(np.float32).reshape(n, K)
        return (q.astype(np.float32) * d + m).reshape(n, K)


def to_f16(x32):
    """f32 -> f16, round to nearest even (numpy's float32 -> float16 conversion rounds correctly)"""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x32, np.float32).astype(np.float16)


def non_finite(h):
    return int((~np.isfinite(np.asarray(h, np.float16))).sum())


def same_f16(a, b):
    """equal f16 bits, NaN matching any NaN"""
    a = np.asarray(a, np.float16); b = np.asarray(b, np.float16)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint16)[~nan], b.view(np.uint16)[~nan])


def fixture_cases(t):
    """(name, blocks [n][K/32 * bytes], K, reference f32 [n][K]) of dequant.npz"""
    yield "edge", DEQ[f"edge_{t}"], 32, DEQ[f"edge_deq_{t}"]
    for K in (768, 4096):
        yield f"rows_{K}", DEQ[f"rows_{t}_{K}"], K, DEQ[f"rows_deq_{t}_{K}"]


@pytest.mark.parametrize("t", QTYPES)
def test_restatement_matches_the_reference(t):
    """The restated f32 equals dequantize_row_<t>'s bit for bit (NaN where it is NaN), so its f16 is the rule's f16."""
    for name, W, K, ref in fixture_cases(t):
        got = dequant(t, W, K)
        nan = np.isnan(ref)
        assert np.array_equal(np.isnan(got), nan), (t, name)
        assert np.array_equal(got.view(np.uint32)[~nan], ref.view(np.uint32)[~nan]), (t, name, int((got != ref).sum()))
        assert same_f16(to_f16(got), to_f16(ref)), (t, name)


@pytest.mark.parametrize("t", ("q4_1", "q5_1"))
def test_fused_and_separate_forms_agree(t):
    """q d is exact in f32 (an integer below 32 times an f16 value), so whether the build contracts q d + m into an FMA cannot change
    the value: both forms equal the reference on every fixture element."""
    for name, W, K, ref in fixture_cases(t):
        a, b = dequant(t, W, K, fused=True), dequant(t, W, K, fused=False)
        nan = np.isnan(ref)
        assert np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan]), (t, name)


@pytest.mark.parametrize("t", QTYPES)
def test_fixture_covers_the_edges(t):
    """The fixture has what the rule has to get right: signed zeros, f16-subnormal results, results at and past the f16 range
    (d = +-65504 with a large code), and NaN / inf scales; the non-finite count of the restatement counts exactly those."""
    names = list(DEQ[f"edge_{t}_names"])
    for n in ("d_zero", "d_neg_zero", "d_min_subnormal", "d_max_subnormal", "d_max", "d_neg_max", "d_inf", "d_neg_inf", "d_nan"):
        assert n in names, (t, n)
    ref = DEQ[f"edge_deq_{t}"]
    h = to_f16(ref)
    big = np.abs(ref.astype(np.float64)) >= 65520
    assert non_finite(h) == int((big | ~np.isfinite(ref)).sum())
    for n in ("d_inf", "d_neg_inf", "d_nan"):
        assert non_finite(h[names.index(n)]) == 32, (t, n)
    assert non_finite(h[names.index("d_max")]) > 0
    if t not in ("q4_1", "q5_1"):                                  # with an offset m, results near zero need q d = -m exactly
        assert ((np.abs(ref) < 2.0 ** -14) & (ref != 0)).any(), "no f16-subnormal result"
        assert (np.signbit(ref) & (ref == 0)).any(), "no -0 result"
    for K in (768, 4096):
        r = DEQ[f"rows_deq_{t}_{K}"]
        assert DEQ[f"rows_{t}_{K}"].shape[0] % 2 == 1
        assert non_finite(to_f16(r)) == int((np.abs(r.astype(np.float64)) >= 65520).sum())


# ---------------------------------------------------------------------------------------------------------------------------
# exact end-to-end files: lossless quantisation to f16-exact values, and the section splice
# ---------------------------------------------------------------------------------------------------------------------------
D_EXP = {"q8_0": -12, "q4_0": -8, "q4_1": -8, "q5_0": -9, "q5_1": -9, "f32": -6}


def lossless_values(t, shape, rng):
    """float32 array of `shape` (last axis a multiple of 32) whose every value is f16-exact and which bark_model_quantize's
    quantize_row_<t> keeps exactly: per block of 32 a power-of-two scale d and integer codes with the block's extreme code present,
    so that the quantiser finds d again (q8_0: a code +-127; q4_0 / q5_0: a code 0, value -8 d / -16 d, the unique largest magnitude;
    q4_1 / q5_1: codes 0 and 15 / 31 with m an integer multiple of d).  "f32": any f16 values."""
    n = int(np.prod(shape))
    nb = n // 32
    if t == "f32":
        return (rng.standard_normal(n) * 0.02).astype(np.float16).astype(np.float32).reshape(shape)
    d = 2.0 ** (D_EXP[t] + rng.integers(-1, 2, (nb, 1)))
    hi = {"q8_0": 127, "q4_0": 15, "q4_1": 15, "q5_0": 31, "q5_1": 31}[t]
    lo = -127 if t == "q8_0" else 0
    c = rng.integers(lo, hi + 1, (nb, 32))
    p = rng.integers(0, 32, nb)
    rows = np.arange(nb)
    if t == "q8_0":
        c[rows, p] = rng.choice([-127, 127], nb)
        v = c * d
    elif t in ("q4_0", "q5_0"):
        c[rows, p] = 0
        v = (c - (hi + 1) // 2) * d
    else:
        c[rows, p] = 0
        c[rows, (p + 1 + rng.integers(0, 31, nb)) % 32] = hi
        v = (c + rng.integers(-hi, 1, (nb, 1))) * d
    return v.astype(np.float32).reshape(shape)


def fine_matrices(cfg):
    """name -> numpy shape of every fine-model tensor fast mode converts (bark.cpp_b200/weights.py names), the wte tables too: they
    are quantised with the rest, and the exact comparison needs them lossless as well"""
    E, L, V = cfg.fine.n_embd, cfg.fine.n_layer, cfg.fine_vocab
    out = {f"model/wte/{i}": (V, E) for i in range(8)}
    out.update({f"model/lm_head/{i}": (V, E) for i in range(7)})
    for l in range(L):
        out.update({f"model/h{l}/attn/c_attn/w": (3 * E, E), f"model/h{l}/attn/c_proj/w": (E, E),
                    f"model/h{l}/mlp/c_fc/w": (4 * E, E), f"model/h{l}/mlp/c_proj/w": (E, 4 * E)})
    return out


def lossless_overrides(cfg, t, seed=7):
    rng = np.random.default_rng([seed, GGML_TYPE[t]])
    return {"fine/" + n: lossless_values(t, s, rng) for n, s in fine_matrices(cfg).items()}


TYPE_SIZE = {0: (1, 4), 1: (1, 2), 2: (32, 18), 3: (32, 20), 6: (32, 22), 7: (32, 24), 8: (32, 34)}   # ggml type: (elements, bytes) per block


def sections(path):
    """(file bytes, section bounds, tensors): bounds [0, vocab end, text end, coarse end, fine end, file end]; tensors[s] maps each
    tensor name of GPT section s (0 text, 1 coarse, 2 fine) to (ggml type, ne, data offset, data bytes)."""
    b = open(path, "rb").read()
    i32 = lambda o, n=1: np.frombuffer(b, "<i4", n, o)              # noqa: E731
    o = 8
    for _ in range(int(i32(4)[0])):
        o += 4 + int(np.frombuffer(b, "<u4", 1, o)[0])
    bounds, tensors = [0, o], []
    for _ in range(3):
        n_t = int(i32(o + 40)[0])
        o += 44
        ts = {}
        for _ in range(n_t):
            n_dims, ln, tt = (int(v) for v in i32(o, 3))
            ne = tuple(int(v) for v in i32(o + 12, n_dims))
            o += 12 + 4 * n_dims
            name = b[o:o + ln].decode()
            o += ln
            per, nbytes = TYPE_SIZE[tt]
            size = int(np.prod(ne)) // per * nbytes
            ts[name] = (tt, ne, o, size)
            o += size
        tensors.append(ts)
        bounds.append(o)
    bounds.append(len(b))
    return b, bounds, tensors


def splice_fine(base, fine_from, out):
    """`base` with its fine-model section replaced by `fine_from`'s: the text and coarse models and the codec stay as in base."""
    b, bb, _ = sections(base)
    f, fb, _ = sections(fine_from)
    with open(out, "wb") as fo:
        fo.write(b[:bb[3]] + f[fb[3]:fb[4]] + b[bb[4]:])
    return out


def fine_values(path, name):
    """float32 values of fine tensor `name` as the file holds them, quantised types through the restatement"""
    b, _, ts = sections(path)
    tt, ne, o, size = ts[2][name]
    raw = np.frombuffer(b, np.uint8, size, o)
    t = {v: k for k, v in GGML_TYPE.items()}[tt]
    if t in ("f32", "f16"):
        return raw.view("<f4" if t == "f32" else "<f2").astype(np.float32).reshape(ne[1], ne[0]), t
    return dequant(t, raw.reshape(ne[1], -1), ne[0]), t


def exact_pair(pkg, weights_mod, cfg_name, t, d):
    """(f16 file, file of type t) whose fine models hold the same f16-exact values, in directory d; every other section of the two
    files is the same bytes, the f16 file's."""
    cfg16 = weights_mod.CONFIGS[cfg_name](weights_mod.F16)
    ov = lossless_overrides(cfg16, t)
    f16 = weights_mod.write_weights(os.path.join(d, f"{cfg_name}_exact_{t}_f16.bin"), cfg16, overrides=ov)
    src = os.path.join(d, f"{cfg_name}_exact_{t}_src.bin")
    if t == "f32":
        weights_mod.write_weights(src, weights_mod.CONFIGS[cfg_name](weights_mod.F32), overrides=ov)
    else:
        assert pkg.lib().bark_model_quantize(f16.encode(), src.encode(), GGML_FTYPE[t])
    return f16, splice_fine(f16, src, os.path.join(d, f"{cfg_name}_exact_{t}.bin"))


@pytest.mark.parametrize("t", ("f32",) + QTYPES)
def test_exact_files_hold_the_f16_values(pkg, weights_mod, tmp_path, t):
    """Every fine tensor of the spliced file of type t (bark_model_quantize's output for the quantised types) dequantises to exactly
    the f16 file's values, which are f16-exact: the premise of the bit-for-bit fast-mode comparisons on the GPU.  The text and coarse
    sections and the codec are the f16 file's bytes."""
    f16, path = exact_pair(pkg, weights_mod, "tiny", t, str(tmp_path))
    b16, bounds16, ts16 = sections(f16)
    b, bounds, ts = sections(path)
    assert b[:bounds[3]] == b16[:bounds16[3]] and b[bounds[4]:] == b16[bounds16[4]:]
    assert set(ts[2]) == set(ts16[2])
    mats = fine_matrices(weights_mod.tiny())
    assert len(mats) == 8 + 7 + 4 * weights_mod.tiny().fine.n_layer and set(mats) <= set(ts[2])
    for name in mats:
        got, tt = fine_values(path, name)
        want, t16 = fine_values(f16, name)
        assert tt == t and t16 == "f16", (name, tt, t16)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, int((got != want).sum()))
        assert np.array_equal(want.astype(np.float16).astype(np.float32), want)
