"""FAST MODE (BARK_B200_MODE=fast): wgmma GEMM + flash-style attention for the fine model's 1024-row passes (csrc/fast_kernels.cu).

Tensor cores cannot replay the reference's 32 IEEE FMA chains, so this path is validated the way SURVEY.md §7 step 6 prescribes:
  * the kernels on inputs whose answer is exact, bit for bit: integer-valued GEMM operands through every epilogue and tile width,
    every finite f16 input of the GELU epilogue against the reference's table, attention with a uniform, a single and a tied maximum;
  * the kernels on random inputs against float64, within error bounds derived in the tests' docstrings;
  * teacher-forced fine passes against the oracle: max |dlogit|, top-1 agreement and the CDF-flip rate (same uniforms, same inputs),
    and bit-identical logits when the same pass runs twice;
  * a whole generation: semantic / coarse ids stay bit-identical (those stages run the parity kernels), fine ids may differ.
The constructions behind the exact answers are checked on the CPU by the tests here that carry no gpu mark.
The parity path stays the contract (tests/test_parity_gpu.py); numbers measured here are printed for DESIGN.md / profiles.
"""
import functools
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR

gpu = pytest.mark.gpu

GEMM_RTOL, GEMM_ATOL = 2e-3, 2e-2          # f16 operands, f32 accumulation in a different order than numpy's
ATT_ATOL = 6e-3                            # probabilities are rounded to f16 before P.V; outputs are O(0.1)
# Teacher-forced fine passes, nn = 2..7, measured on an H100 SXM (700 W limit): worst max |dlogit| tiny 0.0053, mini 0.0073,
# wide 0.0151 (wider rows sum more f16-rounded terms); worst top-1 agreement 99.71 %.  The bounds allow ~2.7x the logit error and
# ~3x the top-1 disagreement.
MAX_DLOGIT = {"tiny": 0.015, "mini": 0.02, "wide": 0.04}
MIN_TOP1 = 0.992

BNS = [0, 64, 128, 256]                    # 0: the tile width the cost model picks for the shape on this device
U32 = 2.0 ** -23                           # f32 unit roundoff when the accumulator truncates instead of rounding to nearest


# ---------------------------------------------------------------------------------------------------------------------------
# GELU: the parity path's definition (epilogue.cuh gelu_lookup) and the pass criterion of the fast epilogue
# ---------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def gelu_table():
    return np.load(os.path.join(GOLDEN_DIR, "gelu_table_f16.npz"))["table"]


def gelu_expected(x16):
    """The parity path's GELU of f16 inputs: 0 for x <= -10, x for x >= 10, the reference's table in between."""
    x16 = np.asarray(x16, np.float16)
    x = x16.astype(np.float32)
    t = gelu_table()[x16.view(np.uint16)].view(np.float16)
    return np.where(x <= -10, np.float16(0), np.where(x >= 10, x16, t)).astype(np.float16)


def f16_ulps(a, b):
    """Distance in f16 steps (+0 and -0 are the same point)."""
    def ordered(h):
        u = np.asarray(h, np.float16).view(np.uint16).astype(np.int64)
        return np.where(u & 0x8000, -(u & 0x7fff), u)
    return np.abs(ordered(a) - ordered(b))


def gelu_ok(got, want):
    """Within one f16 ulp, or within 2^-22: the reference's table is built with float tanhf, whose 1 + tanh is quantised near
    tanh = -1 (steps of 2^-24, so ~2^-22 absolute after the factor 0.5 x for |x| < 10)."""
    got = np.asarray(got, np.float16); want = np.asarray(want, np.float16)
    close = np.abs(got.astype(np.float64) - want.astype(np.float64)) <= 2.0 ** -22
    return np.isfinite(got) & ((f16_ulps(got, want) <= 1) | close)


def gelu64(x):
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * x * (1.0 + 0.044715 * x * x)))


def finite_f16():
    x = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)
    return x[np.isfinite(x)]


def _f32(a):
    return np.asarray(a, np.float32)


def gelu_model_tanh(x16, rel=0.0):
    """0.5 x (1 + tanh y) in float32 with a float tanh whose relative error is `rel` (clamped to [-1, 1]), rounded to f16."""
    x = _f32(x16)
    y = _f32(0.7978845608028654) * x * (_f32(1) + _f32(0.044715) * x * x)
    t = np.clip(_f32(np.tanh(y.astype(np.float64)) * (1.0 + rel)), -1, 1)
    return (_f32(0.5) * x * (_f32(1) + t)).astype(np.float16)


def gelu_model_sigmoid(x16, rel=0.0):
    """x / (1 + e^(-2y)) with relative error `rel`, rounded to f16 (gelu_fast's form)."""
    x = np.asarray(x16, np.float64)
    y = np.sqrt(2.0 / np.pi) * x * (1.0 + 0.044715 * x * x)
    with np.errstate(over="ignore"):
        return (x / (1.0 + np.exp(-2.0 * y)) * (1.0 + rel)).astype(np.float32).astype(np.float16)


def test_gelu_criterion_separates_the_models():
    """The criterion accepts an exact float tanh and the sigmoid form at 2^-20 relative error, and rejects a tanh at the ~2^-11
    relative error PTX documents for tanh.approx.f32: near tanh = -1 that error is amplified by the cancellation in 1 + tanh."""
    x = finite_f16()
    want = gelu_expected(x)
    assert x.size == 63488
    assert gelu_ok(gelu_model_tanh(x), want).all()
    for rel in (2.0 ** -20, -2.0 ** -20):
        assert gelu_ok(gelu_model_sigmoid(x, rel), want).all()
    rejected = max(int((~gelu_ok(gelu_model_tanh(x, rel), want)).sum()) for rel in (2.0 ** -11, -2.0 ** -11))
    assert rejected > 1000, rejected


@gpu
@pytest.mark.parametrize("N", [2, 1])        # 2: the paired f16 store, 1: the scalar store
def test_gelu_epilogue_every_f16_input(pkg, N):
    """GELU16 GEMM with K = 64, A[m][0] = the m-th finite f16 value and W rows = e0: the accumulator holds x exactly, so the epilogue
    sees all 63 488 finite f16 inputs and must reproduce the parity path's GELU within `gelu_ok`.  The earlier 0.5 x (1 + tanh.approx y)
    form failed on an H100 for 335 inputs, by up to 15 ulps (x = -3.582)."""
    x = finite_f16()
    A = np.zeros((x.size, 64), np.float16); A[:, 0] = x
    W = np.zeros((N, 64), np.float16); W[:, 0] = 1
    out = pkg.fast_gemm(A, W, "gelu16")
    want = gelu_expected(x)
    for col in range(N):
        bad = np.flatnonzero(~gelu_ok(out[:, col], want))
        worst = bad[np.argsort(-f16_ulps(out[bad, col], want[bad]))[:5]] if bad.size else bad
        assert bad.size == 0, (f"{bad.size} inputs off by more than 1 ulp / 2^-22, e.g. "
                               + ", ".join(f"x={float(x[i]):.6g}: {float(out[i, col]):.6g} vs {float(want[i]):.6g}" for i in worst))
    print(f"gelu16 N={N}: max {int(f16_ulps(out[:, 0], want).max())} f16 ulps from the table")


# ---------------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------------
PRODUCTION = [c for E in (128, 256, 768, 1024)
              for c in ((1024, 3 * E, E, "qkv16"), (1024, E, E, "resid"), (1024, 4 * E, E, "gelu16"), (1024, E, 4 * E, "resid"),
                        (1024, 1056, E, "f32"))]      # 1056: the lm_head width, a partial last column tile at every BN
GEMM_CASES = PRODUCTION + [(257, 2304, 768, "f32"), (128, 64, 64, "f32"), (100, 96, 128, "f32"), (1024, 1024, 4096, "f32")]
EDGES = [(M, N, K) for M in (1, 127, 129, 1000) for N in (1, 3, 63, 65, 257, 1056) for K in (64, 512, 576, 4096)]
INT_MAX = 4                                # |a|, |w| <= 4: |partial sums| <= 16 K <= 2^16 for K <= 4096


@functools.lru_cache(maxsize=2)
def gemm_operands(M, N, K, data):
    """A [M][K], W [N][K] f16, a residual [M][N] f32 and the product in float64.  "int": integers in [-4, 4], so every product is
    exact and every partial sum is an integer below 2^20: any f32 accumulation order (and any accumulator of >= 21 bits) gives the
    same integer, and the float64 product is exact too.  "random": N(0, 1/4) operands."""
    rng = np.random.default_rng([M, N, K, data == "int"])
    if data == "int":
        A = rng.integers(-INT_MAX, INT_MAX + 1, (M, K)).astype(np.float16)
        W = rng.integers(-INT_MAX, INT_MAX + 1, (N, K)).astype(np.float16)
    else:
        A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
        W = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    R = (rng.standard_normal((M, N)) * 3).astype(np.float32)
    A64, W64 = A.astype(np.float64), W.astype(np.float64)
    return A, W, R, A64 @ W64.T, np.abs(A64) @ np.abs(W64).T


def run_gemm(pkg, A, W, epi, bn, R):
    out, ran = pkg.fast_gemm(A, W, epi, bn, resid=R if epi == "resid" else None, return_bn=True)
    assert ran in (64, 128, 256) and (bn == 0 or ran == bn), (bn, ran)
    return out, ran


def check_gemm_exact(pkg, M, N, K, epi, bn):
    A, W, R, ref, _ = gemm_operands(M, N, K, "int")
    what = f"{epi} {M}x{N}x{K} bn={bn}"
    out, ran = run_gemm(pkg, A, W, epi, bn, R)
    if epi == "f32":
        want = ref.astype(np.float32)
        assert np.array_equal(out, want), f"{what}: {int((out != want).sum())} elements differ"
    elif epi == "resid":
        want = R + ref.astype(np.float32)                               # one IEEE f32 add, as in the kernel
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), f"{what}: {int((out != want).sum())} elements differ"
    elif epi == "qkv16":
        qk, vt = out
        c0 = 2 * N // 3
        want_qk = ref[:, :c0].astype(np.float32).astype(np.float16)    # round to nearest even, as __float2half_rn
        want_vt = ref[:, c0:].T.astype(np.float32).astype(np.float16)
        assert np.array_equal(qk.view(np.uint16), want_qk.view(np.uint16)), f"{what}: Q/K block, {int((qk != want_qk).sum())} elements differ"
        assert np.array_equal(vt.view(np.uint16), want_vt.view(np.uint16)), f"{what}: V^T block, {int((vt != want_vt).sum())} elements differ"
    else:
        ok = gelu_ok(out, gelu_expected(ref.astype(np.float32).astype(np.float16)))
        assert ok.all(), f"{what}: {int((~ok).sum())} GELU outputs off, first at {np.argwhere(~ok)[0]}"
    return ran


def check_gemm_random(pkg, M, N, K, epi, bn):
    """Random operands against float64.  The f16 products are exact in f32, and each of the < K f32 additions of one output loses
    at most 2^-23 of the running magnitude (one ulp: truncation, the worst rounding an accumulator may use), so
        |acc - ref| <= E = K 2^-23 (|A| |W|^T)
    elementwise.  Outputs add their own rounding on top:
        f32     |out - ref|       <= E
        resid   |out - (R + ref)| <= E + 2^-24 (|R + ref| + E)                 one f32 add
        qkv16   |out - ref|       <= E + 2^-11 (|ref| + E) + 2^-25             f16 rounding, subnormal half-step 2^-25
        gelu16  |out - G(ref)|    <= 1.13 D (1 + 2^-9) + 2^-9 |G(ref)| + 2^-21
    with G the float64 GELU, D the qkv16 bound (the epilogue rounds the sum to f16 first), 1.13 the largest slope of G, and 2^-9 and
    2^-21 covering the table's half ulp plus the one ulp or 2^-22 the GELU test above allows."""
    A, W, R, ref, mag = gemm_operands(M, N, K, "random")
    what = f"{epi} {M}x{N}x{K} bn={bn}"
    out, ran = run_gemm(pkg, A, W, epi, bn, R)
    E = K * U32 * mag
    D = E + 2.0 ** -11 * (np.abs(ref) + E) + 2.0 ** -25
    if epi == "f32":
        got, want, bound = out.astype(np.float64), ref, E
    elif epi == "resid":
        want = R.astype(np.float64) + ref
        got, bound = out.astype(np.float64), E + 2.0 ** -24 * (np.abs(want) + E)
    elif epi == "qkv16":
        got, want, bound = np.concatenate([out[0], out[1].T], axis=1).astype(np.float64), ref, D
    else:
        want = gelu64(ref)
        got, bound = out.astype(np.float64), 1.13 * D * (1 + 2.0 ** -9) + 2.0 ** -9 * np.abs(want) + 2.0 ** -21
    err = np.abs(got - want)
    assert np.isfinite(got).all(), f"{what}: {int((~np.isfinite(got)).sum())} non-finite outputs"
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} outputs outside the bound; worst {worst}: err {err[worst]:.3g} > {bound[worst]:.3g}"
    return ran


@gpu
@pytest.mark.parametrize("M,N,K", [(1024, 3072, 768), (1024, 2304, 768), (1024, 768, 768), (1024, 768, 3072), (1024, 1056, 768), (257, 2304, 768), (128, 64, 64), (100, 96, 128), (1024, 1024, 4096)])
def test_umma_gemm_matches_numpy(pkg, M, N, K):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
    W = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    C = pkg.fast_gemm(A, W)
    ref = A.astype(np.float32) @ W.astype(np.float32).T
    assert np.isfinite(C).all()
    err = np.abs(C - ref)
    assert np.allclose(C, ref, rtol=GEMM_RTOL, atol=GEMM_ATOL), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}, ref {ref.flat[err.argmax()]:.4f}"


def test_gemm_integer_operands_stay_exact():
    """The premise of the exact GEMM tests: integer operands of magnitude <= 4 keep every partial sum an integer below 2^20."""
    K = max(k for _, _, k in EDGES)
    assert INT_MAX * INT_MAX * K < 2 ** 20
    A, W, _, ref, mag = gemm_operands(129, 65, 576, "int")
    assert np.array_equal(A, np.round(A)) and np.abs(A).max() <= INT_MAX and np.abs(W).max() <= INT_MAX
    assert mag.max() < 2 ** 20 and np.array_equal(ref, np.round(ref))


@gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("data", ["int", "random"])
@pytest.mark.parametrize("M,N,K,epi", GEMM_CASES)
def test_gemm_matches_reference(pkg, M, N, K, epi, data, bn):
    """The fine pass's GEMMs (QKV, attention and MLP projections, fc with GELU, lm_head) at the widths of every model, with each tile width."""
    ran = (check_gemm_exact if data == "int" else check_gemm_random)(pkg, M, N, K, epi, bn)
    if bn == 0 and data == "int":
        print(f"cost model: {M}x{N}x{K} -> BN {ran}")


@gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("M,N,K", EDGES)
def test_gemm_edges_exact(pkg, M, N, K, bn):
    """Partial row tiles (and rows r0 + 8 past M), odd N (the scalar stores), partial column tiles, a single k-block and K = 4096
    (the mbarrier ring wraps many times), through every epilogue (QKV16 where N % 6 == 0)."""
    for epi in ("f32", "resid", "gelu16") + (("qkv16",) if N % 6 == 0 else ()):
        check_gemm_exact(pkg, M, N, K, epi, bn)


@gpu
def test_gemm_hook_rejects_bad_arguments(pkg):
    """Fails loudly on an unsupported tile width, K % 64 != 0 and a QKV16 width that is not a multiple of 6."""
    A = np.zeros((4, 64), np.float16); W = np.zeros((6, 64), np.float16)
    with pytest.raises(RuntimeError):
        pkg.fast_gemm(A, W, "f32", bn=32)
    with pytest.raises(RuntimeError):
        pkg.fast_gemm(np.zeros((4, 48), np.float16), np.zeros((6, 48), np.float16))
    with pytest.raises(AssertionError):
        pkg.fast_gemm(A, W[:4], "qkv16")


# ---------------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------------
ATT_SHAPES = [(n, H) for n in (128, 256, 1024) for H in (1, 12, 16)]
C_Q = 9                                    # q = 9 k_t: target score 9 * 64 / 8 = 72
MARGIN = 25.0                              # in units of score / 8: other P < e^-25, which rounds to 0 in f16 (smallest step 2^-24)
DOT_MAX = 64 - int(np.ceil(8 * MARGIN / C_Q))     # largest dot product of two different keys that keeps the margin


def pm1_keys(rng, n, H):
    """[H][n][64] random +-1 keys; within a head, no two different keys have a dot product above DOT_MAX."""
    k = rng.choice(np.array([-1, 1], np.int64), size=(H, n, 64))
    for h in range(H):
        while True:
            d = k[h] @ k[h].T
            np.fill_diagonal(d, 0)
            bad = np.unique(np.argwhere(d > DOT_MAX)[:, 0])
            if bad.size == 0:
                break
            k[h, bad] = rng.choice(np.array([-1, 1], np.int64), size=(bad.size, 64))
    return k


def targets(n, H, n_keys):
    """t[h][i]: the key query i of head h points at.  389 is odd, so within 64 consecutive queries (one warpgroup's half of a query tile)
    the targets spread over every key block."""
    i = np.arange(n)
    return np.stack([(i * 389 + 131 * h + 7) % n_keys for h in range(H)])


def heads_to_rows(x):
    """[H][n][64] -> [n][64 H]"""
    H, n, D = x.shape
    return np.ascontiguousarray(x.transpose(1, 0, 2).reshape(n, H * D))


def peaked_case(n, H, ties):
    """Keys, queries and values with one (ties=False) or two equal (ties=True) maximal scores per row, all other scores >= MARGIN below.
    ties: the keys at j and j + n/2 are equal (different key blocks once n >= 256), the query targets j < n/2 and the answer is
    the mean of the two values; values are then positive so that the mean is not 0."""
    rng = np.random.default_rng([n, H, ties])
    half = n // 2 if ties else n
    kk = pm1_keys(rng, half, H)
    if ties:
        kk = np.concatenate([kk, kk], axis=1)
    t = targets(n, H, half)
    qq = np.stack([C_Q * kk[h, t[h]] for h in range(H)])
    mag = rng.integers(1, 17, (H, n, 64))
    vv = mag if ties else mag * rng.choice(np.array([-1, 1]), size=(H, n, 64))
    if ties:
        want = np.stack([(vv[h, t[h]] + vv[h, t[h] + half]) / 2 for h in range(H)])
    else:
        want = np.stack([vv[h, t[h]] for h in range(H)])
    return (heads_to_rows(qq).astype(np.float16), heads_to_rows(kk).astype(np.float16), heads_to_rows(vv).astype(np.float16),
            heads_to_rows(want).astype(np.float16), kk, qq, t)


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("n,H", ATT_SHAPES)
def test_peaked_attention_construction(n, H, ties):
    """Every row's maximal score (or both tied ones) sits >= MARGIN above all others, and the targets of every 64-query half of every
    128-query tile fall in every key block (so a late maximum makes each earlier block the running maximum first)."""
    _, _, _, _, kk, qq, t = peaked_case(n, H, ties)
    half = n // 2 if ties else n
    for h in range(H):
        s = (qq[h] @ kk[h].T) / 8.0
        top = s[np.arange(n), t[h]]
        assert np.all(top == C_Q * 64 / 8)
        s[np.arange(n), t[h]] = -np.inf
        if ties:
            assert np.array_equal(s[np.arange(n), t[h] + half], top)
            s[np.arange(n), t[h] + half] = -np.inf
        assert (top - s.max(1)).min() >= MARGIN
        blocks = t[h] // 128
        for r0 in range(0, n, 64):
            assert set(blocks[r0:r0 + 64]) == set(range(half // 128)) or half < 128, (h, r0)


@gpu
@pytest.mark.parametrize("n,H", ATT_SHAPES)
def test_attention_uniform(pkg, n, H):
    """q = 0: every P is 1 and l = n (a power of two), so the output is f16(mean of v) exactly: V^T addressing, the head mapping and
    every key block counted once."""
    rng = np.random.default_rng([n, H])
    k = rng.standard_normal((n, 64 * H)).astype(np.float16)
    v = rng.integers(-16, 17, (n, 64 * H)).astype(np.float16)
    out = pkg.fast_attention(np.zeros_like(k), k, v, H)
    want = np.broadcast_to((v.astype(np.float64).sum(0) / n).astype(np.float32).astype(np.float16), out.shape)
    assert np.array_equal(out.view(np.uint16), want.view(np.uint16)), f"{int((out != want).sum())} elements differ, first at {np.argwhere(out != want)[0]}"


@gpu
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("n,H", ATT_SHAPES)
def test_attention_peaked(pkg, n, H, ties):
    """One maximal key per row (the output is its value, exactly), or two equal keys in different blocks (the mean of their values):
    the online soft_max's rescale by alpha of o and l, alpha = 1 when a later block ties, and the combination across blocks.  Earlier
    blocks leave at most n 16 e^-25 < 2^-14 behind, which the f16 rounding of a value of magnitude >= 1 removes."""
    q, k, v, want, *_ = peaked_case(n, H, ties)
    out = pkg.fast_attention(q, k, v, H)
    bad = np.argwhere(out.view(np.uint16) != want.view(np.uint16))
    assert bad.size == 0, f"{len(bad)} elements differ, first at {bad[0]}: {float(out[tuple(bad[0])])} vs {float(want[tuple(bad[0])])}"


def attention64(q, k, v, H):
    """float64 soft_max(Q K^T / 8) V per head, and P |V| (the convex combination of |v|) for the error bound."""
    n, E = q.shape
    out, pv = np.zeros((n, E)), np.zeros((n, E))
    for h in range(H):
        c = slice(64 * h, 64 * h + 64)
        s = q[:, c].astype(np.float64) @ k[:, c].astype(np.float64).T / 8.0
        p = np.exp(s - s.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        out[:, c] = p @ v[:, c].astype(np.float64)
        pv[:, c] = p @ np.abs(v[:, c].astype(np.float64))
    return out, pv


@gpu
@pytest.mark.parametrize("n,H", ATT_SHAPES)
def test_attention_random_large_scales(pkg, n, H):
    """q and k rows scaled by up to 8, so exp underflows for most keys, against float64.  Error sources, per output element:
      * scores: 64 exact f16 products summed in f32, each score off by <= d = 64 2^-23 (|q| |k|) / 8, so every weight by a factor
        within e^(+-2 max d);
      * P rounded to f16 before P V, and l summed from the rounded P: weights off by <= 2^-10 relative, plus 2^-25 absolute per key
        for subnormal P (numerator and l, and l >= 1): n 2^-24 max|v|;
      * exp2 and the f32 sums of o (n terms) and l: (2^-20 + n 2^-23) relative;
      * the f16 output: 2^-11 |ref| + 2^-25.
    So |out - ref| <= (2^-10 + e^(2d) - 1 + 2^-20 + n 2^-23) (P |V|) + (2^-11 + n 2^-23) |ref| + n 2^-24 max|v| + 2^-25."""
    rng = np.random.default_rng([n, H, 8])
    q = (rng.standard_normal((n, 64 * H)) * rng.uniform(1, 8, (n, 1))).astype(np.float16)
    k = (rng.standard_normal((n, 64 * H)) * rng.uniform(1, 8, (n, 1))).astype(np.float16)
    v = rng.standard_normal((n, 64 * H)).astype(np.float16)
    out = pkg.fast_attention(q, k, v, H).astype(np.float64)
    ref, pv = attention64(q, k, v, H)
    d = np.zeros((n, 64 * H))
    for h in range(H):
        c = slice(64 * h, 64 * h + 64)
        d[:, c] = (64 * U32 * (np.abs(q[:, c].astype(np.float64)) @ np.abs(k[:, c].astype(np.float64)).T) / 8.0).max(1, keepdims=True)
    vmax = np.abs(v.astype(np.float64)).max()
    bound = (2.0 ** -10 + np.expm1(2 * d) + 2.0 ** -20 + n * U32) * pv + (2.0 ** -11 + n * U32) * np.abs(ref) + n * 2.0 ** -24 * vmax + 2.0 ** -25
    err = np.abs(out - ref)
    assert np.isfinite(out).all()
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert (err <= bound).all(), f"{int((err > bound).sum())} outside the bound; worst {worst}: err {err[worst]:.3g} > {bound[worst]:.3g}"


def attention_ref(q, k, v, H):
    n, E = q.shape
    D = E // H
    out = np.zeros((n, E), np.float32)
    for h in range(H):
        s = (q[:, h * D:(h + 1) * D].astype(np.float32) @ k[:, h * D:(h + 1) * D].astype(np.float32).T) / np.sqrt(D)
        p = np.exp(s - s.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        out[:, h * D:(h + 1) * D] = p @ v[:, h * D:(h + 1) * D].astype(np.float32)
    return out


@gpu
@pytest.mark.parametrize("n,E,H", [(256, 128, 2), (384, 128, 2), (1024, 768, 12), (512, 1024, 16)])
def test_flash_attention_matches_numpy(pkg, n, E, H):
    rng = np.random.default_rng(n + E)
    q, k, v = ((rng.standard_normal((n, E)) * s).astype(np.float16) for s in (1.5, 1.5, 1.0))
    out = pkg.fast_attention(q, k, v, H).astype(np.float32)
    ref = attention_ref(q, k, v, H)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    assert err.max() < ATT_ATOL, f"max err {err.max():.5f} (ref magnitude {np.abs(ref).max():.3f}) at {np.unravel_index(err.argmax(), err.shape)}"


# ---------------------------------------------------------------------------------------------------------------------------
# whole fast fine passes
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("config", ["tiny", "mini", "wide"])
def test_fast_fine_passes_teacher_forced(pkg, orc, weights_file, monkeypatch, config):
    path = weights_file(config, "f16")
    o = orc.Oracle(path, seed=0, n_steps=16)
    ref = o.generate("hello world")
    T = ref["fine"].shape[0]
    buf = np.full((8, 1024), 1024, np.int32)
    buf[:, :T] = ref["fine"].T                                   # the oracle's own codes: every pass sees the reference's inputs
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    report = {}
    with pkg.Bark(path, seed=0, n_steps_text_encoder=16) as b:
        assert b.fast_mode
        for nn in range(2, 8):
            lf = b.fine_eval(buf, nn)
            lo = o.fine_eval(buf, nn)
            d = float(np.abs(lf - lo).max())
            top1 = float((lf[:, :1024].argmax(1) == lo[:, :1024].argmax(1)).mean())
            b.reseed(5); tf, _, _ = b.sample_rows(lf[:, :1024].copy(), 0.5)
            b.reseed(5); to, _, _ = b.sample_rows(lo[:, :1024].copy(), 0.5)
            report[nn] = dict(max_dlogit=round(d, 5), top1=round(top1, 4), cdf_flip_rate=round(float((tf != to).mean()), 5))
            assert d < MAX_DLOGIT[config] and top1 >= MIN_TOP1, report
        b.reseed(0)                                               # back to the load-time RNG state: the stream the oracle's generate consumed
        audio = b.generate("hello world")
        assert np.array_equal(b.tokens(0), ref["semantic"]) and np.array_equal(b.tokens(1), ref["coarse"])      # parity stages untouched
        fine = b.tokens(2)
        report["generate"] = dict(fine_ids_equal=round(float((fine == ref["fine"]).mean()), 4), frames=int(T),
                                  wav_rel=round(float(np.abs(audio - ref["audio"]).max() / np.abs(ref["audio"]).max()), 4))
    print("fast-mode agreement", config, json.dumps(report))


@gpu
def test_fast_fine_pass_deterministic(pkg, weights_file, monkeypatch):
    """The fast pass has no atomics: the same pass twice, with a different pass in between, gives the same logits bit for bit."""
    path = weights_file("wide", "f16")
    buf = np.random.default_rng(3).integers(0, 1024, (8, 1024)).astype(np.int32)
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    with pkg.Bark(path, seed=0, n_steps_text_encoder=16) as b:
        assert b.fast_mode
        first = b.fine_eval(buf, 7)
        b.fine_eval(buf, 3)
        again = b.fine_eval(buf, 7)
    assert np.array_equal(first.view(np.uint32), again.view(np.uint32)), f"{int((first != again).sum())} logits differ"
