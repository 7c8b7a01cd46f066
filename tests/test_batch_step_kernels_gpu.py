"""GPU: the batched decode step's kernels against references built from the C oracle's own pieces, bit for bit.

1. The few-row dense mat-mul (lane_matmul_kernel<T, 1> / <T, 8>, through bark_b200_parity_gemm variant 3 "rows"): every mat-mul of a
   batched step, the 1-row lm_head of a prefill and every parity pass of 2 to 15 rows.  The reference is orc_vec_dot_f16 / _f32 per
   output, the epilogue applied on the host (GELU through orc_gelu_table).  The models only reach it with widths that are multiples of
   128 and output counts that are multiples of 8; these cover every count of chain steps in the last weight group of both types, 9 to
   15 rows (a partial second 8-row block), output counts that leave the last CTA's warps idle, and bark-large's lm_head.  The hook sets
   every padding element of both operands to NaN, so a kernel that folds one into a stored sum fails.
2. The batched attention (attention_batch: attn_scores_batch_kernel<1..4>, attn_softmax_batch_kernel, attn_pv_batch_kernel, through
   bark_b200_batch_attention): each row is the one new query of its own sequence.  The reference is the oracle's single-query
   attention over that row's own pos + 1 keys: orc_vec_dot_f32 for QK^T and P.V, the float scale 1 / sqrt(E / H), orc_soft_max.  The
   models only reach 64-wide heads; these cover every head size, positions on both sides of the %8 / %32 leftover cuts, position 0
   beside 1023, and check the append to the caches, every operand format of the result, that a row's result does not depend on the
   batch around it, and that the multi-row attention kernels give the same bits for the same row.  The hook's caches are NaN from
   row pos on while the kernels run, so a key or value read before the append or from a wrong row fails."""
import ctypes as C
import functools
import types

import numpy as np
import pytest

from conftest import bits

MAX_REF = 4000              # oracle dots per mat-mul case beyond which a sample is taken
MAX_HEADS = 3               # heads per row checked against the oracle when there are more (the others: the cross-checks below)


@pytest.fixture(scope="module")
def ref(orc):
    L = C.CDLL(orc.ORACLE_SO)
    for n in ("orc_vec_dot_f16", "orc_vec_dot_f32"):
        getattr(L, n).restype = C.c_float
        getattr(L, n).argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    L.orc_gelu_table.restype = None
    L.orc_gelu_table.argtypes = [C.c_void_p]
    L.orc_soft_max.restype = None
    L.orc_soft_max.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    tab = np.zeros(65536, np.uint16)
    L.orc_gelu_table(tab.ctypes.data)

    def dots(A, W, idx):
        """the oracle's vec_dot for the (m, o) pairs idx: W row o against A row m"""
        f = L.orc_vec_dot_f16 if A.dtype == np.float16 else L.orc_vec_dot_f32
        K = A.shape[1]
        return np.array([f(K, W[o].ctypes.data, A[m].ctypes.data) for m, o in idx], np.float32)

    def attend(q, k, v, H, heads):
        """single-query attention of q [E] over the n_kv key / value rows k, v [n_kv][E], nothing masked; only `heads` are filled"""
        E, n_kv = q.shape[0], k.shape[0]
        D = E // H
        scale = np.float32(1.0) / np.sqrt(np.float32(E) / np.float32(H))        # bark.cpp:1318, in float
        out = np.full(E, np.nan, np.float32)
        s = np.empty(n_kv, np.float32)
        p = np.empty(n_kv, np.float32)
        for h in heads:
            qh = np.ascontiguousarray(q[h * D:(h + 1) * D])
            kh = np.ascontiguousarray(k[:, h * D:(h + 1) * D])
            vt = np.ascontiguousarray(v[:, h * D:(h + 1) * D].T)                    # V^T rows: one column of V each
            for j in range(n_kv):
                s[j] = np.float32(L.orc_vec_dot_f32(D, kh[j].ctypes.data, qh.ctypes.data)) * scale
            L.orc_soft_max(n_kv, s.ctypes.data, p.ctypes.data)
            for d in range(D):
                out[h * D + d] = L.orc_vec_dot_f32(n_kv, vt[d].ctypes.data, p.ctypes.data)
        return out

    return types.SimpleNamespace(dots=dots, attend=attend, gelu_tab=tab)


def assert_bits(have, want, what):
    bad = np.flatnonzero(bits(have) != bits(want))
    assert bad.size == 0, f"{what}: {bad.size} of {np.size(want)} values differ, first at {bad[0]}: {np.ravel(have)[bad[0]]} vs {np.ravel(want)[bad[0]]}"


# ---- the few-row mat-mul ----------------------------------------------------------------------------------------------------------
ROWS = [1, 2, 7, 8, 9, 15]
OUTS = [1, 7, 9, 33, 3 * 1024]
# chain steps in the last weight group (8 per group for f16, 4 for f32): every count, a second group, and bark-large's 4096
K_F16 = [32, 64, 96, 128, 160, 192, 224, 256, 288, 4096]
K_F32 = [32, 64, 96, 128, 160, 4096]
DT_K = [(np.float16, K) for K in K_F16] + [(np.float32, K) for K in K_F32]
DT_K_IDS = [f"{'f16' if dt == np.float16 else 'f32'}-K{K}" for dt, K in DT_K]


@functools.lru_cache(maxsize=None)
def operands(dt, K, N=max(OUTS), scale=2.0):
    """A [15][K], W [N][K]: the first M rows / N outputs of these are a case's operands"""
    rng = np.random.default_rng(K * 11 + (dt == np.float16) + int(scale))
    A = rng.standard_normal((max(ROWS), K)).astype(dt)
    W = (rng.standard_normal((N, K)) * (scale / np.sqrt(K))).astype(dt)
    return A, W


def sample(M, N, rng):
    """every output of small cases; else whole rows and columns (the first, the last, a random one, the last CTA's 8 outputs) and
    random elements"""
    if M * N <= MAX_REF:
        return [(m, o) for m in range(M) for o in range(N)]
    rows = {0, M - 1, int(rng.integers(M))}
    cols = {0, int(rng.integers(N))} | set(range(max(0, N - 8), N))
    idx = {(m, o) for m in rows for o in range(N)} | {(m, o) for m in range(M) for o in cols}
    idx |= {(int(m), int(o)) for m, o in zip(rng.integers(M, size=MAX_REF // 2), rng.integers(N, size=MAX_REF // 2))}
    return sorted(idx)


def check_store(pkg, ref, A, W, rng, what):
    got, ran = pkg.parity_gemm(A, W, variant="rows", return_variant=True)
    assert ran == 3, (what, ran)
    assert np.isfinite(got).all(), f"{what}: {np.count_nonzero(~np.isfinite(got))} outputs are not finite"
    idx = sample(A.shape[0], W.shape[0], rng)
    assert_bits(np.array([got[m, o] for m, o in idx], np.float32), ref.dots(A, W, idx), what)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("dt,K", DT_K, ids=DT_K_IDS)
@pytest.mark.parametrize("M", ROWS)
def test_rows_kernel_matches_oracle(pkg, ref, dt, K, M):
    A, W = operands(dt, K)
    rng = np.random.default_rng(M * 1000 + K)
    for N in OUTS:
        got = check_store(pkg, ref, A[:M], W[:N], rng, f"{M}x{N}x{K}")
        auto, ran = pkg.parity_gemm(A[:M], W[:N], return_variant=True)          # what lane_matmul runs for M < 16 rows
        assert ran == 3, (M, N, K, ran)
        assert_bits(auto, got, f"{M}x{N}x{K}: variant 0")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float16, np.float32], ids=["f16", "f32"])
def test_rows_kernel_bark_large_lm_head(pkg, ref, dt):
    A, W = operands(dt, 1024, N=10048)
    check_store(pkg, ref, A[:8], W, np.random.default_rng(10048), "8x10048x1024")


def gelu_host(x, tab, dt):
    """gelu_lookup (csrc/epilogue.cuh, ggml_vec_gelu_f32), then the operand type of the next mat-mul"""
    t = tab[x.astype(np.float16).view(np.uint16)].view(np.float16).astype(np.float32)
    return np.where(x <= -10.0, np.float32(0), np.where(x >= 10.0, x, t)).astype(dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,K", [(np.float16, 224), (np.float16, 288), (np.float32, 160), (np.float32, 96)], ids=["f16-K224", "f16-K288", "f32-K160", "f32-K96"])
@pytest.mark.parametrize("epilogue", ["resid", "gelu", "qkv"])
@pytest.mark.parametrize("M,N", [(1, 33), (9, 33), (15, 3 * 1024)])
def test_rows_kernel_epilogues(pkg, ref, epilogue, dt, K, M, N):
    # GELU: products with a standard deviation of 16, so the table and both clamps (x <= -10 -> 0, x >= 10 -> x) are reached
    A, W = operands(dt, K, scale=16.0 if epilogue == "gelu" else 2.0)
    A, W = A[:M], W[:N]
    rng = np.random.default_rng(M + N + K + len(epilogue))
    kw = {}
    if epilogue == "resid":
        kw["resid"] = rng.standard_normal((M, N)).astype(np.float32)
    if epilogue == "gelu":
        kw["gelu_tab"] = ref.gelu_tab
    got, ran = pkg.parity_gemm(A, W, epilogue=epilogue, variant="rows", return_variant=True, **kw)
    assert ran == 3
    idx = sample(M, N, rng)
    d = ref.dots(A, W, idx)
    mi, oi = np.array([i[0] for i in idx]), np.array([i[1] for i in idx])
    if epilogue == "resid":
        want, have = kw["resid"][mi, oi] + d, got[mi, oi]
    elif epilogue == "gelu":
        assert (d <= -10.0).any() and (d >= 10.0).any() and (np.abs(d) < 10.0).any(), "the case misses a GELU branch"
        want, have = gelu_host(d, ref.gelu_tab, dt), got[mi, oi]
        assert have.dtype == dt
    else:
        E = N // 3
        want, have = d, np.array([got[o // E][m, o % E] for m, o in idx], np.float32)
    view = np.uint16 if want.dtype == np.float16 else np.uint32
    bad = np.flatnonzero(np.asarray(have).view(view) != np.asarray(want).view(view))
    assert bad.size == 0, f"{epilogue}: {bad.size} of {len(idx)} checked outputs differ, first at {idx[bad[0]]}"


@pytest.mark.gpu
def test_auto_picks_the_rows_kernel_below_16_rows(pkg):
    for dt, tiled in ((np.float16, 2), (np.float32, 1)):
        A, W = operands(dt, 128)
        for M in (1, 8, 15):
            assert pkg.parity_gemm(A[:M], W[:64], return_variant=True)[1] == 3, (dt, M)
        A17 = np.concatenate([A, A[:2]])
        for M in (16, 17):
            assert pkg.parity_gemm(A17[:M], W[:64], return_variant=True)[1] == tiled, (dt, M)


# ---- the batched attention --------------------------------------------------------------------------------------------------------
HEAD_SIZES = [32, 64, 96, 128]
POSITION_SETS = {                       # name: positions of the launch's rows
    "zero": [0],
    "zero-x3": [0, 0, 0],
    "zero-x8": [0] * 8,
    "cuts": [7, 8, 9, 31, 32, 33, 63, 64],               # key counts on both sides of the %8 and %32 cuts
    "cut-65": [65],
    "first-and-last": [0, 1023],
    "last-x8": [1023] * 8,
    "ragged-1": "r1",
    "ragged-3": "r3",
    "ragged-8": "r8",
}


def positions(name, seed):
    p = POSITION_SETS[name]
    if isinstance(p, str):
        return [int(x) for x in np.random.default_rng(seed).integers(0, 1024, size=int(p[1:]))]
    return list(p)


def batch_operands(pos, E, seed, cap=None):
    """q, k_new, v_new [B][E] and caches [B][cap][E] (cap: a few rows past the last position, at most 1024)"""
    rng = np.random.default_rng(seed)
    B = len(pos)
    cap = cap or min(1024, max(pos) + 6)
    q, kn, vn = (rng.standard_normal((B, E), np.float32) for _ in range(3))
    kc, vc = (rng.standard_normal((B, cap, E), np.float32) for _ in range(2))
    return q, kn, vn, kc, vc


def keys(kc, kn, pos, b):
    """row b's pos + 1 key (or value) rows: its cache up to pos, then its new row"""
    return np.concatenate([kc[b, :pos[b]], kn[b:b + 1]])


def check_batch(pkg, ref, pos, D, H, seed):
    """one launch: every row against the oracle (up to MAX_HEADS heads), and the caches after the append; returns the operands and
    the result"""
    E = D * H
    q, kn, vn, kc, vc = batch_operands(pos, E, seed)
    out, kc2, vc2 = pkg.batch_attention(q, kn, vn, kc, vc, pos, H)
    assert np.isfinite(out).all(), f"{np.count_nonzero(~np.isfinite(out))} outputs are not finite"
    rng = np.random.default_rng(seed + 1)
    for b, p in enumerate(pos):
        heads = range(H) if H <= MAX_HEADS else sorted({0, H - 1, int(rng.integers(H))})
        want = ref.attend(q[b], keys(kc, kn, pos, b), keys(vc, vn, pos, b), H, heads)
        cols = np.concatenate([np.arange(h * D, (h + 1) * D) for h in heads])
        assert_bits(out[b, cols], want[cols], f"row {b} at position {p}")
        for name, new, old, got in (("K", kn, kc, kc2), ("V", vn, vc, vc2)):
            assert_bits(got[b, :p], old[b, :p], f"{name} cache of row {b}: rows before {p}")
            assert_bits(got[b, p], new[b], f"{name} cache of row {b}: the appended row {p}")
            assert np.isnan(got[b, p + 1:]).all(), f"{name} cache of row {b}: a store past row {p}"
    return (q, kn, vn, kc, vc), out


@pytest.mark.gpu
@pytest.mark.parametrize("D", HEAD_SIZES)
@pytest.mark.parametrize("name", list(POSITION_SETS))
def test_batch_attention_matches_oracle(pkg, ref, D, name):
    check_batch(pkg, ref, positions(name, seed=D), D, 2, seed=D * 7 + len(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["zero-x3", "cuts", "first-and-last", "last-x8", "ragged-8"])
def test_batch_attention_16_heads(pkg, ref, name):
    check_batch(pkg, ref, positions(name, seed=16), 64, 16, seed=16 + len(name))


@pytest.mark.gpu
@pytest.mark.parametrize("D", HEAD_SIZES)
def test_batch_attention_operand_formats(pkg, ref, D):
    pos = positions("ragged-8", seed=D + 1)
    ops, out = check_batch(pkg, ref, pos, D, 3, seed=D + 2)
    f16, _, _ = pkg.batch_attention(*ops, pos, 3, act="f16")
    assert f16.dtype == np.float16
    assert np.array_equal(f16.view(np.uint16), out.astype(np.float16).view(np.uint16)), "f16 group-major operand"
    f32, _, _ = pkg.batch_attention(*ops, pos, 3, act="f32_gm")
    assert_bits(f32, out, "f32 group-major operand")


@pytest.mark.gpu
@pytest.mark.parametrize("D", HEAD_SIZES)
def test_batch_rows_do_not_depend_on_the_batch(pkg, ref, D):
    """each row's bits do not depend on B, its place in the batch or the other rows' positions (and so on the launch's max_kv)"""
    H = 2
    pos = positions("ragged-8", seed=D + 3)
    pos[5] = 1023                                       # one row at the last position: max_kv 1024 for the rows beside it
    q, kn, vn, kc, vc = ops = batch_operands(pos, D * H, seed=D + 4, cap=1024)
    out = pkg.batch_attention(*ops, pos, H)[0]
    assert np.isfinite(out).all()
    rng = np.random.default_rng(D)
    for order in (rng.permutation(8), [5, 0, 3], [2], [7, 1]):
        order = list(order)
        sub = [pos[i] for i in order]
        got, _, _ = pkg.batch_attention(q[order], kn[order], vn[order], kc[order], vc[order], sub, H)
        assert_bits(got, out[order], f"rows {order} at positions {sub}")


@pytest.mark.gpu
@pytest.mark.parametrize("D", HEAD_SIZES)
def test_batch_attention_matches_multi_row_kernels(pkg, ref, D):
    """the same query through the multi-row attention (N = 1, n_past = pos, causal) gives the same bits"""
    H = 2
    pos = [0, 9, 33, 200, 1023]
    q, kn, vn, kc, vc = ops = batch_operands(pos, D * H, seed=D + 5)
    out, _, _ = pkg.batch_attention(*ops, pos, H)
    for b, p in enumerate(pos):
        for path in ("fused", "tiled"):
            got = pkg.parity_attention(q[b:b + 1], keys(kc, kn, pos, b), keys(vc, vn, pos, b), H, n_past=p, causal=True, path=path)
            assert_bits(got[0], out[b], f"row {b} at position {p}, {path} path")


@pytest.mark.gpu
def test_batch_attention_invalid_arguments_fail_without_aborting(pkg, ref):
    q, kn, vn, kc, vc = batch_operands([1] * 9, 128, seed=9)
    with pytest.raises(RuntimeError):
        pkg.batch_attention(q, kn, vn, kc, vc, [1] * 9, 2)                            # B = 9
    with pytest.raises(RuntimeError):
        pkg.batch_attention(q[:2, :96], kn[:2, :96], vn[:2, :96], kc[:2, :, :96], vc[:2, :, :96], [1, 1], 2)   # head size 48
    with pytest.raises(RuntimeError):
        pkg.batch_attention(q[:2], kn[:2], vn[:2], kc[:2], vc[:2], [1, kc.shape[1]], 2)   # pos >= cap
    with pytest.raises(RuntimeError):
        pkg.batch_attention(q[:2], kn[:2], vn[:2], kc[:2], vc[:2], [1, -1], 2)          # pos < 0
    big = np.zeros((1, 1025, 128), np.float32)
    with pytest.raises(RuntimeError):
        pkg.batch_attention(q[:1], kn[:1], vn[:1], big, big, [3], 2)                      # cap = 1025
    check_batch(pkg, ref, [0, 5], 64, 2, seed=10)                                         # and the library still works afterwards
