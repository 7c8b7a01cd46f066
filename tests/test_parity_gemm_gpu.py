"""GPU: the parity path's tiled GEMM (lane_gemm_tiled_kernel, through bark_b200_parity_gemm) against a reference built from the C
oracle's own dot products — orc_vec_dot_f16 / orc_vec_dot_f32 per output, the epilogue applied on the host (GELU through
orc_gelu_table) — bit for bit.

The model tests reach the kernel only at the models' own widths.  These cover row counts on both sides of the 32-row block tile,
output counts on both sides of the 16- and 32-wide ones, K with a partial last 128-column group, bark-large's widths, every epilogue,
both operand types and every block-tile variant forced, and the few-row kernel (lane_matmul_kernel, variant 3) forced at the same
shapes.  Every variant must give the same bits on every output; the oracle is asked
for all outputs of the small shapes and for a sample (whole rows, whole columns and random elements) of the big ones.  Each call also
checks the guard bands around its output (GuardBandError)."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits

VARIANTS = {np.float16: (0, 1, 2, 3), np.float32: (0, 1, 3)}     # 3: the few-row kernel, forced at every row count
MAX_REF = 6000              # oracle dots per case beyond which a sample is taken


@pytest.fixture(scope="module")
def ref(orc):
    L = C.CDLL(orc.ORACLE_SO)
    for n in ("orc_vec_dot_f16", "orc_vec_dot_f32"):
        getattr(L, n).restype = C.c_float
        getattr(L, n).argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    L.orc_gelu_table.restype = None
    L.orc_gelu_table.argtypes = [C.c_void_p]
    tab = np.zeros(65536, np.uint16)
    L.orc_gelu_table(tab.ctypes.data)

    def dots(A, W, idx):
        """the oracle's vec_dot for the (m, o) pairs idx: W row o against A row m"""
        f = L.orc_vec_dot_f16 if A.dtype == np.float16 else L.orc_vec_dot_f32
        K = A.shape[1]
        return np.array([f(K, W[o].ctypes.data, A[m].ctypes.data) for m, o in idx], np.float32)
    dots.gelu_tab = tab
    return dots


def sample(M, N, rng):
    if M * N <= MAX_REF:
        return [(m, o) for m in range(M) for o in range(N)]
    rows = {0, M - 1, int(rng.integers(M))}
    cols = {0, N - 1, int(rng.integers(N))}
    idx = {(m, o) for m in rows for o in range(N)} | {(m, o) for m in range(M) for o in cols}
    idx |= {(int(m), int(o)) for m, o in zip(rng.integers(M, size=MAX_REF // 2), rng.integers(N, size=MAX_REF // 2))}
    return sorted(idx)


def operands(M, N, K, dt, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(dt)
    W = (rng.standard_normal((N, K)) * (2.0 / np.sqrt(K))).astype(dt)     # products of order 1: GELU's table range and both clamps
    return A, W, rng


def gelu_host(x, tab, dt):
    """gelu_lookup (csrc/epilogue.cuh, ggml_vec_gelu_f32), then the operand type of the next mat-mul"""
    t = tab[x.astype(np.float16).view(np.uint16)].view(np.float16).astype(np.float32)
    return np.where(x <= -10.0, np.float32(0), np.where(x >= 10.0, x, t)).astype(dt)


def check_variants(pkg, A, W, dt, epilogue="store", **kw):
    """every variant gives the same bits; returns the result and the variant "auto" picked"""
    first, picked = None, None
    for v in VARIANTS[dt]:
        got, ran = pkg.parity_gemm(A, W, epilogue=epilogue, variant=v, return_variant=True, **kw)
        assert ran == v or v == 0, (v, ran)
        flat = np.concatenate([np.ravel(g) for g in got]) if isinstance(got, tuple) else np.ravel(got)
        if first is None:
            first, picked, res = flat, ran, got
        else:
            diff = np.flatnonzero(flat.view(np.uint16 if flat.dtype == np.float16 else np.uint32) !=
                                  first.view(np.uint16 if first.dtype == np.float16 else np.uint32))
            assert diff.size == 0, f"variant {v}: {diff.size} of {flat.size} outputs differ from variant {VARIANTS[dt][0]}'s"
    return res, picked


SHAPES = [   # M, N, K: row counts 16 .. 1024 around the 32-row tile, output counts around the 16 / 32 tiles, K with partial groups
    (16, 1, 32), (17, 15, 96), (33, 17, 160), (91, 33, 768), (257, 768, 96), (513, 1056, 160),
    (16, 2304, 3072), (1024, 2304, 768), (1024, 768, 3072), (91, 768, 768),
    (257, 3072, 1024), (33, 1024, 4096),                                   # bark-large widths (E = 1024)
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float16, np.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_store_matches_oracle(pkg, ref, M, N, K, dt):
    A, W, rng = operands(M, N, K, dt, seed=M * 7 + N * 3 + K)
    got, _ = check_variants(pkg, A, W, dt)
    assert np.isfinite(got).all()
    idx = sample(M, N, rng)
    want = ref(A, W, idx)
    have = np.array([got[m, o] for m, o in idx], np.float32)
    bad = np.flatnonzero(bits(have) != bits(want))
    assert bad.size == 0, f"{bad.size} of {len(idx)} checked outputs differ, first at {idx[bad[0]]}: {have[bad[0]]} vs {want[bad[0]]}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float16, np.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("epilogue", ["resid", "gelu", "qkv"])
@pytest.mark.parametrize("M,N,K", [(33, 51, 160), (91, 2304, 768)])
def test_epilogues_match_oracle(pkg, ref, epilogue, dt, M, N, K):
    A, W, rng = operands(M, N, K, dt, seed=M + N + K + len(epilogue))
    kw = {}
    if epilogue == "resid":
        kw["resid"] = rng.standard_normal((M, N)).astype(np.float32)
    if epilogue == "gelu":
        kw["gelu_tab"] = ref.gelu_tab
    got, _ = check_variants(pkg, A, W, dt, epilogue=epilogue, **kw)
    idx = sample(M, N, rng)
    d = ref(A, W, idx)
    mi, oi = np.array([i[0] for i in idx]), np.array([i[1] for i in idx])
    if epilogue == "resid":
        want, have = kw["resid"][mi, oi] + d, got[mi, oi]
    elif epilogue == "gelu":
        want, have = gelu_host(d, ref.gelu_tab, dt), got[mi, oi]
        assert have.dtype == dt
    else:
        E = N // 3
        want, have = d, np.array([got[o // E][m, o % E] for m, o in idx], np.float32)
    view = np.uint16 if want.dtype == np.float16 else np.uint32
    bad = np.flatnonzero(np.asarray(have).view(view) != np.asarray(want).view(view))
    assert bad.size == 0, f"{epilogue}: {bad.size} of {len(idx)} checked outputs differ, first at {idx[bad[0]]}"


@pytest.mark.gpu
def test_auto_picks_the_32x32_tile_for_f16_and_the_32x16_tile_for_f32(pkg):
    for dt, want in ((np.float16, 2), (np.float32, 1)):
        for M in (91, 1024):
            A, W, _ = operands(M, 768, 128, dt, seed=M)
            assert pkg.parity_gemm(A, W, return_variant=True)[1] == want, (dt, M)


@pytest.mark.gpu
def test_invalid_arguments_fail_without_aborting(pkg):
    A, W, _ = operands(32, 32, 64, np.float32, seed=3)
    with pytest.raises(RuntimeError):
        pkg.parity_gemm(A, W, variant=2)                       # f32 has only the 32 x 16 tile
    with pytest.raises(RuntimeError):
        pkg.parity_gemm(A, W, variant=-1)
    with pytest.raises(RuntimeError):
        pkg.parity_gemm(A, W, variant=4)
    with pytest.raises(RuntimeError):
        pkg.parity_gemm(A[:, :48], W[:, :48])                  # K % 32 != 0
    with pytest.raises(RuntimeError):
        pkg.parity_gemm(A, W[:31], epilogue="qkv")             # N % 3 != 0
    A16, W16, _ = operands(32, 32, 64, np.float16, seed=4)
    assert np.isfinite(pkg.parity_gemm(A16, W16)).all()       # and the library still works afterwards
