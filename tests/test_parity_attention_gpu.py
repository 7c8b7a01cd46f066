"""GPU: the parity path's multi-row attention kernel against a reference built from the C oracle's own pieces — orc_vec_dot_f32 for
QK^T and for P.V, a float32 scale, the -inf causal mask and orc_soft_max (oracle/bark_oracle.c `attention`) — bit for bit.

The model tests only reach 64-wide heads; these cover every head size the kernels are built for, query counts on both sides of the
fused kernel's 32-query tile, key counts on both sides of the % 8 / % 32 cuts where soft_max's and P.V's leftover handling starts, and
a partial last V chunk.  Every shape runs through both paths: the fused kernel and the three kernels used for few rows."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits


@pytest.fixture(scope="module")
def ref(orc):
    L = C.CDLL(orc.ORACLE_SO)
    L.orc_vec_dot_f32.restype = C.c_float
    L.orc_vec_dot_f32.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    L.orc_soft_max.restype = None
    L.orc_soft_max.argtypes = [C.c_int, C.c_void_p, C.c_void_p]

    def attention(q, k, v, H, n_past, causal):
        N, E = q.shape
        n_kv, D = k.shape[0], E // H
        scale = np.float32(1.0) / np.sqrt(np.float32(E) / np.float32(H))        # bark.cpp:1318, in float
        out = np.empty((N, E), np.float32)
        s = np.empty(n_kv, np.float32)
        p = np.empty(n_kv, np.float32)
        for h in range(H):
            kh = [np.ascontiguousarray(k[j, h * D:(h + 1) * D]) for j in range(n_kv)]
            vt = np.ascontiguousarray(v[:, h * D:(h + 1) * D].T)                    # V^T rows: one column of V each
            for i in range(N):
                qv = np.ascontiguousarray(q[i, h * D:(h + 1) * D])
                for j in range(n_kv):
                    s[j] = np.float32(L.orc_vec_dot_f32(D, kh[j].ctypes.data, qv.ctypes.data)) * scale
                    if causal and j > n_past + i:
                        s[j] = -np.inf
                L.orc_soft_max(n_kv, s.ctypes.data, p.ctypes.data)
                for d in range(D):
                    out[i, h * D + d] = L.orc_vec_dot_f32(n_kv, vt[d].ctypes.data, p.ctypes.data)
        return out
    return attention


def operands(N, n_kv, E, seed):
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((N, E), np.float32)
    k = rng.standard_normal((n_kv, E), np.float32)
    v = rng.standard_normal((n_kv, E), np.float32)
    return q, k, v


def check(pkg, ref, N, n_kv, n_past, D, H, causal, seed=0):
    E = D * H
    q, k, v = operands(N, n_kv, E, seed)
    want = ref(q, k, v, H, n_past, causal)
    for path in ("fused", "tiled"):
        got = pkg.parity_attention(q, k, v, H, n_past=n_past, causal=causal, path=path)
        assert np.isfinite(got).all(), path
        bad = np.flatnonzero(bits(got) != bits(want))
        assert bad.size == 0, f"{path}: {bad.size} of {got.size} outputs differ, first at {np.unravel_index(bad[0], got.shape)}"


@pytest.mark.gpu
@pytest.mark.parametrize("D", [32, 64, 96, 128])
@pytest.mark.parametrize("N", [1, 31, 33, 100])
def test_head_sizes_and_query_counts(pkg, ref, D, N):
    check(pkg, ref, N, N, 0, D, 2, causal=True, seed=D + N)


@pytest.mark.gpu
@pytest.mark.parametrize("n_kv", [7, 8, 9, 31, 32, 33, 63, 64, 65, 95, 96, 97, 103, 104])
def test_causal_with_history_across_leftover_cuts(pkg, ref, n_kv):
    N = min(n_kv, 40)
    check(pkg, ref, N, n_kv, n_kv - N, 64, 3, causal=True, seed=n_kv)


@pytest.mark.gpu
@pytest.mark.parametrize("n_kv", [15, 16, 17, 39, 40, 41, 63, 64, 65])
def test_few_rows_with_history_across_leftover_cuts(pkg, ref, n_kv):
    check(pkg, ref, 8, n_kv, n_kv - 8, 64, 2, causal=True, seed=100 + n_kv)


@pytest.mark.gpu
def test_coarse_window_partial_v_chunk(pkg, ref):
    check(pkg, ref, 90, 800, 710, 64, 2, causal=True, seed=800)     # 800 keys: a full V chunk of 512 keys, then a partial one of 288


@pytest.mark.gpu
def test_non_causal_257(pkg, ref):
    check(pkg, ref, 257, 257, 0, 64, 2, causal=False, seed=257)


@pytest.mark.gpu
def test_non_causal_full_head(pkg, ref):
    check(pkg, ref, 1024, 1024, 0, 64, 1, causal=False, seed=1024)
