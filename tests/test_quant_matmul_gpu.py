"""GPU: the quantised mat-muls kernel by kernel (bark_b200_quant_matmul) against the unmodified reference's stored block dots
(tests/golden/ref_pairs/quant_dots.npz) and against the C oracle's quantiser and per-type dots, bit for bit.

Three device implementations are covered: q4_0 on the per-op path (quantize_q8_kernel + q4_matmul_kernel<1,1> / <8,4>), q4_1 / q5_0 /
q5_1 / q8_0 (quantize_q8x_kernel + qx_matmul_kernel), and q4_0 inside the persistent decode step (quantize_act_q8 + row_dot_q4, staged
in shared memory or read from global memory).  The model tests only reach them with well-conditioned activations at the models' widths;
these add row counts on both sides of the 8-row tile, output counts around the 4-, 16- and 128-output tiles (the <8,4> kernel clamps
its last tile), every epilogue, the reference's edge blocks placed in the tile tails and the last block of a row, and integer operands
whose dots are exact.  NaN results (a block holding an inf, d past the f16 range) compare as NaN; every other output by its bits."""
import threading

import numpy as np
import pytest

from conftest import bits
from test_quant_dots import REF, TYPES, exact, f16_bits, same_bits

FINITE = [i for i, n in enumerate(REF["act_names"]) if "inf" not in n and "overflow" not in n]


def assert_same(have, want, what):
    bad = np.argwhere(~same_bits(np.asarray(have, np.float32), np.asarray(want, np.float32)))
    assert bad.size == 0, f"{what}: {len(bad)} of {np.size(want)} outputs differ, first at {tuple(bad[0])}: {have[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def assert_q8_matches_oracle(orc, qtype, A, q, d, s):
    y = orc.quantize_q8(A, orc.vec_dot_type(qtype))
    assert np.array_equal(q, y["qs"].reshape(q.shape)), "quantised bytes differ from the oracle's"
    assert same_bits(d, f16_bits(y["d"])).all(), "d differs from the oracle's"
    if s is not None:
        assert same_bits(s, f16_bits(y["s"])).all(), "s differs from the oracle's"


def operands(qtype, M, N, K, seed, edges=True):
    """A [M][K]: N(0, 1) rows; W [N][K/32 blocks]: blocks drawn from the stored weight edge blocks.  With edges, stored activation
    edge blocks go into the last row (the 8-row tile's tail), the first row and random places, each into the row's last block
    too; the last weight row (the output tiles' tail) ends with an edge block."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    wb = REF[f"w_{qtype}"]
    nb = K // 32
    W = wb[rng.integers(len(wb), size=(N, nb))].reshape(N, -1)
    if edges:
        pool = REF["act"]
        for m in {0, M - 1, int(rng.integers(M))}:
            for b in {nb - 1, int(rng.integers(nb))}:
                A[m, b * 32:(b + 1) * 32] = pool[int(rng.integers(len(pool)))]
    else:
        for m in {0, M - 1}:
            A[m, (nb - 1) * 32:] = REF["act"][FINITE[int(rng.integers(len(FINITE)))]]
    return A, W, rng


@pytest.mark.gpu
@pytest.mark.parametrize("qtype", TYPES)
def test_reference_block_dots(pkg, qtype):
    """every stored weight block against every stored activation block (one block per row: M = all activation blocks, N = all
    weight blocks), then the same one activation row at a time (the single-row kernels), and the quantised blocks themselves"""
    act, W, want = REF["act"], REF[f"w_{qtype}"], REF[f"dot1_{qtype}"].T
    out, q, d, s = pkg.quant_matmul(qtype, W, act, return_q8=True)
    assert_same(out, want, f"{qtype} all blocks")
    kind = "q8_1" if qtype in ("q4_1", "q5_1") else "q8_0"
    names = REF["act_names"]
    bad = np.flatnonzero((q != REF[f"{kind}_qs"]).any(1))
    assert bad.size == 0, f"{kind} bytes differ from the reference's on {list(names[bad])}"
    bad = np.flatnonzero(~same_bits(d[:, 0], f16_bits(REF[f"{kind}_d"])))
    assert bad.size == 0, f"{kind} d differs from the reference's on {list(names[bad])}"
    if s is not None:
        bad = np.flatnonzero(~same_bits(s[:, 0], f16_bits(REF["q8_1_s"])))
        assert bad.size == 0, f"q8_1 s differs from the reference's on {list(names[bad])}"
    for a in range(act.shape[0]):
        assert_same(pkg.quant_matmul(qtype, W, act[a:a + 1]), want[a:a + 1], f"{qtype} activation block {names[a]} alone")


@pytest.mark.gpu
@pytest.mark.parametrize("qtype", TYPES)
def test_reference_row_dots(pkg, qtype):
    """rows of eight blocks with edge blocks inside and at the end: all rows together, and one at a time"""
    A, W, want = REF["rows_act"], REF[f"rows_w_{qtype}"], REF[f"rows_dot_{qtype}"].T
    assert_same(pkg.quant_matmul(qtype, W, A), want, qtype)
    for m in (0, A.shape[0] - 1):
        assert_same(pkg.quant_matmul(qtype, W, A[m:m + 1]), want[m:m + 1], f"{qtype} row {m}")


@pytest.mark.gpu
@pytest.mark.parametrize("qtype", TYPES)
def test_integer_rows_are_exact(pkg, qtype):
    W, A = REF[f"int_w_{qtype}"], REF["int_act"]
    want = exact(qtype, W, A).T
    assert np.array_equal(pkg.quant_matmul(qtype, W, A).astype(np.float64), want)
    assert np.array_equal(pkg.quant_matmul(qtype, W[:, :W.shape[1] // 32], A[:3, :32]).astype(np.float64), exact(qtype, W[:, :W.shape[1] // 32], A[:3, :32]).T)


SHAPES = [   # M, N, K: rows around the 8-row tile, outputs around the 4-, 16- and 128-output tiles, K from one block to 128
    (1, 1, 32), (2, 3, 64), (7, 4, 96), (8, 15, 128), (9, 16, 4096), (17, 17, 32), (64, 127, 64), (513, 128, 96), (1, 129, 4096),
    (2, 1056, 128), (9, 3072, 32), (8, 127, 4096), (513, 129, 128), (7, 3072, 96), (1, 3072, 128), (17, 1056, 4096),
]


@pytest.mark.gpu
@pytest.mark.parametrize("qtype", TYPES)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_store_matches_oracle(pkg, orc, qtype, M, N, K):
    A, W, _ = operands(qtype, M, N, K, seed=M * 31 + N * 7 + K + len(qtype))
    out, q, d, s = pkg.quant_matmul(qtype, W, A, return_q8=True)
    assert_same(out, orc.quant_matmul(qtype, W, A), f"{qtype} {M}x{N}x{K}")
    assert_q8_matches_oracle(orc, qtype, A, q, d, s)


def gelu_host(x, tab):
    """gelu_lookup (csrc/epilogue.cuh) into f32 rows, the operand a quantised model's next mat-mul quantises"""
    t = tab[x.astype(np.float16).view(np.uint16)].view(np.float16).astype(np.float32)
    return np.where(x <= -10.0, np.float32(0), np.where(x >= 10.0, x, t)).astype(np.float32)


@pytest.fixture(scope="module")
def gelu_tab(orc):
    import ctypes as C
    L = C.CDLL(orc.ORACLE_SO)
    L.orc_gelu_table.argtypes = [C.c_void_p]
    tab = np.zeros(65536, np.uint16)
    L.orc_gelu_table(tab.ctypes.data)
    return tab


@pytest.mark.gpu
@pytest.mark.parametrize("qtype", TYPES)
@pytest.mark.parametrize("epilogue", ["resid", "gelu", "qkv"])
@pytest.mark.parametrize("M,N,K", [(9, 129, 96), (64, 1056, 128), (1, 3072, 4096)])
def test_epilogues_match_oracle(pkg, orc, gelu_tab, qtype, epilogue, M, N, K):
    A, W, rng = operands(qtype, M, N, K, seed=M + N + K + len(epilogue), edges=False)
    d = orc.quant_matmul(qtype, W, A)
    if epilogue == "resid":
        resid = rng.standard_normal((M, N)).astype(np.float32)
        assert_same(pkg.quant_matmul(qtype, W, A, "resid", resid=resid), resid + d, f"{qtype} resid")
    elif epilogue == "gelu":
        assert_same(pkg.quant_matmul(qtype, W, A, "gelu", gelu_tab=gelu_tab), gelu_host(d, gelu_tab), f"{qtype} gelu")
    else:
        E = N // 3
        got = pkg.quant_matmul(qtype, W, A, "qkv")
        for i in range(3):
            assert_same(got[i], d[:, i * E:(i + 1) * E], f"{qtype} qkv part {i}")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["decode_staged", "decode_global"])
@pytest.mark.parametrize("K,N", [(128, 1), (128, 17), (128, 2304), (768, 63), (768, 3072), (32, 5), (4096, 129)])
def test_decode_path_matches_oracle(pkg, orc, path, K, N):
    """the persistent decode step's q4_0 pieces: rows in groups of four per warp (a partial last group), every epilogue"""
    A, W, rng = operands("q4_0", 1, N, K, seed=K + N)
    out, q, d, _ = pkg.quant_matmul("q4_0", W, A, path=path, return_q8=True)
    want = orc.quant_matmul("q4_0", W, A)
    assert_same(out, want, f"{path} {N}x{K}")
    assert_q8_matches_oracle(orc, "q4_0", A, q, d, None)
    assert_same(out, pkg.quant_matmul("q4_0", W, A), "decode path vs per-op path")
    if N % 3 == 0:
        A, W, rng = operands("q4_0", 1, N, K, seed=K + N + 1, edges=False)
        want = orc.quant_matmul("q4_0", W, A)
        resid = rng.standard_normal((1, N)).astype(np.float32)
        assert_same(pkg.quant_matmul("q4_0", W, A, "resid", path=path, resid=resid), resid + want, f"{path} resid")
        got = pkg.quant_matmul("q4_0", W, A, "qkv", path=path)
        for i in range(3):
            assert_same(got[i], want[:, i * (N // 3):(i + 1) * (N // 3)], f"{path} qkv part {i}")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["decode_staged", "decode_global"])
def test_decode_path_reference_rows(pkg, path):
    A, W, want = REF["rows_act"], REF["rows_w_q4_0"], REF["rows_dot_q4_0"].T
    for m in range(A.shape[0]):
        assert_same(pkg.quant_matmul("q4_0", W, A[m:m + 1], path=path), want[m:m + 1], f"{path} row {m}")
    W, A = REF["int_w_q4_0"], REF["int_act"]
    assert np.array_equal(pkg.quant_matmul("q4_0", W, A[:1], path=path).astype(np.float64), exact("q4_0", W, A[:1]).T)


@pytest.mark.gpu
@pytest.mark.parametrize("qtype,ftype", [("q4_0", 2), ("q4_1", 3)])
def test_a_context_on_the_same_thread_is_unaffected(pkg, orc, weights_file, tmp_path, qtype, ftype):
    """the hook quantises into its own scratch and puts the thread's scratch pointers back: a context's quantised passes between and
    after hook calls (and the hook on a thread that never had a context) give the oracle's logits"""
    path = str(tmp_path / f"tiny_{qtype}.bin")
    assert pkg.lib().bark_model_quantize(weights_file("tiny", "f16").encode(), path.encode(), ftype)
    o = orc.Oracle(path, seed=0, n_steps=8)
    A, W, _ = operands(qtype, 9, 40, 128, seed=5)
    want_hook = orc.quant_matmul(qtype, W, A)
    errors = []
    t = threading.Thread(target=lambda: errors.append(not same_bits(pkg.quant_matmul(qtype, W, A), want_hook).all()))
    t.start(); t.join()
    assert errors == [False], "the hook on a fresh thread"
    with pkg.Bark(path, seed=0, n_steps_text_encoder=8) as b:
        toks, pg, po = o.tokenize("Hello, world"), 0, 0
        for step in range(4):
            assert_same(pkg.quant_matmul(qtype, W, A), want_hook, f"hook before step {step}")
            lg, pg = b.gpt_eval(0, toks, pg, True)
            lo, po = o.gpt_eval(0, toks, po, True)
            assert np.array_equal(bits(lg), bits(lo)), f"semantic step {step} after the hook: logits differ from the oracle's"
            toks = np.array([int(np.argmax(lo[:10000]))], np.int32)
        buf = np.random.default_rng(3).integers(0, 1024, (8, 1024)).astype(np.int32); buf[2:, :] = 1024
        assert_same(pkg.quant_matmul(qtype, W[:7], A[:2]), want_hook[:2, :7], "hook before the fine pass")
        assert np.array_equal(bits(b.fine_eval(buf, 2)), bits(o.fine_eval(buf, 2))), "fine pass after the hook"


@pytest.mark.gpu
def test_invalid_arguments_fail_without_aborting(pkg, orc):
    A, W, _ = operands("q4_0", 2, 6, 64, seed=1)
    with pytest.raises(RuntimeError):
        pkg.quant_matmul("q4_0", W, A, path="decode_staged")              # the decode path takes one row
    with pytest.raises(RuntimeError):
        pkg.quant_matmul("q4_0", W[:5], A, "qkv")                         # N % 3 != 0
    A1, W1, _ = operands("q8_0", 1, 6, 64, seed=2)
    with pytest.raises(RuntimeError):
        pkg.quant_matmul("q8_0", W1, A1, path="decode_global")            # the decode path is q4_0 only
    assert_same(pkg.quant_matmul("q4_0", W, A), orc.quant_matmul("q4_0", W, A), "after the rejected calls")
