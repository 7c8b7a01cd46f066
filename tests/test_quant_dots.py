"""The C oracle's activation quantisers and quantised block dots (oracle/bark_oracle.c: quantize_row_q8_0 / q8_1 and the five
vec_dot restatements) against the unmodified reference's own, on edge blocks, bit for bit — and an integer-exact check that needs no
restatement at all.  The reference's results are stored in tests/golden/ref_pairs/quant_dots.npz (tests/golden/make_golden_quant_dots.py).

The model tests reach these paths only with LayerNorm / GELU activations of a few widths: these pin the round-half ties, the f16
rounding of d (ties, subnormal, overflow), 127 / amax overflowing to inf, blocks holding an inf (cvtps_epi32's INT_MIN, saturated to
-128 by the packs; q8_1's s sums the int32 values), and weight blocks with d = +-0, subnormal or +-65504, extreme codes, every q5
fifth bit and the q4_1 / q5_1 minimum."""
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR

REF = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "quant_dots.npz"))
TYPES = ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0")


def same_bits(a, b):
    """equal bits, or both NaN (a NaN's sign and payload are not part of what is checked)"""
    a, b = np.asarray(a), np.asarray(b)
    ua = a.view(np.uint16 if a.dtype == np.float16 else np.uint32)
    ub = b.view(np.uint16 if b.dtype == np.float16 else np.uint32)
    return (ua == ub) | (np.isnan(a) & np.isnan(b))


def f16_bits(u):
    return np.asarray(u, np.uint16).view(np.float16)


@pytest.mark.parametrize("kind", ["q8_0", "q8_1"])
def test_quantiser_matches_the_reference(orc, kind):
    y = orc.quantize_q8(REF["act"], kind)
    names = REF["act_names"]
    bad = np.flatnonzero((y["qs"].reshape(len(names), 32) != REF[f"{kind}_qs"]).any(1))
    assert bad.size == 0, f"{kind} bytes differ on {list(names[bad])}"
    bad = np.flatnonzero(~same_bits(f16_bits(y["d"].ravel()), f16_bits(REF[f"{kind}_d"])))
    assert bad.size == 0, f"{kind} d differs on {list(names[bad])}"
    if kind == "q8_1":
        bad = np.flatnonzero(~same_bits(f16_bits(y["s"].ravel()), f16_bits(REF["q8_1_s"])))
        assert bad.size == 0, f"q8_1 s differs on {list(names[bad])}"


def test_fixtures_hold_the_non_finite_conversion():
    """what the reference does where 127 / amax overflows or a block holds an inf: every non-finite product is the byte -128, and
    q8_1's s is f16(d * the wrapped int32 sum of INT_MIN values) — the divergence the kernels' conversion had"""
    names = list(REF["act_names"])
    for n in ("amax_below_127_over_fltmax", "amax_denormal", "amax_tiny_single"):
        i = names.index(n)
        assert (REF["q8_0_qs"][i] == -128).all() and (REF["q8_1_qs"][i] == -128).all(), n
        assert REF["q8_0_d"][i] & 0x7fff == 0, n                          # d = amax / 127 rounds to +-0 in f16
    i = names.index("pos_inf")
    assert REF["q8_0_qs"][i][7] == -128 and (np.delete(REF["q8_0_qs"][i], 7) == 0).all()   # inf * 0 = NaN; finite * 0 = 0
    assert f16_bits(REF["q8_1_s"][i]) == -np.inf                          # d = inf times the sum INT_MIN
    assert np.isnan(f16_bits(REF["q8_1_s"][names.index("two_inf")]))      # two INT_MIN wrap to 0: inf * 0


@pytest.mark.parametrize("qtype", TYPES)
def test_block_dots_match_the_reference(orc, qtype):
    """every weight edge block against every activation edge block (n = 32)"""
    W, act, want = REF[f"w_{qtype}"], REF["act"], REF[f"dot1_{qtype}"]
    Y = orc.quantize_q8(act, orc.vec_dot_type(qtype))
    have = np.array([[orc.vec_dot_q(qtype, W[w], Y[a]) for a in range(act.shape[0])] for w in range(W.shape[0])], np.float32)
    bad = np.argwhere(~same_bits(have, want))
    assert bad.size == 0, (f"{len(bad)} dots differ, first weight {REF[f'w_{qtype}_names'][bad[0][0]]} x activation "
                           f"{REF['act_names'][bad[0][1]]}: {have[tuple(bad[0])]} vs {want[tuple(bad[0])]}")


@pytest.mark.parametrize("qtype", TYPES)
def test_row_dots_match_the_reference(orc, qtype):
    """rows of eight blocks (accumulation across blocks, hsum_float_8, the summs chain) with edge blocks inside and at the end"""
    have = orc.quant_matmul(qtype, REF[f"rows_w_{qtype}"], REF["rows_act"]).T
    bad = np.argwhere(~same_bits(have, REF[f"rows_dot_{qtype}"]))
    assert bad.size == 0, f"{len(bad)} row dots differ, first at {tuple(bad[0])}"


def decode_blocks(qtype, W, K):
    """the integer codes [N][K] and, for q4_1 / q5_1, the f16 minima [N][K/32] of weight rows in file blocks"""
    bb = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}[qtype]
    N, nb = W.shape[0], K // 32
    blk = W.reshape(N, nb, bb)
    m = blk[:, :, 2:4].copy().view("<u2").reshape(N, nb).view(np.float16).astype(np.float64) if qtype in ("q4_1", "q5_1") else None
    if qtype == "q8_0":
        return blk[:, :, 2:].view(np.int8).astype(np.int64).reshape(N, K), None
    nib = blk[:, :, bb - 16:]
    codes = np.concatenate([nib & 15, nib >> 4], axis=2).astype(np.int64)
    if qtype in ("q5_0", "q5_1"):
        off = 2 if qtype == "q5_0" else 4
        qh = blk[:, :, off:off + 4].copy().view("<u4").reshape(N, nb, 1).astype(np.int64)
        codes |= ((qh >> np.arange(32)) & 1) << 4
    if qtype == "q4_0":
        codes -= 8
    if qtype == "q5_0":
        codes -= 16
    return codes.reshape(N, K), m


def exact(qtype, W, A):
    """[N][M] in float64: exact for these operands (every partial sum is an integer below 2^24)"""
    K = A.shape[1]
    codes, m = decode_blocks(qtype, W, K)
    qa = A.astype(np.int64)
    assert (np.abs(A).reshape(A.shape[0], -1, 32).max(2) == 127).all() and (qa == A).all()
    out = (codes @ qa.T).astype(np.float64)
    if m is not None:
        s = qa.reshape(A.shape[0], -1, 32).sum(2).astype(np.float64)        # d_a = 1: s = sum(q_a), f16-exact for |s| <= 2048
        assert (np.abs(s) <= 2048).all()
        out += m @ s.T
    return out


@pytest.mark.parametrize("qtype", TYPES)
def test_integer_rows_are_exact(orc, qtype):
    """d_w = 1 and amax 127 (d_a = 1): the reference's dot and the oracle's are exactly the integer sum, computed here with no
    restatement of either"""
    W, A = REF[f"int_w_{qtype}"], REF["int_act"]
    want = exact(qtype, W, A)
    assert np.array_equal(REF[f"int_dot_{qtype}"].astype(np.float64), want), "the stored reference dots are not the exact sums"
    assert np.array_equal(orc.quant_matmul(qtype, W, A).T.astype(np.float64), want)
