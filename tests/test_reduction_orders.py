"""CPU restatements of the parity path's reductions — the bit-exactness arguments, executable.

1. p2_scores reduces EIGHT dot products together with a transposed butterfly (stages xor 16, 8, 4 swap halves of the per-lane values,
   then xor 1 and xor 2 on the survivor).  Claim: for every task the result is bit-identical to lane_tree_reduce (common.cuh), the
   reference's GGML_F32x8_REDUCE order (ggml.c:1405-1422), and it ends up on the lanes the kernel publishes from.
2. block_layernorm combines the 16 warp partials with a 4-level xor butterfly started from partial[lane & 15].  Claim: every lane
   ends with the same bits (the bracket logic needs all threads to take the same decision).
3. The four row reductions whose bracket decides when to replay the reference's sequential sum (LayerNorm, soft_max; below), and
   rows built so that the bracket must refuse them.
IEEE float32 / float64 additions in numpy are the same operations as __fadd_rn / DADD.
"""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from conftest import bits


def lane_tree_reduce(a):
    """a: [32] float32 lane partials -> [32] results (every lane), stage order xor 16, 8, 4, 1, 2."""
    a = a.astype(np.float32).copy()
    lanes = np.arange(32)
    for m in (16, 8, 4, 1, 2):
        a = (a + a[lanes ^ m]).astype(np.float32)
    return a


def transposed_butterfly(r):
    """r: [32 lanes][8 tasks] float32 -> (value per lane, task index per lane), as written in p2_scores."""
    r = r.astype(np.float32).copy()
    lanes = np.arange(32)
    u16, u8, u4 = (lanes & 16) != 0, (lanes & 8) != 0, (lanes & 4) != 0
    new = r.copy()
    for i in range(4):
        keep = np.where(u16, r[:, i + 4], r[:, i]); send = np.where(u16, r[:, i], r[:, i + 4])
        new[:, i] = (keep + send[lanes ^ 16]).astype(np.float32)
    r = new.copy()
    for i in range(2):
        keep = np.where(u8, r[:, i + 2], r[:, i]); send = np.where(u8, r[:, i], r[:, i + 2])
        new[:, i] = (keep + send[lanes ^ 8]).astype(np.float32)
    r = new.copy()
    keep = np.where(u4, r[:, 1], r[:, 0]); send = np.where(u4, r[:, 0], r[:, 1])
    v = (keep + send[lanes ^ 4]).astype(np.float32)
    v = (v + v[lanes ^ 1]).astype(np.float32)
    v = (v + v[lanes ^ 2]).astype(np.float32)
    mine = u16 * 4 + u8 * 2 + u4 * 1
    return v, mine


def test_transposed_butterfly_is_lane_tree_reduce_per_task():
    rng = np.random.default_rng(0)
    for trial in range(200):
        scale = np.float32(10.0 ** rng.integers(-6, 6))
        r = (rng.standard_normal((32, 8)) * scale).astype(np.float32)
        if trial % 7 == 0: r[rng.integers(0, 32), rng.integers(0, 8)] = np.float32(1e30)     # cancellation-prone cases
        v, mine = transposed_butterfly(r)
        for lane in range(32):
            ref = lane_tree_reduce(r[:, mine[lane]])
            assert v[lane].tobytes() == ref[lane].tobytes(), (trial, lane, mine[lane])
        # the publishing lanes (lane & 3 == 0) cover the eight tasks exactly once
        assert sorted(mine[np.arange(32) % 4 == 0].tolist()) == list(range(8))


def test_layernorm_partial_butterfly_gives_every_lane_the_same_bits():
    rng = np.random.default_rng(1)
    lanes = np.arange(32)
    for trial in range(200):
        part = (rng.standard_normal(16) * 10.0 ** rng.integers(-8, 8)).astype(np.float64)
        q = part[lanes & 15].copy()
        for o in (8, 4, 2, 1):
            q = q + q[lanes ^ o]
        assert len({x.tobytes() for x in q}) == 1
        # and it is the pairwise tree the previous per-thread version computed: ((p0+p8)+(p4+p12)) + ...
        t = part.copy()
        for st in (8, 4, 2, 1):
            t[:st] = t[:st] + t[st:2 * st]
        assert q[0].tobytes() == t[0].tobytes()


# ================================================================================================================================
# The row reductions behind bit-identical token ids: LayerNorm (layernorm_act_kernel, gpt_kernels.cu; block_layernorm,
# decode_kernels.cu) and soft_max (softmax_row, epilogue.cuh; softmax_exp_rcp, decode_kernels.cu).  The reference sums every row
# sequentially in double (oracle/bark_oracle.c orc_norm, orc_soft_max); the kernels sum it as a tree, widen the tree sum into a
# bracket and replay the sequential loop when the two ends of the bracket give different floats.  Below: each kernel's summation
# order and bracket decision restated exactly as written, and row builders whose rows the bracket must refuse — for most of them
# the tree alone would give a different float than the sequential sum.  tests/test_parity_rows_gpu.py runs the same rows on the
# GPU against the oracle.
# ================================================================================================================================
f32 = np.float32
LANES = np.arange(32)
EPS = f32(1e-5)


def _fma(a, b, c):
    """double fma, rounded once (IEEE)"""
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _butterfly(v, levels):
    """xor butterfly over the last axis (32 lanes, or 16 partials indexed lane & 15): v[l] += v[l ^ o] per level, dtype kept"""
    v = v.copy()
    idx = np.arange(v.shape[-1])
    for o in levels:
        v = v + v[..., idx ^ o]
    return v


def _seq(vals):
    s = 0.0
    for v in vals:
        s += float(v)
    return s


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------------
def ln_reference(x, g, b=None):
    """orc_norm (the reference's ggml_compute_forward_norm_f32) x g (+ b), restated: sequential double sums"""
    E = x.size
    with np.errstate(all="ignore"):
        mean = f32(_seq(x) / E)
        v = (x - mean).astype(f32)
        var = f32(_seq((v * v).astype(f32)) / E)
        scale = f32(1.0) / np.sqrt(f32(var + EPS))
        y = ((v * scale).astype(f32) * g).astype(f32)
        return y if b is None else (y + b).astype(f32)


def ln_multi(x, g=None, b=None, force_pass=False):
    """layernorm_act_kernel: lane l sums x[l], x[l+32], ... in double, then the xor butterfly 16..1; mean and variance each bracketed
    by +-slack * sum|x| (sum of squares for the variance) before the division.  Returns a dict: the tree floats, the sequential
    floats, which bracket failed, the output."""
    E = x.size
    xp = np.zeros((E + 31) // 32 * 32, f32); xp[:E] = x
    slack = 2.0 * float(E) * 2.0 ** -53 * (1.0 + 1e-6)
    r = {}
    with np.errstate(all="ignore"):
        xd = xp.reshape(-1, 32).astype(np.float64)
        s = a = np.zeros(32)
        for row in xd:
            s = s + row; a = a + np.abs(row)
        s = float(_butterfly(s, (16, 8, 4, 2, 1))[0]); a = float(_butterfly(a, (16, 8, 4, 2, 1))[0])
        d = slack * a
        r["mean_tree"] = mean = f32(s / E)
        r["mean_seq"] = f32(_seq(x) / E)
        r["mean_replay"] = bool(f32((s - d) / E) != f32((s + d) / E)) and not force_pass
        if r["mean_replay"]:
            mean = r["mean_seq"]
        v = (x - mean).astype(f32)
        vp = np.zeros_like(xp); vp[:E] = (v * v).astype(f32)
        s2 = np.zeros(32)
        for row in vp.reshape(-1, 32).astype(np.float64):
            s2 = s2 + row
        s2 = float(_butterfly(s2, (16, 8, 4, 2, 1))[0])
        d = slack * s2
        r["var_tree"] = var = f32(s2 / E)
        r["var_seq"] = f32(_seq((v * v).astype(f32)) / E)
        r["var_replay"] = bool(f32((s2 - d) / E) != f32((s2 + d) / E)) and not force_pass
        if r["var_replay"]:
            var = r["var_seq"]
        if g is not None:
            scale = f32(1.0) / np.sqrt(f32(var + EPS))
            y = ((v * scale).astype(f32) * g).astype(f32)
            r["out"] = y if b is None else (y + b).astype(f32)
    return r


def ln_block(x, g=None, b=None, force_pass=False):
    """block_layernorm (512 threads): thread t owns x[t] and x[t + 512], its double sum goes through the warp butterfly 16..1, the 16
    warp partials through the butterfly 8, 4, 2, 1 started from partial[lane & 15].  The decision multiplies by inv_E = 1/E and widens
    the half-width by the reciprocal's error (2^-50 |c|) and, for the mean, the float |x| sum's error (1.001)."""
    E = x.size
    assert E <= 1024
    xp = np.zeros(1024, f32); xp[:E] = x
    h = np.arange(1024) < E
    slack = 2.0 * float(E) * 2.0 ** -53 * (1.0 + 1e-6)
    inv_E = 1.0 / E
    r = {}

    def block_sum(t):                       # t: [512] per-thread doubles (or floats) -> the butterfly result every thread holds
        w = _butterfly(t.reshape(16, 32), (16, 8, 4, 2, 1))[:, 0]
        return _butterfly(w[LANES & 15], (8, 4, 2, 1))[0]

    with np.errstate(all="ignore"):
        x0, x1 = xp[:512], xp[512:]
        S = float(block_sum(x0.astype(np.float64) + x1.astype(np.float64)))
        A = float(block_sum((np.abs(x0) + np.abs(x1)).astype(f32)))
        c = S * inv_E
        hw = (slack * A * 1.001) * inv_E + abs(c) * 2.0 ** -50
        mean = f32(c - hw)
        r["mean_tree"] = f32(S / E)
        r["mean_seq"] = f32(_seq(x) / E)
        r["mean_replay"] = bool(mean != f32(c + hw)) and not force_pass
        if r["mean_replay"]:
            mean = r["mean_seq"]
        v = (xp - mean).astype(f32)
        sq = np.where(h, (v * v).astype(f32).astype(np.float64), 0.0)
        S2 = float(block_sum(sq[:512] + sq[512:]))
        c = S2 * inv_E
        hw = (slack * S2) * inv_E + c * 2.0 ** -50
        var = f32(c - hw)
        r["var_tree"] = f32(S2 / E)
        r["var_seq"] = f32(_seq((v[:E] * v[:E]).astype(f32)) / E)
        r["var_replay"] = bool(var != f32(c + hw)) and not force_pass
        if r["var_replay"]:
            var = r["var_seq"]
        if g is not None:
            scale = f32(1.0) / np.sqrt(f32(var + EPS))
            y = ((v[:E] * scale).astype(f32) * g).astype(f32)
            r["out"] = y if b is None else (y + b).astype(f32)
    return r


LN_IMPLS = {"multi": ln_multi, "decode": ln_block}


def ln_mean_row(E):
    """Order-discriminating mean: x[0] = E and x[32] = 3E 2^-24 (lane 0 / thread 0 and thread 32), so the sequential mean is exactly
    the float midpoint 1 + 3 2^-24, which rounds to even: up, to 1 + 2^-22.  Four d = -(double ulp of E) / 4 sit in x[1], x[17], x[9],
    x[25]: the warp butterfly adds them to each other (16, then 8) before they meet x[0]'s lane, so the tree sum is one double ulp
    lower and its mean rounds down; the sequential sum loses each d against E.  The sequential float is the upper one, so a decision
    that kept the bracket's low end (block_layernorm) would be wrong too."""
    x = np.zeros(E, f32)
    x[0] = E; x[32] = f32(3 * E * 2.0 ** -24)
    d = f32(-np.spacing(np.float64(E)) / 4)
    for i in (1, 17, 9, 25):
        x[i] = d
    return x


def ln_var_row(E):
    """Order-discriminating variance on a row whose mean is exactly 0 (every partial sum exact): lane 0 / the lane-0 threads hold
    E/128 pairs +-1 and E/128 pairs +-2^-12, so the sequential sum of squares is (E/64)(1 + 2^-24) and the variance the float midpoint
    2^-6 (1 + 2^-24), which rounds to even (down).  Four +-d in the last 32 columns, lanes 1, 17, 9, 25, have squares D of a fraction
    of the double ulp of that sum: lost one by one sequentially, added up by the tree into more than half an ulp, so the tree's
    variance rounds up."""
    x = np.zeros(E, f32)
    k = E // 128
    x[0:E:32] = [1.0, -1.0] * k + [2.0 ** -12, -2.0 ** -12] * k
    e = math.floor(math.log2(2 * k))                      # the sum of squares lies in [2^e, 2^(e+1))
    d = 1.25 * 2.0 ** ((e - 54) / 2) if e % 2 == 0 else 1.25 * 2.0 ** ((e - 55) / 2)
    for i, s in zip((1, 17, 9, 25), (1, 1, -1, -1)):
        x[E - 32 + i] = s * d
    return x


def ln_cancel_row(E, seed):
    """+-2^60 around small values: the mean depends on the summation order by far more than one ulp"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(E).astype(f32)
    x[3] = f32(2.0 ** 60); x[E - 5] = f32(-2.0 ** 60)
    return x


def ln_overflow_row(E):
    """v * v overflows to inf while x - mean stays finite: the variance brackets compare NaN ends (inf - inf) and replay, the
    variance is inf, the scale 0 and every output a signed zero (times g, plus b)"""
    x = np.zeros(E, f32)
    x[0:8] = [3e19, -3e19, 2e19, -2e19, 1.0, -1.0, 5.0, -5.0]
    return x


def ln_random_rows(E, n, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, E)) * rng.choice([0.02, 1.0, 30.0], (n, 1)) + rng.standard_normal((n, 1))).astype(f32)


LN_E = [128, 256, 768, 1024]


def ln_gain(E, seed=7):
    rng = np.random.default_rng(seed)
    return (1.0 + 0.02 * rng.standard_normal(E)).astype(f32), (0.02 * rng.standard_normal(E)).astype(f32)


@pytest.mark.parametrize("impl", list(LN_IMPLS))
@pytest.mark.parametrize("E", LN_E)
def test_layernorm_builders_defeat_the_tree(impl, E):
    f = LN_IMPLS[impl]
    g, b = ln_gain(E)
    r = f(ln_mean_row(E), g, b)
    assert r["mean_replay"] and r["mean_tree"] != r["mean_seq"], (r["mean_tree"], r["mean_seq"])
    assert r["mean_seq"] == f32(1 + 2.0 ** -22)
    r = f(ln_var_row(E), g, b)
    assert r["var_replay"] and r["var_tree"] != r["var_seq"], (r["var_tree"], r["var_seq"])
    for seed in range(3):
        r = f(ln_cancel_row(E, seed), g, b)
        assert r["mean_replay"] and abs(float(r["mean_tree"]) - float(r["mean_seq"])) > 1e-3 * abs(float(r["mean_seq"]))
    r = f(ln_overflow_row(E), g, b)
    assert r["var_replay"] and np.isinf(r["var_seq"])
    assert np.array_equal(bits(r["out"]), bits(ln_reference(ln_overflow_row(E), g, b)))


@pytest.mark.parametrize("impl", list(LN_IMPLS))
@pytest.mark.parametrize("E", LN_E)
def test_layernorm_restatement_matches_the_reference_and_random_rows_do_not_replay(impl, E):
    f = LN_IMPLS[impl]
    g, b = ln_gain(E)
    for x in [ln_mean_row(E), ln_var_row(E), ln_cancel_row(E, 0), ln_overflow_row(E)]:
        assert np.array_equal(bits(f(x, g, b)["out"]), bits(ln_reference(x, g, b)))
    for x in ln_random_rows(E, 16, E):
        r = f(x, g, b)
        assert not r["mean_replay"] and not r["var_replay"]
        assert np.array_equal(bits(r["out"]), bits(ln_reference(x, g, b)))


@pytest.mark.parametrize("impl", list(LN_IMPLS))
@pytest.mark.parametrize("E", LN_E)
def test_layernorm_forced_pass_would_be_wrong(impl, E):
    """A bracket that always passed (the decision without its replay) gives a different output than the reference on the built
    rows: what the GPU tests would see if a kernel's bracket were too narrow."""
    f = LN_IMPLS[impl]
    g, b = ln_gain(E)
    # (block_layernorm keeps the low end of the bracket, which on ln_var_row is the sequential float: ln_mean_row is built for it)
    for x in [ln_mean_row(E)] + ([ln_var_row(E)] if impl == "multi" else []):
        assert not np.array_equal(bits(f(x, g, b, force_pass=True)["out"]), bits(ln_reference(x, g, b))), impl


# ---- soft_max ------------------------------------------------------------------------------------------------------------------
class Exps:
    """ggml_v_expf (orc_v_expf, the oracle's restatement of the 8-wide AVX2 polynomial) and libm expf (the n_kv % 8 tail)"""

    def __init__(self, orc):
        L = C.CDLL(orc.ORACLE_SO)
        L.orc_v_expf.restype = C.c_float; L.orc_v_expf.argtypes = [C.c_float]
        L.orc_soft_max.restype = None; L.orc_soft_max.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        L.orc_norm.restype = None; L.orc_norm.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_float]
        m = C.CDLL("libm.so.6")
        m.expf.restype = C.c_float; m.expf.argtypes = [C.c_float]
        self.L, self.m = L, m

    def v(self, a):
        return np.array([self.L.orc_v_expf(float(t)) for t in np.ravel(a)], f32).reshape(np.shape(a))

    def tail(self, a):
        return np.array([self.m.expf(float(t)) for t in np.ravel(a)], f32).reshape(np.shape(a))

    def soft_max(self, s):
        s = np.ascontiguousarray(s, f32); p = np.empty_like(s)
        self.L.orc_soft_max(s.size, s.ctypes.data, p.ctypes.data)
        return p

    def norm(self, x):
        x = np.ascontiguousarray(x, f32); y = np.empty_like(x)
        self.L.orc_norm(x.size, x.ctypes.data, y.ctypes.data, EPS)
        return y


def _chunk_sums(e8):
    """the in-chunk float tree of the 8-wide code: (hi128 + lo128), then movehl, then movehdup"""
    t0, t1, t2, t3 = e8[:, 4] + e8[:, 0], e8[:, 5] + e8[:, 1], e8[:, 6] + e8[:, 2], e8[:, 7] + e8[:, 3]
    return ((t0 + t2) + (t1 + t3)).astype(f32)


def _softmax_decision(tsum, nchunks, tail, csum, force_pass):
    """the bracket both soft_max implementations take on the tree sum (identical code in softmax_row and softmax_exp_rcp)"""
    r = {}
    dl = 2.0 * float(nchunks + 8) * 2.0 ** -53 * tsum * (1.0 + 1e-6)
    lo, hi = tsum - dl, tsum + dl
    tt = tsum
    for t in tail:
        lo += float(t); hi += float(t); tt += float(t)
    mid = 0.5 * (lo + hi)
    y = float(f32(1.0) / f32(mid))                         # __frcp_rn((float) mid), then two Newton steps
    e = _fma(-mid, y, 1.0); y = _fma(y, e, y)
    e = _fma(-mid, y, 1.0); y = _fma(y, e, y)
    rw = (hi - lo) * y * 0.5 + 2.0 ** -48
    r["f_lo"] = sc = f32(y * (1.0 - rw))
    r["replay"] = bool(sc != f32(y * (1.0 + rw))) and not force_pass
    seq = _seq(list(csum) + list(tail))
    r["sc_seq"] = f32(1.0 / seq)
    r["sc_tree"] = f32(1.0 / tt)
    r["sc"] = r["sc_seq"] if r["replay"] else sc
    return r


def softmax_multi(s, ex, force_pass=False):
    """softmax_row (one warp): chunk c of 8 columns belongs to lane c % 32, slot c / 32; lane l's double sum adds its slots 0..3 (zero
    where it owns no chunk), then the xor butterfly 16..1; the n % 8 tail (libm expf) is added to both ends of the bracket."""
    n = s.size
    nc = n >> 3
    with np.errstate(all="ignore"):
        d = (s - s.max()).astype(f32)
    e = np.concatenate([ex.v(d[:8 * nc]), ex.tail(d[8 * nc:])]).astype(f32)
    csum = _chunk_sums(e[:8 * nc].reshape(nc, 8))
    slots = np.zeros((4, 32), f32)
    slots.reshape(-1)[:nc] = csum
    tsum = np.zeros(32)
    for slot in range(4):
        tsum = tsum + slots[slot].astype(np.float64)
    tsum = float(_butterfly(tsum, (16, 8, 4, 2, 1))[0])
    r = _softmax_decision(tsum, nc, e[8 * nc:], csum, force_pass)
    r["e"], r["out"] = e, (e * r["sc"]).astype(f32)
    return r


def softmax_decode(s, ex, force_pass=False):
    """softmax_exp_rcp (warp 0 of the block): lane l adds the chunk sums c = l, l + 32, ... in order, then the xor butterfly 16..1.
    Adding a zero slot is exact, so this is softmax_row's tree; restated separately all the same.  P.V forms p * (1/sum)."""
    n = s.size
    nc = n >> 3
    with np.errstate(all="ignore"):
        d = (s - s.max()).astype(f32)
    e = np.concatenate([ex.v(d[:8 * nc]), ex.tail(d[8 * nc:])]).astype(f32)
    csum = _chunk_sums(e[:8 * nc].reshape(nc, 8))
    lane = np.zeros(32)
    for l in range(32):
        acc = 0.0
        for c in range(l, nc, 32):
            acc += float(csum[c])
        lane[l] = acc
    tsum = float(_butterfly(lane, (16, 8, 4, 2, 1))[0])
    r = _softmax_decision(tsum, nc, e[8 * nc:], csum, force_pass)
    r["e"], r["out"] = e, (e * r["sc"]).astype(f32)
    return r


SOFTMAX_IMPLS = {"multi": softmax_multi, "decode": softmax_decode}
NKV = [1, 7, 8, 9, 33, 257, 1024]
ZERO = f32(-200.0)                                       # exp(-200 - 0) is exactly 0 through both exps


def _largest_input_below(fn, target, lo=-104.0):
    """the largest float x in [lo, 0] with fn(x) <= target, for fn increasing: bisection over the bit patterns of negative floats"""
    key = lambda x: -int(np.array(abs(x), f32).view(np.int32))
    val = lambda k: -np.array(-k, np.int32).view(f32)
    a, b = key(lo), 0                                    # fn(lo) <= target < fn(0) = 1
    while b - a > 1:
        m = (a + b) // 2
        if float(fn(val(m))) <= target:
            a = m
        else:
            b = m
    return f32(val(a))


def _single_chunk_row(ex, vexp):
    """n_kv = 8: the sum is the float S = fl(1 + e(x_a)).  Floats S in [1, 2) whose 1/S falls inside the bracket around a float
    midpoint are rare (about one in 2^22): find them all at once, then the x_a that gives one of them."""
    S = (np.arange(2 ** 23, dtype=np.int64) + 0x3f800000).astype(np.int32).view(f32).astype(np.float64)
    y = 1.0 / S
    rw = 2.0 * 2 * 9 * 2.0 ** -53 * S * (1.0 + 1e-6) * y * 0.5 + 2.0 ** -48
    cand = np.flatnonzero((y * (1 - rw)).astype(f32) != (y * (1 + rw)).astype(f32))
    for i in cand:
        target = S[i]
        xa = _largest_input_below(lambda x: f32(1) + vexp(x), target)
        s = np.full(8, ZERO, f32); s[0] = 0.0; s[1] = xa
        if _chunk_sums(np.array([[1, vexp(xa), 0, 0, 0, 0, 0, 0]], f32))[0] == target and softmax_multi(s, ex)["replay"]:
            return s
    raise AssertionError("no one-chunk row")


def softmax_built_row(n, ex):
    """Scores of n_kv = n whose 1/sum lands within the bracket of a float midpoint M.  The sum is steered to 1/M by three tuned terms:
    a chunk [0, x_a, zeros] with chunk sum 1 + e(x_a) in [1, 2) (one float ulp of control), then e(x_c) near 2^-24 and e(x_d) near 2^-43
    (libm expf in the tail when n % 8 != 0, else the vector exp); every other column is -200 (exp exactly 0).  Where the tree exists,
    the odd lanes' chunks (1, 3, 5, 7) each hold one t of about 3/8 of a double ulp of the sum: sequentially each t is lost, the
    butterfly adds them up on the odd lanes before they meet lane 0, so the tree sum is an ulp higher and float(1/sum) differs.
    Returns (scores, kind) with kind "order" (tree and sequential floats differ) or "replay" (the bracket fails but no tree exists
    that could differ: n_kv < 33 has at most one chunk), or None when no row can force the replay (n_kv = 1: the sum is exactly 1)."""
    nc, tail = n >> 3, n & 7
    if n == 1:
        return None
    vexp = lambda x: ex.v(np.array([x], f32))[0]
    lexp = lambda x: ex.tail(np.array([x], f32))[0]
    if nc >= 4 and (tail or nc >= 65):
        kind = "order"
        odd = [c for c in (1, 3, 5, 7) if c < nc]
        pos_c = 2 * 8 if tail else 32 * 8                 # cC: chunk 2 (lane 2, meets lane 0 at xor 2) or chunk 32 (lane 0, slot 1)
        pos_d, fd = (nc * 8, lexp) if tail else (64 * 8, vexp)
    elif n == 8:                                          # one chunk, no tail: the sum is one float S = 1 + e(x_a)
        return _single_chunk_row(ex, vexp), "replay"
    elif nc == 1:                                         # one chunk and a tail: the chunk sum, then e(x_d) in the tail
        kind, odd, pos_c, pos_d, fd = "replay", [], None, 8, lexp
    else:                                                 # no chunk: 1 + e(x_a) + e(x_c) + e(x_d), all in the tail
        kind, odd, pos_c, pos_d, fd = "replay", [], 2, 3, lexp
    fc = lexp if (pos_c is not None and pos_c >= 8 * nc) else vexp
    fa = lexp if nc == 0 else vexp
    for k in range(int(0.70 * 2 ** 24), int(0.70 * 2 ** 24) + 4000):
        M = Fraction(2 * k + 1, 2 ** 25)                  # float midpoint in (0.5, 1)
        T = 1 / M
        s = np.full(n, ZERO, f32)
        s[0] = 0.0
        xa = _largest_input_below(fa, float(T - 1) - 2.0 ** -22)
        s[1] = xa
        cA = float(f32(1) + fa(xa)) if nc >= 1 else 1.0 + float(fa(xa))
        R1 = T - Fraction(cA)
        P = cA
        if pos_c is not None:
            xc = _largest_input_below(fc, float(R1) * (1 - 2.0 ** -16))
            s[pos_c] = xc
            P = cA + float(fc(xc))
        R2 = float(T - Fraction(P))
        if R2 <= 0:
            continue
        if odd:
            t_target = 0.375 * 2.0 ** -52
            xt = _largest_input_below(vexp, t_target)
            for c in odd:
                s[8 * c] = xt
        xd = _largest_input_below(fd, R2)
        for step in range(-40, 41):
            cand = xd
            for _ in range(abs(step)):
                cand = np.nextafter(cand, f32(0) if step > 0 else f32(-200))
            s[pos_d] = cand
            r = softmax_multi(s, ex)
            if not r["replay"]:
                continue
            if kind == "replay" or (r["sc_tree"] != r["sc_seq"] and r["f_lo"] != r["sc_seq"]):
                return s.copy(), kind
    raise AssertionError(f"no built row for n_kv = {n}")


def softmax_random_rows(n, rows, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((rows, n)) * rng.choice([0.1, 1.0, 4.0, 20.0], (rows, 1))).astype(f32)


@pytest.fixture(scope="module")
def exps(orc):
    return Exps(orc)


@pytest.fixture(scope="module")
def built_softmax(exps):
    return {n: softmax_built_row(n, exps) for n in NKV}


@pytest.mark.parametrize("impl", list(SOFTMAX_IMPLS))
@pytest.mark.parametrize("n", NKV)
def test_softmax_builders_defeat_the_tree(exps, built_softmax, impl, n):
    f = SOFTMAX_IMPLS[impl]
    if built_softmax[n] is None:
        assert n == 1          # one column: the sum is exactly 1, 1/sum exactly 1, and both ends of the bracket round there
        return
    s, kind = built_softmax[n]
    r = f(s, exps)
    assert r["replay"], n
    if kind == "order":
        assert r["sc_tree"] != r["sc_seq"], n
        assert r["f_lo"] != r["sc_seq"], n
        assert not np.array_equal(bits(f(s, exps, force_pass=True)["out"]), bits(exps.soft_max(s)))
    else:
        assert n < 33          # at most one chunk: the tree and the sequential order add the same terms in the same order
    assert np.array_equal(bits(r["out"]), bits(exps.soft_max(s)))


@pytest.mark.parametrize("n", NKV)
def test_softmax_restatements_agree_and_random_rows_do_not_replay(exps, n):
    for s in softmax_random_rows(n, 12, n):
        a, b = softmax_multi(s, exps), softmax_decode(s, exps)
        assert not a["replay"] and not b["replay"]
        assert np.array_equal(bits(a["out"]), bits(b["out"]))
        assert np.array_equal(bits(a["out"]), bits(exps.soft_max(s)))
