"""GPU: the parity path's four row reductions — layernorm_act_kernel and softmax_row (the multi-row passes and the attention kernels),
block_layernorm and softmax_exp_rcp (the persistent decode kernels) — against the C oracle (orc_norm x g + b, orc_soft_max) bit for
bit, through bark_b200_parity_rows.

Each kernel sums a row as a tree and replays the reference's sequential sum only when a bracket around the tree sum cannot settle
the float.  Random rows rarely reach that replay, so the rows here come from the builders in tests/test_reduction_orders.py, which
show on the CPU that the bracket fails on them and (where a tree exists) that the tree alone would round differently.  The hook's
replay count must be positive on those rows, and on random rows equal to the count the restated decisions give.  Also: soft_max
rows whose exps go through the -inf, underflow and subnormal branches of both exps, one built soft_max row through both attention
paths, and the replay inside the real decode kernels: a mini model whose embeddings put builder rows into layer 0's ln_1."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits
from test_reduction_orders import (LN_E, LN_IMPLS, NKV, SOFTMAX_IMPLS, Exps, f32, ln_cancel_row, ln_gain, ln_mean_row, ln_overflow_row,
                                   ln_random_rows, ln_var_row, softmax_built_row, softmax_multi, softmax_random_rows)

IMPLS = ["multi", "decode"]


@pytest.fixture(scope="module")
def ex(orc):
    return Exps(orc)


def ln_ref(ex, x, g, b):
    y = (ex.norm(x) * g).astype(f32)                     # ggml_norm, then ggml_mul (and ggml_add) in float
    return y if b is None else (y + b).astype(f32)


def same(got, want):
    bad = np.flatnonzero(bits(got) != bits(want))
    return bad.size == 0, f"{bad.size} of {got.size} differ, first at {np.unravel_index(bad[0], got.shape) if bad.size else None}"


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("E", LN_E)
@pytest.mark.parametrize("impl", IMPLS)
def test_layernorm_built_rows(pkg, ex, impl, E, bias):
    g, b = ln_gain(E)
    b = b if bias else None
    rows = {"mean": ln_mean_row(E), "variance": ln_var_row(E), "overflow": ln_overflow_row(E)}
    rows.update({f"cancel{s}": ln_cancel_row(E, s) for s in range(3)})
    for name, x in rows.items():
        got, replays = pkg.parity_rows(x, "layernorm", impl, g, b)
        ok, msg = same(got[0], ln_ref(ex, x, g, b))
        assert ok, f"{impl} E={E} {name}: {msg}"
        assert replays > 0, f"{impl} E={E} {name}: the bracket passed"


@pytest.mark.gpu
@pytest.mark.parametrize("E", LN_E)
@pytest.mark.parametrize("impl", IMPLS)
def test_layernorm_random_rows(pkg, ex, impl, E):
    g, b = ln_gain(E)
    x = ln_random_rows(E, 64, E)
    got, replays = pkg.parity_rows(x, "layernorm", impl, g, b)
    want = np.stack([ln_ref(ex, r, g, b) for r in x])
    ok, msg = same(got, want)
    assert ok, msg
    # rows whose mean is small against their spread have wide brackets: an occasional random row does take the replay, and the
    # kernel must take it exactly where the restated decision does
    restated = [LN_IMPLS[impl](r) for r in x]
    assert replays == sum(r["mean_replay"] + r["var_replay"] for r in restated)


@pytest.fixture(scope="module")
def built(ex):
    return {n: softmax_built_row(n, ex) for n in NKV}


@pytest.mark.gpu
@pytest.mark.parametrize("n", NKV)
@pytest.mark.parametrize("impl", IMPLS)
def test_softmax_built_and_random_rows(pkg, ex, built, impl, n):
    if built[n] is not None:                              # (n_kv = 1: no row forces the replay, see softmax_built_row)
        s, kind = built[n]
        got, replays = pkg.parity_rows(s, "softmax", impl)
        ok, msg = same(got[0], ex.soft_max(s))
        assert ok, f"{impl} n_kv={n} ({kind}): {msg}"
        assert replays > 0, f"{impl} n_kv={n} ({kind}): the bracket passed"
    s = softmax_random_rows(n, 64, 1000 + n)
    got, replays = pkg.parity_rows(s, "softmax", impl)
    ok, msg = same(got, np.stack([ex.soft_max(r) for r in s]))
    assert ok, f"{impl} n_kv={n} random: {msg}"
    assert replays == sum(SOFTMAX_IMPLS[impl](r, ex)["replay"] for r in s)


def exp_branch_inputs(count, seed):
    """count distinct scores below -19: uniform over [-104, -19] (subnormal results and glibc's underflow to 0 at -103.97) and over
    [-200, -87] (ggml_v_expf's |n| > 126 and |n| > 192 branches), runs of consecutive floats across each branch threshold, and -inf"""
    rng = np.random.default_rng(seed)
    runs = []
    for t in (-87.33654, -87.68, -88.72284, -103.97208, -103.28, -133.43):
        c = np.array([t], f32).view(np.int32)[0]
        runs.append((c + np.arange(-2000, 2000)).astype(np.int32).view(f32))
    x = np.concatenate(runs + [rng.uniform(-104, -19, count).astype(f32), rng.uniform(-200, -87, count).astype(f32), [f32(-np.inf)]])
    x = np.unique(x)
    rng.shuffle(x)
    assert x.size >= count
    return x[:count]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [8, 7])                   # 8: the vector exp for every column; 7: libm expf (the tail) for every column
@pytest.mark.parametrize("impl", IMPLS)
def test_softmax_exp_branches(pkg, ex, impl, n):
    per_row = n - 1
    x = exp_branch_inputs(2 ** 18, n)
    x = np.concatenate([x, np.full(-x.size % per_row, f32(-np.inf))]).reshape(-1, per_row)
    s = np.concatenate([np.zeros((x.shape[0], 1), f32), x], axis=1)      # the max is the 0 in column 0
    got, _ = pkg.parity_rows(s, "softmax", impl)
    want = np.stack([ex.soft_max(r) for r in s])
    ok, msg = same(got, want)
    assert ok, f"{impl} n_kv={n}: {msg}"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [33, 257, 1024])
def test_softmax_row_inside_attention(pkg, ex, orc, built, n):
    """A built row through parity_attention, both paths: one head of 64 (scale exactly 1/8), q = e0 and k_j = 8 s_j e0, so every
    score is exactly s_j; the output must be the oracle's P.V with P = orc_soft_max(s)."""
    s, kind = built[n]
    assert kind == "order"
    L = C.CDLL(orc.ORACLE_SO)
    L.orc_vec_dot_f32.restype = C.c_float
    L.orc_vec_dot_f32.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    D = 64
    q = np.zeros((1, D), f32); q[0, 0] = 1.0
    k = np.zeros((n, D), f32); k[:, 0] = f32(8) * s
    v = np.random.default_rng(n).standard_normal((n, D)).astype(f32)
    p = ex.soft_max(s)
    vt = np.ascontiguousarray(v.T)
    want = np.array([[L.orc_vec_dot_f32(n, vt[d].ctypes.data, p.ctypes.data) for d in range(D)]], f32)
    r = softmax_multi(s, ex)                              # what the kernel would give if it kept the bracket's low end instead
    p_lo = (r["e"] * r["f_lo"]).astype(f32)
    alt = np.array([[L.orc_vec_dot_f32(n, vt[d].ctypes.data, p_lo.ctypes.data) for d in range(D)]], f32)
    assert not np.array_equal(bits(alt), bits(want))
    for path in ("fused", "tiled"):
        got = pkg.parity_attention(q, k, v, 1, path=path)
        ok, msg = same(got, want)
        assert ok, f"{path} n_kv={n}: {msg}"


# ---- the replay inside the real decode kernels --------------------------------------------------------------------------------
ZERO_TOKEN = 7                                           # coarse token whose wte row is zero: its embedding at position p is wpe[p]
BUILT_POS = {5: "mean", 9: "variance", 12: "cancel"}     # positions whose wpe row is a LayerNorm builder row (layer 0's ln_1 input)


@pytest.fixture(scope="module")
def built_model(weights_mod, tmp_path_factory):
    """mini f16 (E = 256) with the coarse model's wte row ZERO_TOKEN zero and wpe rows BUILT_POS replaced by builder rows"""
    cfg = weights_mod.mini(weights_mod.F16)
    E, rng = cfg.coarse.n_embd, np.random.default_rng(5)
    wte = (0.02 * rng.standard_normal((cfg.coarse_vocab, E))).astype(f32)
    wte[ZERO_TOKEN] = 0.0
    wpe = (0.02 * rng.standard_normal((cfg.coarse.block_size, E))).astype(f32)
    make = {"mean": ln_mean_row, "variance": ln_var_row, "cancel": lambda E: ln_cancel_row(E, 0)}
    for p, kind in BUILT_POS.items():
        wpe[p] = make[kind](E)
    path = str(tmp_path_factory.mktemp("built") / "mini_built_f16.bin")
    return weights_mod.write_weights(path, cfg, overrides={"coarse/model/wte/0": wte, "coarse/model/wpe": wpe})


def zeros(n):
    return np.full(n, ZERO_TOKEN, np.int32)


@pytest.mark.gpu
def test_replay_in_a_coarse_prefill(pkg, orc, built_model):
    with pkg.Bark(built_model) as b:
        before = b.layernorm_fallbacks()
        lg, n = b.gpt_eval(1, zeros(16), 0, False)
        lo, no = orc.Oracle(built_model).gpt_eval(1, zeros(16), 0, False)
        assert n == no and np.array_equal(bits(lg), bits(lo)), f"{int((lg != lo).sum())} logits differ"
        assert b.layernorm_fallbacks() > before


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["grid", "multi"])
def test_replay_in_single_token_steps(pkg, orc, built_model, monkeypatch, mode):
    """BARK_B200_DECODE unset: gpt_decode_step_kernel; multi: one kernel per op"""
    monkeypatch.delenv("BARK_B200_DECODE", raising=False)
    if mode != "grid":
        monkeypatch.setenv("BARK_B200_DECODE", mode)
    o = orc.Oracle(built_model)
    with pkg.Bark(built_model) as b:
        lg, n = b.gpt_eval(1, zeros(4), 0, False)
        lo, no = o.gpt_eval(1, zeros(4), 0, False)
        assert np.array_equal(bits(lg), bits(lo))
        before = b.layernorm_fallbacks()
        for pos in range(4, 14):                          # steps at positions 4 .. 13, crossing every built position
            lg, n = b.gpt_eval(1, zeros(1), n, False)
            lo, no = o.gpt_eval(1, zeros(1), no, False)
            assert n == no and np.array_equal(bits(lg), bits(lo)), f"{mode}, step at position {pos}: {int((lg != lo).sum())} logits differ"
        assert b.layernorm_fallbacks() > before, mode


@pytest.mark.gpu
def test_replay_in_a_batched_step(pkg, orc, built_model):
    slots, pos = [2, 5, 0], sorted(BUILT_POS)             # one row per built position
    oracles = [orc.Oracle(built_model) for _ in slots]
    with pkg.Bark(built_model) as b:
        for s, p, o in zip(slots, pos, oracles):
            lg, n = b.gpt_eval_slot(1, s, zeros(p), 0, False)
            lo, no = o.gpt_eval(1, zeros(p), 0, False)
            assert n == no == p and np.array_equal(bits(lg), bits(lo))
        before = b.layernorm_fallbacks()
        lg, n_past = b.gpt_step_batch(1, slots, zeros(len(slots)), pos)
        for r, (p, o) in enumerate(zip(pos, oracles)):
            lo, no = o.gpt_eval(1, zeros(1), p, False)
            assert n_past[r] == no and np.array_equal(bits(lg[r]), bits(lo)), f"row {r} at position {p}: {int((lg[r] != lo).sum())} logits differ"
        assert b.layernorm_fallbacks() > before
