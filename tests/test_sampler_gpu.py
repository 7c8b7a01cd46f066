"""GPU: sample_rows_kernel at 256 and 1024 threads on the rows tests/test_sampler_orders.py builds on the decision edges, through
bark_b200_sample_given_u, against the C oracle (orc_sample_u) with the same uniform.

Per row: the final token and the eos_p bits equal the oracle's; the kernel flags every row the restated threshold bracket refuses; and
where no entry's glibc exp lies within 2^-48 of a float midpoint (so CUDA's exp rounds the same and the exp bracket is quiet on both),
the kernel's flags and its own tokens before the replay (device_tokens) equal the restated device order exactly.  Among the threshold
rows of every width and thread count some are decisive: the kernel's own token is wrong there and only the replay makes it right.
"""
import math

import numpy as np
import pytest

from conftest import bits
from test_sampler_orders import (EXP_MIDPOINTS, THREADS, THRESHOLD_SHAPES, argmax_cases, canonical, device_pick, device_runs, device_sample,
                                 edge_cases, exp_cases, f32, f64, ref_probs, threshold_cases)

# How many fixture x (tests/golden/sampler/exp_midpoints.npz) CUDA's double exp, rounded to float, sends to the other float than glibc's:
# measured by test_exp_rounding_against_glibc on an H100 80GB HBM3 (CUDA 12.9), at both thread counts.  A toolkit whose exp rounds
# differently makes this test fail; the tokens stay right as long as the exp bracket fires.
CUDA_EXP_ROUNDS_DIFFERENTLY = 0


def run_rows(pkg, l, temp, us, T):
    """The hook on one logits row repeated for every u (at most 1024 rows per call)."""
    outs = []
    for s in range(0, us.size, 1024):
        u = us[s:s + 1024]
        outs.append(pkg.sample_given_u(np.repeat(l[None], u.size, 0), temp, u, T))
    return {k: np.concatenate([o[k] for o in outs]) for k in ("tokens", "device_tokens", "flags", "eos_p")}


def check_rows(pkg, orc, name, l, temp, us, T):
    """All assertions of the module docstring for one case; returns the number of decisive rows."""
    out = run_rows(pkg, l, temp, us, T)
    want = [orc.sample_u(l, temp, u) for u in us]
    for r, (t, e) in enumerate(want):
        assert out["tokens"][r] == t and bits(out["eos_p"][r]) == bits(f32(e)), \
            f"{name} T={T} u={us[r].hex()}: token {out['tokens'][r]} (device {out['device_tokens'][r]}), oracle {t}"
    tok, flag, margin = device_sample(l, temp, us, T)
    if temp != 0:
        p, _ = ref_probs(l, temp)
        runs, total = device_runs(p, T)
        _, thr_flag = device_pick(runs, total, p.size, us)
        assert out["flags"][thr_flag].all(), f"{name} T={T}: a row the threshold bracket refuses was not flagged"
    if margin > 2.0 ** -48:
        assert np.array_equal(out["flags"] != 0, flag), f"{name} T={T}: flags differ from the restatement"
        assert np.array_equal(out["device_tokens"], tok), f"{name} T={T}: the kernel's tokens differ from the restated device order"
    return int((out["device_tokens"] != out["tokens"]).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("T", THREADS)
@pytest.mark.parametrize("n, temp", THRESHOLD_SHAPES)
def test_threshold_rows(pkg, orc, n, temp, T):
    decisive = sum(check_rows(pkg, orc, name, l, t, us, T) for name, l, t, us in threshold_cases(n, temp))
    assert decisive > 0, f"n={n} temp={temp} T={T}: no row where the threshold bracket decided the token"


@pytest.mark.gpu
@pytest.mark.parametrize("T", THREADS)
def test_edge_rows(pkg, orc, T):
    for name, l, temp, us in edge_cases():
        check_rows(pkg, orc, name, l, temp, us, T)


@pytest.mark.gpu
@pytest.mark.parametrize("T", THREADS)
def test_argmax_rows(pkg, orc, T):
    for name, l, temp, us in argmax_cases(T):
        check_rows(pkg, orc, name, l, temp, us, T)


@pytest.mark.gpu
@pytest.mark.parametrize("T", THREADS)
def test_exp_rows(pkg, orc, T):
    for name, l, temp, us in exp_cases():
        check_rows(pkg, orc, name, l, temp, us, T)
        assert pkg.sample_given_u(l, temp, us[:1], T)["flags"][0] == 1, f"{name} T={T}: the exp bracket did not fire"


def exp_reveal_rows(x, T):
    """For fixture x: the row [x / 2, 0] at temp 0.5 (l - max = x exactly), the two floats A (glibc's rounding of exp(x)) and B (the
    float on the other side of the nearest midpoint), and a u between the two outcomes: the kernel's own token is 0 for one of them
    and 1 for the other, so device_tokens tells which float CUDA's exp rounded to.  Returns (logits, u, token with A, token with B)."""
    l = np.array([f32(x) / f32(2), 0], f32)
    y = math.exp(float(x))
    A = f32(y)
    lo, hi = (float(A) + float(np.nextafter(A, f32(-np.inf)))) / 2, (float(A) + float(np.nextafter(A, f32(np.inf)))) / 2
    B = np.nextafter(A, f32(-np.inf) if abs(y - lo) < abs(y - hi) else f32(np.inf))
    ratio, runs_totals = [], []
    for e0 in (A, B):
        e = np.array([e0, 1.0], f32)
        p = (e / np.add.accumulate(e, dtype=f32)[-1]).astype(f32)
        runs, total = device_runs(p, T)
        runs_totals.append((runs, total))
        ratio.append(runs[0] / total)
    u = (ratio[0] + ratio[1]) / 2
    toks = [int(device_pick(r, t, 2, [u])[0][0]) for r, t in runs_totals]
    assert toks[0] != toks[1], f"x={x!r}: u does not separate the two floats"
    return l, u, toks[0], toks[1]


@pytest.mark.gpu
@pytest.mark.parametrize("T", THREADS)
def test_exp_rounding_against_glibc(pkg, orc, T):
    """How many fixture x CUDA's exp rounds to a different float than glibc's: the row is flagged and replayed either way, so the final
    token is the oracle's; the kernel's own token shows the float it used."""
    differ = []
    for x in EXP_MIDPOINTS["x"]:
        l, u, tok_a, tok_b = exp_reveal_rows(float(x), T)
        out = pkg.sample_given_u(l, 0.5, [u], T)
        assert out["flags"][0] == 1 and out["tokens"][0] == orc.sample_u(l, 0.5, u)[0], float(x)
        assert out["device_tokens"][0] in (tok_a, tok_b), float(x)
        if out["device_tokens"][0] == tok_b:
            differ.append(float(x))
    assert len(differ) == CUDA_EXP_ROUNDS_DIFFERENTLY, f"T={T}: CUDA's exp rounds differently from glibc's for x in {differ}"


@pytest.mark.gpu
def test_production_sampler_agrees_with_the_hook(pkg, orc, weights_file):
    """bark_b200_sample_rows (the library's fine-pass entry point, its uniforms from the context's std::mt19937 after reseed) on built
    rows: tokens and eos_p equal the oracle's with the uniforms predicted from orc_mt_seed / orc_mt_next, and the hook's."""
    seed = 20261
    with pkg.Bark(weights_file("tiny", "f16")) as b:
        for n, temp in ((1024, 0.7), (10048, 0.5)):
            name, l, _, _ = threshold_cases(n, temp)[0]
            rows = 64
            b.reseed(seed)
            tok, eos, _ = b.sample_rows(np.repeat(l[None], rows, 0), temp)
            w = orc.mt_words(seed, 2 * rows)
            us = np.array([canonical(w[2 * r], w[2 * r + 1]) for r in range(rows)], f64)
            hook = pkg.sample_given_u(np.repeat(l[None], rows, 0), temp, us)
            for r in range(rows):
                t, e = orc.sample_u(l, temp, us[r])
                assert tok[r] == t == hook["tokens"][r] and bits(eos[r]) == bits(f32(e)) == bits(hook["eos_p"][r]), f"{name} row {r}"


@pytest.mark.gpu
def test_hook_refuses_bad_arguments(pkg):
    l = np.zeros((2, 64), f32)
    assert pkg.sample_given_u(l, 0.7, [0.5, 0.25])["tokens"].shape == (2,)
    bad = [(np.zeros((1, 1), f32), 0.7, [0.5], 0), (np.zeros((1, 16385), f32), 0.7, [0.5], 0), (np.zeros((1025, 8), f32), 0.7, [0.5] * 1025, 0),
           (l, 0.7, [0.5, 1.0], 0), (l, 0.7, [-0.25, 0.5], 0), (l, 0.7, [float("nan"), 0.5], 0), (l, -0.7, [0.5, 0.5], 0),
           (l, float("inf"), [0.5, 0.5], 0), (l, float("nan"), [0.5, 0.5], 0), (l, 0.7, None, 0), (l, 0.7, [0.5, 0.5], 512)]
    for logits, temp, u, T in bad:
        with pytest.raises(RuntimeError):
            pkg.sample_given_u(logits, temp, u, T)
