"""CPU: the device sampler's decision against the reference's, both restated exactly as written, on rows built on the edges.

The reference (gpt_sample, bark.cpp:184-270, then libstdc++'s std::discrete_distribution): float l / temp, the max, float(exp(double(l -
max))) with glibc's exp, a sequential float sum, a float division; then accumulate in double, divide by that sum, partial_sum, the last
entry forced to 1, and lower_bound of one generate_canonical<double,53> draw u.  Argmax (temp 0): the first strict maximum.

sample_rows_kernel (csrc/sampling.cu) takes CUDA's double exp instead and forms the cumulative sums in another order: thread t of T sums
the chunk [t c, t c + c), c = ceil(n / T), in double; a shuffle-up scan (o = 1, 2, 4, 8, 16) and the sums of the warp totals give
run = before + incl - part at the chunk's start; then run += p[i] and the first i < n - 1 with run >= u * total wins.  Two brackets
flag the rows it cannot prove, and the host replays them with the reference's order:
  * exp:       float(y (1 - 2^-50)) != float(y (1 + 2^-50)) for some entry y = exp(l - max);
  * threshold: |run - u total| <= 8 n 2^-53 total at some i < n - 1.
The restatements below check that the reference restatement is the oracle (orc_sample_u) and libstdc++ itself (compiled here with
g++), that on every built row the device order either agrees with the reference or is flagged, and that the threshold bracket is what
makes it so: with eps = 0 the device order picks a different token on a large share of the threshold rows without flagging them.
tests/test_sampler_gpu.py runs the same rows through the kernel.
"""
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN_DIR, bits

f32, f64 = np.float32, np.float64
THREADS = (256, 1024)
EPS_SCALE = 8.0                                  # sampling.cu: eps = 8 n 2^-53 total
INT_MAX = 0x7fffffff
EXP_MIDPOINTS = np.load(os.path.join(GOLDEN_DIR, "sampler", "exp_midpoints.npz"))   # tests/golden/make_golden_exp_midpoints.py


# ------------------------------------------------------------------------------------------------------------------------------------
# the two orders
# ------------------------------------------------------------------------------------------------------------------------------------
def ref_probs(logits, temp):
    """gpt_sample up to the probabilities: (p float32 [n], y = glibc's exp(l - max) as double [n])."""
    l = np.asarray(logits, f32) / f32(0.7 if temp == 0 else temp)       # the argmax path still divides by 0.7
    d = l - l.max()
    y = np.array([math.exp(float(v)) for v in d], f64)
    e = y.astype(f32)
    s = np.add.accumulate(e, dtype=f32)[-1]                               # sequential float sum
    return (e / s).astype(f32), y


def ref_cp(p):
    """discrete_distribution's table: accumulate in double, divide by it, partial_sum, last entry 1."""
    q = p.astype(f64)
    cp = np.add.accumulate(q / np.add.accumulate(q)[-1])
    cp[-1] = 1.0
    return cp


def ref_pick(cp, u):
    """lower_bound(cp, u) for every u (cp is non-decreasing up to its last entry, which is 1 > u)."""
    u = np.atleast_1d(np.asarray(u, f64))
    return np.argmax(cp[None, :] >= u[:, None], axis=1)


def ref_sample(logits, temp, u):
    """(tokens [len(u)], eos_p) of the reference."""
    p, _ = ref_probs(logits, temp)
    if temp == 0:
        return np.full(np.size(u), int(np.argmax(p))), p[-1]
    return ref_pick(ref_cp(p), u), p[-1]


def exp_ambiguous(y):
    """The kernel's exp bracket on each entry, restated with glibc's value in place of CUDA's."""
    return (y * (1.0 - 2.0 ** -50)).astype(f32) != (y * (1.0 + 2.0 ** -50)).astype(f32)


def midpoint_margin(y):
    """Relative distance of each y to the nearest float rounding boundary."""
    f = y.astype(f32)
    lo = (f.astype(f64) + np.nextafter(f, f32(-np.inf)).astype(f64)) / 2
    hi = (f.astype(f64) + np.nextafter(f, f32(np.inf)).astype(f64)) / 2
    return np.minimum(np.abs(y - lo), np.abs(y - hi)) / np.maximum(y, 2.0 ** -1074)


def device_runs(p, T):
    """sample_rows_kernel<T>'s running sums run_i for i < n - 1, and total, in its order."""
    n = p.size
    c, NW = -(-n // T), T // 32
    chunks = np.zeros(T * c, f64)
    chunks[:n] = p
    chunks = chunks.reshape(T, c)                                       # thread t: [t c, t c + c) (past n: zeros, exact)
    part = np.add.accumulate(chunks, axis=1)[:, -1]
    incl = part.reshape(NW, 32)
    for o in (1, 2, 4, 8, 16):                                          # __shfl_up_sync: lanes >= o add the value o lanes down
        nxt = incl.copy()
        nxt[:, o:] = incl[:, o:] + incl[:, :-o]
        incl = nxt
    acc = np.add.accumulate(incl[:, 31])                                # before += s_d[w] (w < warp), total += s_d[w]
    before = np.concatenate([[0.0], acc[:-1]])
    start = (np.repeat(before, 32) + incl.reshape(-1)) - part
    runs = np.add.accumulate(np.concatenate([start[:, None], chunks], axis=1), axis=1)[:, 1:]
    return runs.reshape(-1)[:n - 1], acc[-1]


def device_pick(runs, total, n, u, eps_scale=EPS_SCALE):
    """(tokens, threshold flags) for every u: the first i < n - 1 with run_i >= u total (else n - 1); the bracket |run - thr| <= eps."""
    thr = np.atleast_1d(np.asarray(u, f64))[:, None] * total
    eps = eps_scale * n * 2.0 ** -53 * total
    ge = runs[None, :] >= thr
    tok = np.where(ge.any(axis=1), np.argmax(ge, axis=1), n - 1)
    return tok, (np.abs(runs[None, :] - thr) <= eps).any(axis=1)


def device_argmax(p, T, ge=False):
    """The kernel's argmax: strided per thread (first strict maximum; ge=True: `>=`), then xor butterfly and warp sums, ties to the
    lower index."""
    n, NW = p.size, T // 32
    best = np.full(T, -np.inf, f32)
    bi = np.full(T, INT_MAX, np.int64)
    for t in range(min(T, n)):
        v = p[t::T]
        j = int(np.argmax(v)) if not ge else len(v) - 1 - int(np.argmax(v[::-1]))
        best[t], bi[t] = v[j], t + j * T
    best, bi = best.reshape(NW, 32), bi.reshape(NW, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        ob, oi = best[:, lanes ^ o], bi[:, lanes ^ o]
        take = (ob > best) | ((ob == best) & (oi < bi))
        best, bi = np.where(take, ob, best), np.where(take, oi, bi)
    b, i = best[0, 0], bi[0, 0]
    for w in range(1, NW):
        if best[w, 0] > b or (best[w, 0] == b and bi[w, 0] < i):
            b, i = best[w, 0], bi[w, 0]
    return int(i)


def device_sample(logits, temp, u, T, eps_scale=EPS_SCALE, ge=False):
    """The kernel's tokens (before any replay) and flags for every u; and the exp margin of the row (smallest midpoint_margin)."""
    p, y = ref_probs(logits, temp)
    u = np.atleast_1d(np.asarray(u, f64))
    exp_flag = bool(exp_ambiguous(y).any())
    if temp == 0:
        tok, flag = np.full(u.size, device_argmax(p, T, ge)), np.zeros(u.size, bool)
    else:
        runs, total = device_runs(p, T)
        tok, flag = device_pick(runs, total, p.size, u, eps_scale)
    return tok, flag | exp_flag, float(midpoint_margin(y).min())


# ------------------------------------------------------------------------------------------------------------------------------------
# uniforms: generate_canonical<double,53> over two mt19937 words returns (w0 + 2^32 w1) / 2^64
# ------------------------------------------------------------------------------------------------------------------------------------
def on_grid(u):
    return 0.0 <= u < 1.0 and math.floor(u * 2.0 ** 64) == u * 2.0 ** 64


def canonical(w0, w1):
    r = (float(w0) + float(w1) * 2.0 ** 32) / 2.0 ** 64
    return r if r < 1.0 else math.nextafter(1.0, 0.0)


def words(u):
    k = int(u * 2.0 ** 64)
    return k & 0xffffffff, k >> 32


# ------------------------------------------------------------------------------------------------------------------------------------
# builders: each returns a list of cases (name, logits float32 [n], temp, u float64 [k]); one logits row, many uniforms
# ------------------------------------------------------------------------------------------------------------------------------------
def cp_uniforms(cp, idx):
    """u = cp[i] and its two neighbours for each i: the reference's own decision edges, where the device's sums can fall either side."""
    us = []
    for i in idx:
        for u in (cp[i], math.nextafter(cp[i], 0.0), math.nextafter(cp[i], 1.0)):
            if on_grid(u):
                us.append(u)
    return np.array(us, f64)


THRESHOLD_SHAPES = [(1024, 0.7), (1024, 0.5), (10048, 0.7), (10048, 0.5)]


def threshold_cases(n, temp):
    """Random rows (logits ~ 3 N(0, 1)) with u on cp[i] or one ulp either side, i spread over the row: here the device's sums differ
    from the reference's in the last bits, so whichever side of u each lands on is a coin toss the bracket must catch."""
    out = []
    for seed in range(2):
        rng = np.random.default_rng(1000 * n + int(temp * 10) + seed)
        logits = (rng.standard_normal(n) * 3).astype(f32)
        cp = ref_cp(ref_probs(logits, temp)[0])
        idx = np.unique(np.linspace(0, n - 2, 160).astype(int))
        out.append((f"threshold n={n} temp={temp} seed={seed}", logits, temp, cp_uniforms(cp, idx)))
    return out


def exp_cases():
    """Rows whose l - max is a fixture x: glibc's exp(x) lies within 2^-50 of a float midpoint, so CUDA's exp (<= 1 ulp off) may
    round to the other float and the exp bracket must fire.  x = -2^-25 is the guaranteed one: exp is the midpoint 1 - 2^-25 plus
    four double ulps.  temp 0.5 and logit x / 2 make l - max exactly x."""
    out = []
    rng = np.random.default_rng(7)
    for x in EXP_MIDPOINTS["x"]:
        logits = np.concatenate([[f32(x) / f32(2)], [f32(0)], (-1 - 6 * rng.random(62)).astype(f32)]).astype(f32)
        out.append((f"exp x={float(x)!r}", logits, 0.5, np.array([0.0, 0.25, 0.5, 0.75, 0.999], f64)))
    return out


def edge_cases():
    out = []
    rng = np.random.default_rng(11)
    # u = 0 when p0 = 0: cp[0] = 0 >= 0, so the reference returns index 0, a token of probability zero
    l = (rng.standard_normal(300) * 2).astype(f32); l[0] = f32(-500)
    out.append(("u=0, p0=0", l, 0.7, np.array([0.0, 2.0 ** -64, 2.0 ** -40], f64)))
    # u = 1 - 2^-53 with underflowed trailing entries: the last nonzero cp rounds to 1, so the answer is not the forced last entry
    for seed in range(200):
        l = (np.random.default_rng(seed).standard_normal(500) * 2).astype(f32); l[-8:] = f32(-500)
        cp = ref_cp(ref_probs(l, 0.7)[0])
        if cp[-9] == 1.0:
            break
    assert cp[-9] == 1.0, "no row found whose last nonzero cumulative sum rounds to 1"
    out.append(("u=1-2^-53, trailing zeros", l, 0.7, np.array([1 - 2.0 ** -53, 1 - 2.0 ** -52, 1 - 2.0 ** -30], f64)))
    # leading and trailing zero-probability runs
    l = (rng.standard_normal(1000) * 2).astype(f32); l[:200] = f32(-1000); l[-300:] = f32(-1000)
    cp = ref_cp(ref_probs(l, 0.5)[0])
    out.append(("zero runs", l, 0.5, np.concatenate([[0.0, 0.5, 1 - 2.0 ** -53], cp_uniforms(cp, [0, 199, 200, 201, 698, 699, 700, 998])])))
    # all mass in one entry
    for j in (0, 37, 511):
        l = np.full(512, f32(-1000)); l[j] = f32(3)
        out.append((f"one entry j={j}", l, 0.7, np.array([0.0, 2.0 ** -64, 0.5, 1 - 2.0 ** -53], f64)))
    # subnormal probabilities and entries next to the exp underflow boundary: l - max from 0 down to -104 (float exp is 0 below
    # about -103.97, subnormal below -87.34)
    l = np.concatenate([np.linspace(0, -80, 64), np.linspace(-86, -104, 900), [-103.97, -103.972, -103.9721, -103.98]]).astype(f32)
    cp = ref_cp(ref_probs(l, 1.0)[0])
    out.append(("subnormal tail", l, 1.0, np.concatenate([[0.0, 0.5, 1 - 2.0 ** -53], cp_uniforms(cp, np.linspace(0, l.size - 2, 40).astype(int))])))
    # widths around the thread counts: n < T leaves empty chunks, n % 8 != 0 reaches the tail of the sequential float4 sum
    for n in (2, 7, 9, 255, 257, 1023, 1025, 16384):
        l = (np.random.default_rng(n).standard_normal(n) * 3).astype(f32)
        cp = ref_cp(ref_probs(l, 0.7)[0])
        us = np.concatenate([cp_uniforms(cp, np.unique(np.linspace(0, n - 2, 24).astype(int))), [0.0, 0.3, 0.9, 1 - 2.0 ** -53]])
        out.append((f"width n={n}", l, 0.7, us))
    return out


def argmax_cases(T):
    """temp 0.  Distinct logits whose probabilities round to the same float (exp of l - max within 2^-26 of 0 is 1.0): the first index
    wins although its logit is smaller.  Equal maxima in one thread (i, i + T), across threads (i, i + 1) and across warps (i, i + 64)."""
    out = []
    rng = np.random.default_rng(T)
    for name, a, b in (("one thread", 5, 5 + T), ("across threads", 40, 41), ("across warps", 3, 3 + 64)):
        for distinct in (False, True):
            l = (rng.standard_normal(max(2 * T, 1024) + 3) - 6).astype(f32)
            l[a], l[b] = (f32(-1e-9), f32(0)) if distinct else (f32(2.5), f32(2.5))
            out.append((f"argmax T={T} {name}{' distinct logits' if distinct else ''}", l, 0.0, np.zeros(1, f64)))
    return out


def all_cases():
    cases = [c for n, t in THRESHOLD_SHAPES for c in threshold_cases(n, t)] + exp_cases() + edge_cases()
    return cases + [c for T in THREADS for c in argmax_cases(T)]


# ------------------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cases():
    return all_cases()


def test_reference_restatement_is_the_oracle(orc, cases):
    for name, l, temp, us in cases:
        want, eos = ref_sample(l, temp, us)
        for u, w in zip(us, want):
            t, e = orc.sample_u(l, temp, u)
            assert t == w and bits(f32(e)) == bits(eos), f"{name} u={u.hex()}: oracle {t} restatement {w}"


CPP = r'''
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
// a URNG that returns two given 32-bit words: generate_canonical<double,53> over a 32-bit generator takes exactly two
struct Words {
    using result_type = uint32_t;
    uint32_t w[2]; int k;
    static constexpr uint32_t min() { return 0; }
    static constexpr uint32_t max() { return 0xffffffffu; }
    uint32_t operator()() { if (k > 1) { fprintf(stderr, "more than two draws\n"); exit(2); } return w[k++]; }
};
int main(int argc, char ** argv) {
    FILE * in = fopen(argv[1], "rb"), * out = fopen(argv[2], "wb");
    int32_t n; float temp; uint32_t w[2];
    while (fread(&n, 4, 1, in) == 1) {
        if (fread(&temp, 4, 1, in) != 1 || fread(w, 4, 2, in) != 2) return 3;
        std::vector<float> p((size_t) n);
        if (fread(p.data(), 4, (size_t) n, in) != (size_t) n) return 3;
        for (float & v : p) v /= temp;                          // gpt_sample, bark.cpp:184-270
        float mx = -INFINITY;
        for (float v : p) mx = v > mx ? v : mx;
        float sum = 0.0f;
        for (float & v : p) { v = (float) exp((double) (v - mx)); sum += v; }
        for (float & v : p) v /= sum;
        Words g{{w[0], w[1]}, 0};
        std::discrete_distribution<int> dist(p.begin(), p.end());
        const int32_t tok = dist(g);
        fwrite(&tok, 4, 1, out); fwrite(&p.back(), 4, 1, out);
    }
    return 0;
}
'''


def test_reference_restatement_is_libstdcxx(cases, tmp_path):
    """std::discrete_distribution<int> itself, fed the two mt19937 words behind each u (only uniforms on the k 2^-64 grid, the values
    the library's generator can return)."""
    src, exe = tmp_path / "dd.cpp", tmp_path / "dd"
    src.write_text(CPP)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", str(src), "-o", str(exe)])
    blob, want = bytearray(), []
    for name, l, temp, us in cases:
        if temp == 0:
            continue
        toks, eos = ref_sample(l, temp, us)
        for u, t in zip(us, toks):
            if not on_grid(u):
                continue
            w0, w1 = words(u)
            assert canonical(w0, w1) == u
            blob += np.int32(l.size).tobytes() + f32(temp).tobytes() + np.array([w0, w1], np.uint32).tobytes() + l.tobytes()
            want.append((name, u, int(t), bits(eos)))
    (tmp_path / "in.bin").write_bytes(bytes(blob))
    subprocess.check_call([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    got = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.int32).reshape(-1, 2)
    assert got.shape[0] == len(want) > 2000
    for (name, u, t, eb), (gt, ge) in zip(want, got):
        assert gt == t and np.uint32(ge) == eb, f"{name} u={u.hex()}: libstdc++ {gt} restatement {t}"


@pytest.mark.parametrize("T", THREADS)
def test_device_order_agrees_or_flags(cases, T):
    """On every built row the device order picks the reference's token or flags the row for the host replay."""
    for name, l, temp, us in cases:
        if name.startswith("argmax") and f"T={T}" not in name:
            continue
        want, _ = ref_sample(l, temp, us)
        tok, flag, _ = device_sample(l, temp, us, T)
        bad = np.flatnonzero((tok != want) & ~flag)
        assert bad.size == 0, f"{name} T={T}: device order picks {tok[bad[0]]}, reference {want[bad[0]]} at u={us[bad[0]].hex()}, unflagged"


@pytest.mark.parametrize("T", THREADS)
@pytest.mark.parametrize("n, temp", THRESHOLD_SHAPES)
def test_threshold_bracket_is_needed(n, temp, T):
    """Without the threshold bracket (eps = 0, which flags only run == thr exactly) the device order picks a different token than the
    reference on a large share of the threshold rows without flagging them (a quarter to a half); with it every one is flagged."""
    missed = total = 0
    for name, l, temp_, us in threshold_cases(n, temp):
        want, _ = ref_sample(l, temp_, us)
        tok, flag, _ = device_sample(l, temp_, us, T)
        tok0, flag0, _ = device_sample(l, temp_, us, T, eps_scale=0.0)
        assert np.array_equal(tok, tok0)
        assert flag[tok != want].all(), name
        missed += int(((tok0 != want) & ~flag0).sum()); total += us.size
    assert total >= 850 and missed >= total // 5, f"{missed} of {total} differ unflagged"


def test_exp_bracket_fires_on_the_fixture():
    x = EXP_MIDPOINTS["x"]
    assert x.size >= 4 and f32(-2.0 ** -25) in x
    for v, y in zip(x, EXP_MIDPOINTS["exp"]):
        assert math.exp(float(v)) == y, "glibc's exp differs from the fixture's"
        assert exp_ambiguous(np.array([y]))[0], float(v)
    y = math.exp(-2.0 ** -25)
    assert y - (1 - 2.0 ** -25) == 4 * 2.0 ** -53             # the midpoint plus four double ulps
    for name, l, temp, us in exp_cases():
        p, yy = ref_probs(l, temp)
        assert yy[0] in EXP_MIDPOINTS["exp"] and exp_ambiguous(yy).any(), name
        for T in THREADS:
            assert device_sample(l, temp, us, T)[1].all(), name


@pytest.mark.parametrize("T", THREADS)
def test_argmax_ties_go_to_the_first_index(T):
    for name, l, temp, us in argmax_cases(T):
        p, _ = ref_probs(l, 0.0)
        first = int(np.argmax(p))
        ties = np.flatnonzero(p == p[first])
        assert ties.size == 2, name
        assert device_argmax(p, T) == first, name
        if "distinct" in name:
            assert l[ties[0]] < l[ties[1]], name
        if "one thread" in name:                                  # `>=` inside a thread would keep the later index
            assert device_argmax(p, T, ge=True) == ties[1], name


def test_edges_pick_what_the_reference_picks():
    c = {name: (l, temp, us) for name, l, temp, us in edge_cases()}
    l, temp, us = c["u=0, p0=0"]
    assert ref_sample(l, temp, us[:1])[0][0] == 0 and ref_probs(l, temp)[0][0] == 0
    l, temp, us = c["u=1-2^-53, trailing zeros"]
    assert ref_sample(l, temp, us[:1])[0][0] < l.size - 8
    for j in (0, 37, 511):
        l, temp, us = c[f"one entry j={j}"]
        assert list(ref_sample(l, temp, us)[0]) == [0, j, j, j]
    p = ref_probs(*c["subnormal tail"][:2])[0]
    assert ((p > 0) & (p < np.finfo(f32).tiny)).sum() > 100 and (p == 0).any()
