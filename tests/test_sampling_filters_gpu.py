"""GPU: the top-k / top-p filter of the semantic and coarse stages (DESIGN.md §14) through the C-ABI.  Filtered generations against the
unmodified reference's (tests/golden/ref_pairs/sampling.npz) and against the restatement (tests/history_oracle.py filtered by
tests/sampling_oracle.py on the C oracle); the sampler / decode / prefix-reuse variants, the batch, fast mode, clearing and validation;
and filter_rows_kernel itself through bark_b200_sample_filtered_given_u on rows at the rule's edges."""
import ctypes as C
import os

import numpy as np
import pytest

import history_oracle as H
import sampling_oracle as SO
from conftest import FIXTURE_DIR, GOLDEN_DIR, assert_pinned, bits

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "sampling.npz"))
CASES = [str(c) for c in G["cases"]]
WAV_RTOL = 1e-3


def wav_rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def stored_prompt(key):
    if not int(G[key + "_prompted"]):
        return None
    return {k: G[f"{key}_{k}"] for k in ("semantic_prompt", "coarse_prompt", "fine_prompt")}


def set_settings(b, settings):
    for stage in ("semantic", "coarse"):
        k, p = settings.get(stage, (None, None))
        b.set_sampling(stage, top_k=k, top_p=p)


def run(b, text, prompt=None):
    audio = b.generate(text, history_prompt=prompt)
    t = [b.tokens(i).copy() for i in range(4)]
    return dict(semantic=t[0], coarse=t[1], fine=t[2], prompt=t[3], audio=audio)


def assert_same(got, want, what):
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], want[k]), f"{what}: {k} ids differ"
    assert got["audio"].shape == want["audio"].shape and wav_rel(got["audio"], want["audio"]) < WAV_RTOL, what


def q4_path(pkg, weights_file, config, src_ftype):
    src = weights_file(config, src_ftype)
    dst = os.path.join(FIXTURE_DIR, f"{config}_{src_ftype}_1234_q4_0.bin")
    if not os.path.exists(dst):
        assert pkg.lib().bark_model_quantize(src.encode(), (dst + ".tmp").encode(), 2)
        os.replace(dst + ".tmp", dst)
    return dst


@pytest.mark.parametrize("key", CASES)
def test_stored_cases_match_the_reference(pkg, weights_file, key):
    config, ftype, _ = key.split("_", 2)
    with pkg.Bark(weights_file(config, ftype), seed=int(G[key + "_seed"]), n_steps_text_encoder=int(G[key + "_n_steps"])) as b:
        set_settings(b, SO.stored_settings(G, key))
        got = run(b, str(G[key + "_text"]), stored_prompt(key))
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], G[f"{key}_{k}"]), f"{key}: {k} ids differ from the reference's"
    if key + "_audio" in G.files:
        assert wav_rel(got["audio"], G[key + "_audio"]) < WAV_RTOL
    assert_pinned(got["audio"], G, key + "_audio", f"{key} waveform")


def random_settings(rng):
    out = {}
    for stage in ("semantic", "coarse"):
        k = [None, 1, 5, 50, 400][int(rng.integers(0, 5))]
        p = [None, 0.0, 0.3, 0.9, 1.0][int(rng.integers(0, 5))]
        if k is None and p is None:
            k = 20
        out[stage] = (k, p)
    return out


RESTATEMENT = [("mini_f16", {}), ("tiny_q4_0", {}), ("tiny_f16", {"BARK_B200_SAMPLE_FLAG_EVERY": "3"}),
               ("tiny_f16", {"BARK_B200_DECODE": "multi"}), ("tiny_f16", {"BARK_B200_KV_REUSE": "0"}),
               ("mini_f16", {"BARK_B200_SAMPLE_FLAG_EVERY": "2"})]


@pytest.mark.parametrize("case", range(len(RESTATEMENT)))
def test_against_the_restatement(pkg, orc, weights_file, monkeypatch, case):
    weights, env = RESTATEMENT[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    path = q4_path(pkg, weights_file, "tiny", "f16") if weights == "tiny_q4_0" else weights_file(*weights.split("_"))
    settings = random_settings(np.random.default_rng(100 + case))
    n_steps = 24
    prompt = H.random_prompt(np.random.default_rng(200 + case), 40, 60) if case % 2 else None
    want = SO.generate(orc.Oracle(path, seed=case, n_steps=n_steps), "hello world", n_steps, prompt, settings)
    with pkg.Bark(path, seed=case, n_steps_text_encoder=n_steps) as b:
        set_settings(b, settings)
        assert_same(run(b, "hello world", prompt), want, f"case {case} {settings} {env}")


def test_batch_items_equal_their_own_runs(pkg, weights_file):
    path = weights_file("tiny", "f16")
    rng = np.random.default_rng(46)
    settings = {"semantic": (30, 0.8), "coarse": (None, 0.7)}
    prompts = [H.random_prompt(rng, 120, 40), None, H.random_prompt(rng, 10, 0)]
    texts, seeds = ["hello world", "the fox", "quick brown"], [3, 4, 5]
    for with_prompts in (False, True):
        singles = []
        for t, s, p in zip(texts, seeds, prompts):
            with pkg.Bark(path, seed=s, n_steps_text_encoder=24) as b:
                set_settings(b, settings)
                singles.append(run(b, t, p if with_prompts else None))
        with pkg.Bark(path, seed=9, n_steps_text_encoder=24) as b:
            set_settings(b, settings)
            audios = b.generate_batch(texts, seeds, history_prompts=prompts if with_prompts else None)
            for i, want in enumerate(singles):
                for stage, k in enumerate(("semantic", "coarse", "fine", "prompt")):
                    assert np.array_equal(b.batch_tokens(i, stage), want[k]), (with_prompts, i, k)
                assert np.array_equal(bits(audios[i]), bits(want["audio"])), (with_prompts, i)


def test_fast_mode_semantic_and_coarse_ids(pkg, orc, weights_file, monkeypatch):
    """BARK_B200_MODE=fast changes only the fine passes: filtered semantic and coarse ids equal the restatement's."""
    path = weights_file("mini", "f16")
    settings = {"semantic": (50, 0.9), "coarse": (5, None)}
    want = SO.generate(orc.Oracle(path, seed=2, n_steps=30), "hello world", 30, None, settings)
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    with pkg.Bark(path, seed=2, n_steps_text_encoder=30) as b:
        assert b.fast_mode
        set_settings(b, settings)
        got = run(b, "hello world")
    for k in ("prompt", "semantic", "coarse"):
        assert np.array_equal(got[k], want[k]), k


def test_cleared_filter_gives_the_unfiltered_ids(pkg, weights_file):
    path = weights_file("tiny", "f16")
    with pkg.Bark(path, seed=1, n_steps_text_encoder=16) as b, pkg.Bark(path, seed=8, n_steps_text_encoder=16) as fresh:
        set_settings(b, {"semantic": (5, 0.5), "coarse": (5, 0.5)})
        b.generate("hello world")
        b.set_sampling("semantic"); b.set_sampling("coarse")
        b.reseed(8)
        a = b.generate("the fox")
        want = fresh.generate("the fox")
        for i in range(4):
            assert np.array_equal(b.tokens(i), fresh.tokens(i)), i
        assert np.array_equal(bits(a), bits(want))
        assert pkg.lib().bark_b200_set_sampling(b.ctx, 0, None) == 1


def test_invalid_settings_are_rejected(pkg, weights_file):
    """Each refusal returns 0 and leaves the stage's settings as they were: the run after it equals a run with those settings."""
    path = weights_file("tiny", "f16")
    L = pkg.lib()
    good = {"semantic": (7, 0.6), "coarse": (None, 0.8)}
    with pkg.Bark(path, seed=2, n_steps_text_encoder=16) as b, pkg.Bark(path, seed=2, n_steps_text_encoder=16) as r:
        set_settings(b, good); set_settings(r, good)
        bad = [pkg.SamplingStruct(-1, 0, 1.0), pkg.SamplingStruct(0, 1, 1.5), pkg.SamplingStruct(0, 1, -0.1),
               pkg.SamplingStruct(0, 1, float("nan")), pkg.SamplingStruct(5, 1, float("inf"))]
        for stage in (0, 1):
            for s in bad:
                assert L.bark_b200_set_sampling(b.ctx, stage, C.byref(s)) == 0
        for stage in (2, -1):
            assert L.bark_b200_set_sampling(b.ctx, stage, C.byref(pkg.SamplingStruct(5, 0, 1.0))) == 0
        assert L.bark_b200_set_sampling(None, 0, None) == 0
        with pytest.raises(ValueError):
            b.set_sampling("fine", top_k=5)
        with pytest.raises(ValueError):
            b.set_sampling("semantic", top_p=2.0)
        got, want = run(b, "hello world"), run(r, "hello world")
        for k in ("prompt", "semantic", "coarse", "fine"):
            assert np.array_equal(got[k], want[k]), k


# ---- filter_rows_kernel on rows at the rule's edges ----

def ref_cumsum(y):
    """c_j of the rule for a row already in sorted order (numpy's exp may differ from libm's in rare last bits)."""
    m = np.float32(y.max())
    e = np.exp((y - m).astype(np.float64)).astype(np.float32)
    s = np.cumsum(e, dtype=np.float32)[-1]
    return np.cumsum(e / s, dtype=np.float32)


def edge_rows(n, rng):
    """[(row, top_k, top_p)] at the rule's edges for rows of n logits."""
    out = []
    ties = rng.integers(-6, 7, n).astype(np.float32)
    out += [(ties, 50, None), (ties, 1, None), (ties, n, None), (ties, n + 5, None)]                      # ties at the k-th value
    order = np.argsort(ties, kind="stable")[::-1]
    c = ref_cumsum(ties[order])
    blk = np.flatnonzero(ties[order] == ties[order][0])                                                 # the tied maxima
    out += [(ties, None, float(c[blk[len(blk) // 2]])), (ties, None, 0.0), (ties, None, 1.0)]            # a cut inside the tie block
    x = (rng.standard_normal(n) * 2).astype(np.float32)
    x[rng.integers(0, n, 8)] = 0.0
    x[rng.integers(0, n, 8)] = -0.0
    order = np.argsort(x, kind="stable")[::-1]
    c = ref_cumsum(x[order])
    for j in (3, n // 3):
        t = np.float32(c[j])
        for p in (np.nextafter(t, np.float32(-1)), t, np.nextafter(t, np.float32(2))):                 # c_{j} exactly top_p and one ulp off
            if 0 <= p <= 1:
                out.append((x, None, float(p)))
                out.append((x, 5, float(p)))
    return out


def midpoint_rows(n):
    """Rows whose filter exp arguments (logit minus row max) are the stored near-midpoint x: the filter must flag them."""
    mids = np.load(os.path.join(GOLDEN_DIR, "sampler", "exp_midpoints.npz"))["x"].astype(np.float32)
    out = []
    for i, a in enumerate(mids):
        row = np.full(n, -40.0, np.float32)
        row[(7 * i + 3) % n] = 0.0
        row[(11 * i + 5) % n] = a
        out.append((row, None, 0.95))
        out.append((row, 3, 0.999))
    return out


def oracle_row(orc, row, k, p, temp, u):
    filt, _, kept = SO.filter_row(row, k, p)
    tok, eos = orc.sample_u(filt, temp, u)
    return tok, eos, kept


@pytest.mark.parametrize("n", [10048, 1024])
@pytest.mark.parametrize("threads", [256, 1024])
@pytest.mark.parametrize("rows", [1, 8])
def test_hook_matches_the_oracle_on_edge_rows(pkg, orc, n, threads, rows):
    rng = np.random.default_rng(n + threads + rows)
    cases = edge_rows(n, rng)
    mids = midpoint_rows(n)
    temps = (0.7, 0.0)
    for group, must_flag in ((cases, False), (mids, True)):
        for row, k, p in group:
            for temp in temps:
                u = rng.random(rows)
                out = pkg.sample_filtered_given_u(np.repeat(row[None], rows, 0), temp, u, top_k=k, top_p=p, threads=threads)
                for r in range(rows):
                    tok, eos, kept = oracle_row(orc, row, k, p, temp, u[r])
                    what = (n, threads, rows, k, p, temp, r)
                    assert out["tokens"][r] == tok, what
                    assert np.float32(out["eos_p"][r]).tobytes() == np.float32(eos).tobytes(), what
                    if must_flag:
                        assert out["flags"][r] & 2, ("midpoint row not flagged by the filter",) + what
                    elif not out["flags"][r] & 2:
                        assert out["kept"][r] == kept, what


def test_hook_without_filter_is_sample_given_u(pkg):
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((8, 1024)) * 3).astype(np.float32)
    u = rng.random(8)
    a = pkg.sample_filtered_given_u(x, 0.7, u)
    b = pkg.sample_given_u(x, 0.7, u)
    assert np.array_equal(a["tokens"], b["tokens"]) and np.array_equal(bits(a["eos_p"]), bits(b["eos_p"])) and (a["kept"] == 1024).all()
