"""GPU: speaker history prompts through the C-ABI.  Prompted generations against the unmodified reference's (stored in
tests/golden/ref_pairs/history.npz) and against the restatement (tests/history_oracle.py) on the C oracle; the stage entry points,
the sampler / decode / prefix-reuse variants, the batch, validation, clearing and fast mode.  Ids bit-identical, waveforms within the
generation tolerance of tests/test_parity_gpu.py."""
import ctypes as C
import os

import numpy as np
import pytest

import history_oracle as H
from conftest import FIXTURE_DIR, GOLDEN_DIR, assert_pinned, bits

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "history.npz"))
CASES = [str(c) for c in G["cases"]]
WAV_RTOL = 1e-3


def wav_rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def stored_prompt(key):
    return {k: G[f"{key}_{k}"] for k in ("semantic_prompt", "coarse_prompt", "fine_prompt")}


def ids(b):
    return [b.tokens(i).copy() for i in range(4)]


def assert_same(got, want, what):
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], want[k]), f"{what}: {k} ids differ"
    assert got["audio"].shape == want["audio"].shape and wav_rel(got["audio"], want["audio"]) < WAV_RTOL, what


def ctx_audio(pkg, b):
    """What bark_get_audio_data returns now."""
    n = pkg.lib().bark_get_audio_data_size(b.ctx)
    return np.ctypeslib.as_array(pkg.lib().bark_get_audio_data(b.ctx), shape=(n,)).copy()


def run(b, text, prompt):
    audio = b.generate(text, history_prompt=prompt)
    t = ids(b)
    return dict(semantic=t[0], coarse=t[1], fine=t[2], prompt=t[3], audio=audio)


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
        got = run(b, str(G[key + "_text"]), stored_prompt(key))
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], G[f"{key}_{k}"]), f"{key}: {k} ids differ from the reference's"
    if key + "_audio" in G.files:
        assert wav_rel(got["audio"], G[key + "_audio"]) < WAV_RTOL
    assert_pinned(got["audio"], G, key + "_audio", f"{key} waveform")          # the codec is bit-exact (tests/test_parity_gpu.py)


def restatement_cases():
    rng = np.random.default_rng(41)
    out = [("mini_f16", None, 20), ("tiny_q4_0", None, 16)]
    for lo, hi, n_f in ((2, 40, 0), (100, 400, int(rng.integers(1, 700))), (40, 120, 512)):
        n_s = int(rng.choice([n for n in range(lo, hi) if len(H.coarse_lengths(n))]))
        out.append(("tiny_f16", H.random_prompt(rng, n_s, n_f), 24))
    return out


@pytest.mark.parametrize("case", range(5))
def test_against_the_restatement(pkg, orc, weights_file, case):
    """mini f16 and tiny q4_0 with a chained prompt (the oracle's own first generation), tiny f16 with random valid prompts."""
    weights, prompt, n_steps = restatement_cases()[case]
    path = q4_path(pkg, weights_file, "tiny", "f16") if weights == "tiny_q4_0" else weights_file(*weights.split("_"))
    if prompt is None:
        prompt = H.chained_prompt(orc.Oracle(path, seed=11, n_steps=n_steps).generate("the quick brown fox"))
    want = H.generate(orc.Oracle(path, seed=case, n_steps=n_steps), "hello world", n_steps, prompt)
    with pkg.Bark(path, seed=case, n_steps_text_encoder=n_steps) as b:
        assert_same(run(b, "hello world", prompt), want, f"case {case}")


def test_stage_entry_points(pkg, orc, weights_file):
    """set_history_prompt, then tokenize / set_tokens + forward(0, 1, 2) stage by stage against the restatement's stages."""
    path = weights_file("tiny", "f16")
    p = H.random_prompt(np.random.default_rng(43), 150, 600)
    P = H.as_prompt(p)
    o = orc.Oracle(path, seed=0, n_steps=20)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=20) as b:
        b.set_history_prompt(p)
        want_prompt = H.prompt_ids(o, "hello world", P)
        assert np.array_equal(b.tokenize("hello world"), want_prompt) and np.array_equal(b.tokens(3), want_prompt)
        b.forward(0)
        sem = H.semantic(o, want_prompt, 20)
        assert np.array_equal(b.tokens(0), sem)
        b.reseed(5); o.reseed(5)
        sem = np.random.default_rng(44).integers(0, 10000, 70).astype(np.int32)
        b.set_tokens(0, sem); b.forward(1)
        co = H.coarse(o, sem, P)
        assert np.array_equal(b.tokens(1), co)
        b.reseed(6); o.reseed(6)
        b.set_tokens(1, co); b.forward(2)
        assert np.array_equal(b.tokens(2), H.fine(o, co, P))


def test_sampler_paths_agree(pkg, weights_file, monkeypatch):
    """A prompted generation, then an unprompted one on the same context: same ids, waveforms and RNG state under forced host
    replays, the per-op decode and the full coarse re-prefill as on the default path."""
    path = weights_file("mini", "f16")
    p = H.random_prompt(np.random.default_rng(45), 220, 300)
    runs = []
    for env in ({}, {"BARK_B200_SAMPLE_FLAG_EVERY": "5"}, {"BARK_B200_DECODE": "multi"}, {"BARK_B200_KV_REUSE": "0"}):
        for k in ("BARK_B200_SAMPLE_FLAG_EVERY", "BARK_B200_DECODE", "BARK_B200_KV_REUSE"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        with pkg.Bark(path, seed=3, n_steps_text_encoder=70) as b:
            a1 = b.generate("one two three", history_prompt=p); t1 = ids(b)
            a2 = b.generate("four"); t2 = ids(b)
        runs.append((a1, t1, a2, t2))
    for a1, t1, a2, t2 in runs[1:]:
        for i in range(4):
            assert np.array_equal(t1[i], runs[0][1][i]) and np.array_equal(t2[i], runs[0][3][i])
        assert np.array_equal(bits(a1), bits(runs[0][0])) and np.array_equal(bits(a2), bits(runs[0][2]))


def test_batch_items_equal_their_own_runs(pkg, weights_file):
    path = weights_file("tiny", "f16")
    rng = np.random.default_rng(46)
    prompts = [H.random_prompt(rng, 120, 40), None, H.random_prompt(rng, 10, 0), None]
    texts, seeds = ["hello world", "the fox", "quick brown", "hello"], [3, 4, 5, 6]
    singles = []
    for t, s, p in zip(texts, seeds, prompts):
        with pkg.Bark(path, seed=s, n_steps_text_encoder=24) as b:
            singles.append(run(b, t, p))
    with pkg.Bark(path, seed=9, n_steps_text_encoder=24) as b:
        ctx_prompt = H.random_prompt(rng, 30, 10)
        b.set_history_prompt(ctx_prompt)
        before_audio = b.generate("the quick"); before = ids(b)
        audios = b.generate_batch(texts, seeds, history_prompts=prompts)
        for i, want in enumerate(singles):
            got = dict(semantic=b.batch_tokens(i, 0), coarse=b.batch_tokens(i, 1), fine=b.batch_tokens(i, 2), prompt=b.batch_tokens(i, 3),
                       audio=audios[i])
            assert_same(got, want, f"item {i}")
            assert np.array_equal(bits(audios[i]), bits(want["audio"]))
        plain = b.generate_batch(texts[1:2], seeds[1:2])                         # the context's prompt does not apply to a batch
        assert np.array_equal(b.batch_tokens(0, 2), singles[1]["fine"]) and np.array_equal(bits(plain[0]), bits(singles[1]["audio"]))
        for i in range(4):
            assert np.array_equal(b.tokens(i), before[i])
        assert np.array_equal(bits(ctx_audio(pkg, b)), bits(before_audio))
        after = b.generate("the quick")                                         # RNG and prompt of the context untouched
    with pkg.Bark(path, seed=9, n_steps_text_encoder=24) as r:
        r.set_history_prompt(ctx_prompt)
        r.generate("the quick")
        assert np.array_equal(bits(after), bits(r.generate("the quick")))


def bad_prompts():
    rng = np.random.default_rng(47)
    good = H.random_prompt(rng, 20, 10)
    out = []
    for k, v in (("semantic_prompt", np.zeros(0, np.int32)), ("coarse_prompt", np.zeros((2, 0), np.int32))):
        out.append(dict(good, **{k: v}))
    for k, bad in (("semantic_prompt", 10000), ("semantic_prompt", -1), ("coarse_prompt", 1024), ("coarse_prompt", -3),
                   ("fine_prompt", 1024), ("fine_prompt", -1)):
        p = {kk: vv.copy() for kk, vv in good.items()}
        p[k].reshape(-1)[p[k].size // 2] = bad
        out.append(p)
    n_s = 20                                                                   # 29 n_s < 20 n_c < 31 n_s: n_c in 30 ... 30
    for n_c in (29, 31):
        out.append(dict(good, coarse_prompt=rng.integers(0, 1024, (2, n_c)).astype(np.int32)))
    assert good["semantic_prompt"].size == n_s and good["coarse_prompt"].shape[1] == 30
    return good, out


def test_invalid_prompts_are_rejected(pkg, weights_file):
    """Every rule rejects its input (return 0); RNG, ids, waveform and the prompt in place stay as they were."""
    path = weights_file("tiny", "f16")
    good, bad = bad_prompts()
    L = pkg.lib()
    with pkg.Bark(path, seed=2, n_steps_text_encoder=16) as b, pkg.Bark(path, seed=2, n_steps_text_encoder=16) as r:
        b.set_history_prompt(good); r.set_history_prompt(good)
        a0 = b.generate("hello world"); r.generate("hello world")
        t0 = ids(b)
        for i, p in enumerate(bad):
            st, _keep = pkg._history_struct(p)
            assert L.bark_b200_set_history_prompt(b.ctx, C.byref(st)) == 0, f"bad prompt {i} accepted"
            with pytest.raises(ValueError):
                b.set_history_prompt(p)
        st, _keep = pkg._history_struct(good)
        st.n_fine_frames = -1
        assert L.bark_b200_set_history_prompt(b.ctx, C.byref(st)) == 0, "negative fine frame count accepted"
        for i in range(4):
            assert np.array_equal(b.tokens(i), t0[i])
        assert np.array_equal(bits(ctx_audio(pkg, b)), bits(a0))
        with pytest.raises(RuntimeError):
            b.generate_batch(["a", "b"], [1, 2], history_prompts=[None, bad[0]])
        assert np.array_equal(bits(b.generate("hello world")), bits(r.generate("hello world")))       # same RNG, same prompt
        assert np.array_equal(b.tokens(3), r.tokens(3)) and b.tokens(3)[256] == good["semantic_prompt"][0]


def test_cleared_prompt_leaves_nothing_behind(pkg, weights_file):
    path = weights_file("tiny", "f16")
    p = H.random_prompt(np.random.default_rng(48), 300, 600)
    with pkg.Bark(path, seed=1, n_steps_text_encoder=16) as b, pkg.Bark(path, seed=8, n_steps_text_encoder=16) as fresh:
        b.generate("hello world", history_prompt=p)
        b.set_history_prompt(p); b.generate("hello world"); b.set_history_prompt(None)
        b.reseed(8)
        a = b.generate("the fox")
        want = fresh.generate("the fox")
        for i in range(4):
            assert np.array_equal(b.tokens(i), fresh.tokens(i)), i
        assert np.array_equal(bits(a), bits(want))
        assert (b.tokens(3)[256:512] == 10000).all()


def test_fast_mode_semantic_and_coarse_ids(pkg, weights_file, monkeypatch):
    """BARK_B200_MODE=fast changes only the fine passes: prompted semantic and coarse ids equal parity mode's."""
    path = weights_file("mini", "f16")
    p = H.random_prompt(np.random.default_rng(49), 80, 100)
    runs = []
    for mode in ("parity", "fast"):
        monkeypatch.setenv("BARK_B200_MODE", mode)
        with pkg.Bark(path, seed=2, n_steps_text_encoder=30) as b:
            assert b.fast_mode == (mode == "fast")
            b.generate("hello world", history_prompt=p)
            runs.append(ids(b))
    for i in (0, 1, 3):
        assert np.array_equal(runs[0][i], runs[1][i]), i
