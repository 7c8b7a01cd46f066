"""GPU: long-form generation (bark_b200_set_long_form, DESIGN.md §18).  A long-form call against the loop it stands for, on a second
context with the same seed: set chunk k's prompt, generate chunk k's text, in order.  Chunk texts, every id of every chunk, each chunk's
waveform, the joined waveform, the progress callbacks and the state left behind (RNG, restored prompt) bit for bit; on tiny f16, mini
f16, tiny q4_0 and the BERT-vocabulary tiny model with a mixed-language text.  Also: the fixed voice with a reference-matched prompt
and without one, own ids that are no valid prompt, a one-sentence text (the bench clip), the environment knob, refusals, the batch and
fast mode."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

import bert_fixture
import history_oracle as H
from conftest import FIXTURE_DIR, GOLDEN_DIR, bits

pytestmark = pytest.mark.gpu

BG = bert_fixture.load()
HG = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "history.npz"))
TEXT = "Hello world. The quick brown fox jumps over the lazy dog! Is it 3.5 or 4? [laughs] That was fun."
MIXED = "Hello, world! Привет мир. 你好世界。こんにちは！ Straße und Zürich."
AFTER = "the quick brown fox"


def ids(b):
    return [b.tokens(i).copy() for i in range(4)]


def ctx_audio(pkg, b):
    n = pkg.lib().bark_get_audio_data_size(b.ctx)
    return np.ctypeslib.as_array(pkg.lib().bark_get_audio_data(b.ctx), shape=(n,)).copy()


def stats(b):
    s, per_model = b.stats()
    return [getattr(s, k) for k, _ in s._fields_ if k != "t_load_us"], per_model[:, 2].tolist()


def recorder():
    calls = []
    return calls, lambda ctx, step, progress, user: calls.append((step, progress))


@pytest.fixture(scope="module")
def bert_path(weights_mod):
    p = os.path.join(FIXTURE_DIR, "tiny_f16_1234_bert_vocab.bin")
    if not os.path.exists(p):
        os.makedirs(FIXTURE_DIR, exist_ok=True)
        weights_mod.write_weights(p + ".tmp", dataclasses.replace(weights_mod.tiny(), extra_words=BG["extra_words"]), seed=1234)
        os.replace(p + ".tmp", p)
    return p


def q4_path(pkg, weights_file):
    src = weights_file("tiny", "f16")
    dst = os.path.join(FIXTURE_DIR, "tiny_f16_1234_q4_0.bin")
    if not os.path.exists(dst):
        assert pkg.lib().bark_model_quantize(src.encode(), (dst + ".tmp").encode(), 2)
        os.replace(dst + ".tmp", dst)
    return dst


def long_form(pkg, path, seed, n_steps, text, voice="chain", prompt=None, gap=6000, budget=48, **kw):
    """The long-form call: (joined waveform, chunks, progress calls, statistics, next plain generation's waveform and ids)."""
    calls, cb = recorder()
    with pkg.Bark(path, seed=seed, n_steps_text_encoder=n_steps, progress=cb, **kw) as b:
        if prompt is not None:
            b.set_history_prompt(prompt)
        b.set_long_form(voice, max_chunk_ids=budget, gap_samples=gap)
        audio = b.generate(text)
        chunks, st, got_calls = b.long_chunks(), stats(b), list(calls)
        assert np.array_equal(bits(ctx_audio(pkg, b)), bits(audio))
        b.set_long_form(None)
        after = b.generate(AFTER), ids(b)
        assert pkg.lib().bark_b200_long_chunks(b.ctx) == 0
    return audio, chunks, got_calls, st, after


def manual_loop(pkg, path, seed, n_steps, texts, voice="chain", prompt=None, **kw):
    """The loop long form stands for: per chunk its prompt P_k set, then generate.  Returns per chunk (waveform, ids, whether its own ids
    were a valid prompt), the progress calls, and the next plain generation after the context's prompt is put back."""
    calls, cb = recorder()
    out = []
    with pkg.Bark(path, seed=seed, n_steps_text_encoder=n_steps, progress=cb, **kw) as r:
        cur = prompt
        for k, t in enumerate(texts):
            if k > 0 and voice == "chain":
                own = r.last_generation_prompt()
                try:
                    r.set_history_prompt(own)
                    cur = own
                    out[-1] = out[-1][:2] + (True,)
                except ValueError:
                    pass
            r.set_history_prompt(cur)
            a = r.generate(t)
            out.append((a, ids(r), False))
        got_calls = list(calls)
        r.set_history_prompt(prompt)
        after = r.generate(AFTER), ids(r)
    return out, got_calls, after


def assert_equals_loop(pkg, path, seed, n_steps, text, vocab=None, tokenizer=None, voice="chain", prompt=None, gap=6000, budget=48, **kw):
    if tokenizer:
        kw["tokenizer"] = tokenizer
    audio, chunks, calls, _, after = long_form(pkg, path, seed, n_steps, text, voice, prompt, gap, budget, **kw)
    texts = [c["text"] for c in chunks]
    if vocab is not None:
        assert texts == pkg.split_text(vocab, text, tokenizer=tokenizer or "reference", max_chunk_ids=budget)
    assert len(texts) >= 2
    loop, want_calls, want_after = manual_loop(pkg, path, seed, n_steps, texts, voice, prompt, **kw)
    start = 0
    for k, (c, (a, t, _)) in enumerate(zip(chunks, loop)):
        for stage, name in ((0, "semantic"), (1, "coarse"), (2, "fine"), (3, "prompt")):
            assert np.array_equal(c[name], t[stage]), f"chunk {k}: {name} ids differ from the loop's"
        assert c["start"] == start and c["n_samples"] == a.size
        assert np.array_equal(bits(audio[start:start + a.size]), bits(a)), f"chunk {k}: waveform differs from the loop's"
        start += a.size + gap
    want = np.concatenate([np.concatenate([a, np.zeros(gap, np.float32)]) if k + 1 < len(loop) else a for k, (a, _, _) in enumerate(loop)])
    assert np.array_equal(bits(audio), bits(want))
    assert calls == want_calls
    assert np.array_equal(bits(after[0]), bits(want_after[0]))
    for i in range(4):
        assert np.array_equal(after[1][i], want_after[1][i])
    return chunks, loop


@pytest.mark.parametrize("model", ["tiny_f16", "mini_f16", "tiny_q4_0", "bert_vocab"])
def test_chain_equals_the_manual_loop(pkg, weights_mod, weights_file, bert_path, model):
    if model == "bert_vocab":
        assert_equals_loop(pkg, bert_path, 3, 20, MIXED, vocab=BG["vocab"], tokenizer="bert")
        return
    config, ftype = model.split("_", 1)
    path = q4_path(pkg, weights_file) if ftype == "q4_0" else weights_file(config, ftype)
    vocab = weights_mod.synth_vocab(weights_mod.CONFIGS[config](weights_mod.F16))
    chunks, loop = assert_equals_loop(pkg, path, 1, 20, TEXT, vocab=vocab, gap=1234)
    assert any(valid for _, _, valid in loop[:-1]), "no chunk handed its own ids on: the case does not test the chain"


@pytest.mark.parametrize("with_prompt", [True, False])
def test_fixed_equals_the_manual_loop(pkg, weights_file, with_prompt):
    key = "tiny_f16_chained"
    prompt = {k: HG[f"{key}_{k}"] for k in ("semantic_prompt", "coarse_prompt", "fine_prompt")} if with_prompt else None
    assert_equals_loop(pkg, weights_file("tiny", "f16"), 2, 16, TEXT, voice="fixed", prompt=prompt, gap=0)


def test_invalid_own_ids_keep_the_previous_prompt(pkg, weights_file):
    """Five semantic ids make seven coarse frames, which do not align (29 n_s < 20 n_c fails): every chunk k >= 1 keeps the context's
    prompt.  (One semantic id, the other case that never aligns, makes one frame, below the codec's seven.)"""
    prompt = H.random_prompt(np.random.default_rng(61), 120, 40)
    _, loop = assert_equals_loop(pkg, weights_file("tiny", "f16"), 4, 5, TEXT, prompt=prompt)
    assert not any(valid for _, _, valid in loop), "a chunk's own ids were a valid prompt"
    for _, t, _ in loop:
        assert np.array_equal(t[3][256:376], prompt["semantic_prompt"])


def test_one_sentence_is_plain_generation(pkg, weights_file):
    """Long form on a text that is one chunk equals long form off, bit for bit; on the bench clip that is the reference's output."""
    g = np.load(os.path.join(GOLDEN_DIR, "small_f16_n138.npz"))
    for path, seed, n_steps, text in ((weights_file("tiny", "f16"), 5, 16, "hello world, one sentence only!"),
                                      (weights_file("small", "f16", int(g["weight_seed"])), int(g["seed"]), int(g["n_steps"]), str(g["prompt"]))):
        runs = []
        for on in (True, False):
            with pkg.Bark(path, seed=seed, n_steps_text_encoder=n_steps) as b:
                if on:
                    b.set_long_form("chain")
                runs.append((b.generate(text), ids(b), stats(b)[1]))
                assert pkg.lib().bark_b200_long_chunks(b.ctx) == (1 if on else 0)
        assert np.array_equal(bits(runs[0][0]), bits(runs[1][0]))
        for i in range(4):
            assert np.array_equal(runs[0][1][i], runs[1][1][i])
        assert runs[0][2] == runs[1][2]
    assert np.array_equal(runs[0][1][0], g["semantic"]) and np.array_equal(runs[0][1][2], g["fine"])
    assert float(np.abs(runs[0][0] - g["audio"]).max() / np.abs(g["audio"]).max()) < 1e-3


def test_environment_knob(pkg, weights_file, monkeypatch):
    path = weights_file("tiny", "f16")
    monkeypatch.setenv("BARK_B200_LONG_FORM", "chain")
    with pkg.Bark(path, seed=6, n_steps_text_encoder=12) as b:
        a_env = b.generate(TEXT)
        c_env = b.long_chunks()
    for v in ("", "off"):
        monkeypatch.setenv("BARK_B200_LONG_FORM", v)
        with pkg.Bark(path, seed=6, n_steps_text_encoder=12) as b:
            assert b.long_form is None
            b.generate(TEXT)
            assert b.long_chunks() == []
            b.reseed(6)
            b.set_long_form("chain")
            a_set = b.generate(TEXT)
            c_set = b.long_chunks()
        assert np.array_equal(bits(a_env), bits(a_set))
        assert [c["text"] for c in c_env] == [c["text"] for c in c_set]
        for x, y in zip(c_env, c_set):
            assert np.array_equal(x["fine"], y["fine"])
    for bad in ("CHAIN", "on", "1"):
        monkeypatch.setenv("BARK_B200_LONG_FORM", bad)
        with pytest.raises(RuntimeError):
            pkg.Bark(path)


def test_refusals_change_nothing(pkg, weights_file, capfd):
    """Invalid settings keep the previous ones; a refused text and a sharded context leave ids, waveform, statistics, prompt, RNG and
    chunk results as they were."""
    path = weights_file("tiny", "f16")
    L = pkg.lib()
    prompt = H.random_prompt(np.random.default_rng(62), 60, 20)
    with pkg.Bark(path, seed=7, n_steps_text_encoder=12) as b, pkg.Bark(path, seed=7, n_steps_text_encoder=12) as r:
        for x in (b, r):
            x.set_history_prompt(prompt)
            x.set_long_form("chain", max_chunk_ids=40, gap_samples=100)
        a0 = b.generate(TEXT); r.generate(TEXT)
        t0, st0, ch0 = ids(b), stats(b), b.long_chunks()
        for voice, budget, gap in ((2, 48, 0), (-1, 48, 0), (0, 0, 0), (0, 256, 0), (0, 48, -1), (0, 48, 240001)):
            assert L.bark_b200_set_long_form(b.ctx, C.byref(pkg.LongFormStruct(voice, budget, gap))) == 0
        with pytest.raises(ValueError):
            b.set_long_form("both")
        for text in (b"caf\xc3 \xff", b"", " \t ".encode(), "日本語。".encode(), b"a. " * 1025):
            assert L.bark_generate_audio(b.ctx, text, 1) is False
        assert "invalid UTF-8" in capfd.readouterr().err

        def unchanged():
            for i in range(4):
                assert np.array_equal(b.tokens(i), t0[i])
            assert np.array_equal(bits(ctx_audio(pkg, b)), bits(a0))
            assert stats(b) == st0
            got = b.long_chunks()
            assert [c["text"] for c in got] == [c["text"] for c in ch0] and all(np.array_equal(x["fine"], y["fine"]) for x, y in zip(got, ch0))
        unchanged()
        a1 = b.generate(TEXT)                                           # settings, prompt and RNG as they were: same as r
        assert np.array_equal(bits(a1), bits(r.generate(TEXT)))
        now = b.long_chunks()
        assert now[1]["start"] == now[0]["n_samples"] + 100
    with pkg.Bark(path, seed=7, n_steps_text_encoder=12) as b, pkg.Bark(path, seed=7, n_steps_text_encoder=12) as r:
        a0 = b.generate("hello world"); r.generate("hello world")
        t0, st0, ch0 = ids(b), stats(b), []
        b.shard_connect(b.shard_init(0, 1))
        b.set_long_form("chain")
        assert L.bark_generate_audio(b.ctx, TEXT.encode(), 1) is False
        assert "sharded" in capfd.readouterr().err
        unchanged()
        b.set_long_form(None)


def test_batch_ignores_long_form(pkg, weights_file):
    path = weights_file("tiny", "f16")
    texts, seeds = ["Hello world. Second sentence!", "One. Two. Three."], [3, 4]
    runs = []
    for on in (False, True):
        with pkg.Bark(path, seed=1, n_steps_text_encoder=16) as b:
            if on:
                b.set_long_form("chain")
            audios = b.generate_batch(texts, seeds)
            runs.append((audios, [[b.batch_tokens(i, s) for s in range(4)] for i in range(2)]))
            assert b.long_chunks() == []
    for i in range(2):
        assert np.array_equal(bits(runs[0][0][i]), bits(runs[1][0][i]))
        for s in range(4):
            assert np.array_equal(runs[0][1][i][s], runs[1][1][i][s])


def test_fast_mode_equals_the_loop(pkg, weights_file, monkeypatch):
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    path = weights_file("mini", "f16")
    with pkg.Bark(path) as b:
        assert b.fast_mode
    assert_equals_loop(pkg, path, 8, 16, TEXT)
