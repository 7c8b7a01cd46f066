"""GPU: upstream Bark's text tokenizer on a context (DESIGN.md §17).  A tiny model whose vocabulary is the fixture's
(tests/golden/tokenizer/bert_tokenizer.npz): the 513-id prompts and raw ids against the oracle's, a BERT generation against the unchanged pipeline
fed the oracle's prompt, batches, the environment knob, refused texts, and the default tokenizer's ids as before."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

import bert_fixture
import history_oracle as H
from conftest import FIXTURE_DIR, bits

pytestmark = pytest.mark.gpu

G = bert_fixture.load()
CASES = {name: (text, ids, G["prompt"][i]) for i, (name, text, ids) in enumerate(G["cases"])}
PARITY_TEXTS = ["Hello, world! 123 café", "hello world", "the quick brown fox", "Ünïcödé Straße — naïve façade", "abc123 x[MASK]y"]


@pytest.fixture(scope="module")
def path(weights_mod):
    """tiny f16 (weight seed 1234) written with the fixture's vocabulary."""
    p = os.path.join(FIXTURE_DIR, "tiny_f16_1234_bert_vocab.bin")
    if not os.path.exists(p):
        os.makedirs(FIXTURE_DIR, exist_ok=True)
        weights_mod.write_weights(p + ".tmp", dataclasses.replace(weights_mod.tiny(), extra_words=G["extra_words"]), seed=1234)
        os.replace(p + ".tmp", p)
    return p


def ids(b):
    return [b.tokens(i).copy() for i in range(4)]


def stats(b):
    s, per_model = b.stats()
    return [getattr(s, k) for k, _ in s._fields_], per_model.tolist()


def ctx_audio(pkg, b):
    n = pkg.lib().bark_get_audio_data_size(b.ctx)
    return np.ctypeslib.as_array(pkg.lib().bark_get_audio_data(b.ctx), shape=(n,)).copy()


def test_prompts_and_text_ids_equal_the_oracle(pkg, path):
    """tokenize and text_ids under BERT for every case, without and with a history prompt (positions 256-512 as today)."""
    hist = H.random_prompt(np.random.default_rng(51), 300, 0)
    with pkg.Bark(path, tokenizer="bert") as b:
        assert b.tokenizer == "bert"
        for name, (text, want_ids, want_prompt) in CASES.items():
            assert np.array_equal(b.text_ids(text), want_ids), name
            assert np.array_equal(b.text_ids(text, tokenizer="bert"), want_ids), name
            assert np.array_equal(b.tokenize(text), want_prompt), name
            assert np.array_equal(b.tokens(3), want_prompt), name
        b.set_history_prompt(hist)
        for name, (text, _, want_prompt) in CASES.items():
            want = want_prompt.copy()
            want[256:512] = hist["semantic_prompt"][-256:]
            assert np.array_equal(b.tokenize(text), want), name


def test_bert_generation_is_the_pipeline_on_the_oracle_prompt(pkg, path):
    """generate(t) under BERT equals, in every id and every waveform bit, a fresh reference-tokenizer context with the same seed fed
    the oracle's prompt through set_tokens(3) and run stage by stage."""
    for name, seed in (("lang_ru", 3), ("lang_zh", 4), ("mixed_scripts", 5)):
        text, _, want_prompt = CASES[name]
        with pkg.Bark(path, seed=seed, n_steps_text_encoder=24, tokenizer="bert") as b:
            audio = b.generate(text)
            got = ids(b)
        with pkg.Bark(path, seed=seed, n_steps_text_encoder=24) as r:
            assert r.tokenizer == "reference"
            r.set_tokens(3, want_prompt)
            for stage in range(3):
                r.forward(stage)
            want = ids(r)
            want_audio = r.encodec_decode(np.ascontiguousarray(r.tokens(2).T))
        assert np.array_equal(got[3], want_prompt), name
        for i in range(3):
            assert np.array_equal(got[i], want[i]), f"{name}: stage {i} ids differ"
        assert np.array_equal(bits(audio), bits(want_audio)), f"{name}: waveform differs"


def test_batch_items_equal_their_own_runs(pkg, path):
    names = ["lang_de", "lang_ja", "lang_hi", "lang_ko", "emoji_zwj"]
    texts, seeds = [CASES[n][0] for n in names], [11, 12, 13, 14, 15]
    singles = []
    for t, s in zip(texts, seeds):
        with pkg.Bark(path, seed=s, n_steps_text_encoder=20, tokenizer="bert") as b:
            singles.append((b.generate(t), ids(b)))
    with pkg.Bark(path, seed=1, n_steps_text_encoder=20) as b:
        b.set_tokenizer("bert")
        audios = b.generate_batch(texts, seeds)
        for i, (a, t) in enumerate(singles):
            for stage in range(4):
                assert np.array_equal(b.batch_tokens(i, stage), t[stage]), f"item {i} stage {stage}"
            assert np.array_equal(bits(audios[i]), bits(a)), f"item {i} waveform"
            assert np.array_equal(b.batch_tokens(i, 3), CASES[names[i]][2])


def test_environment_knob(pkg, path, monkeypatch):
    """BARK_B200_TOKENIZER=bert at load equals set_tokenizer("bert"); reference or empty is the default; anything else refuses the load."""
    text = CASES["lang_pl"][0]
    monkeypatch.setenv("BARK_B200_TOKENIZER", "bert")
    with pkg.Bark(path, seed=7, n_steps_text_encoder=16) as b:
        assert b.tokenizer == "bert"
        a_env, t_env = b.generate(text), ids(b)
    for v in ("reference", ""):
        monkeypatch.setenv("BARK_B200_TOKENIZER", v)
        with pkg.Bark(path, seed=7, n_steps_text_encoder=16) as b:
            assert b.tokenizer == "reference"
            assert not np.array_equal(b.tokenize(text), CASES["lang_pl"][2])
            b.set_tokenizer("bert")
            a_set, t_set = b.generate(text), ids(b)
        for i in range(4):
            assert np.array_equal(t_env[i], t_set[i])
        assert np.array_equal(bits(a_env), bits(a_set))
    for bad in ("BERT", "bert-base", "1"):
        monkeypatch.setenv("BARK_B200_TOKENIZER", bad)
        with pytest.raises(RuntimeError):
            pkg.Bark(path)


def test_refused_text_leaves_the_state(pkg, path, capfd):
    """Invalid UTF-8 under BERT: bark_generate_audio and the batch return false, bark_b200_tokenize writes nothing; ids, waveform,
    statistics, the last batch and the RNG stay as they were."""
    L = pkg.lib()
    with pkg.Bark(path, seed=2, n_steps_text_encoder=16, tokenizer="bert") as b, \
            pkg.Bark(path, seed=2, n_steps_text_encoder=16, tokenizer="bert") as r:
        a0 = b.generate("Привет мир"); r.generate("Привет мир")
        ba = b.generate_batch(["你好", "hello"], [1, 2])
        t0, st0 = ids(b), stats(b)
        bt = [b.batch_tokens(i, 2).copy() for i in range(2)]
        bad = b"caf\xc3 \xff"
        assert L.bark_generate_audio(b.ctx, bad, 1) is False
        out = np.full(513, -7, np.int32)
        L.bark_b200_tokenize(b.ctx, bad, out.ctypes.data_as(C.c_void_p))
        assert (out == -7).all()
        assert L.bark_b200_text_ids(b.ctx, 1, bad, None, 0) == -1
        arr = (C.c_char_p * 2)(b"hello", bad)
        sd = (C.c_uint32 * 2)(1, 2)
        assert L.bark_b200_generate_batch(b.ctx, arr, sd, 2, 1) is False
        assert "invalid UTF-8" in capfd.readouterr().err
        for i in range(4):
            assert np.array_equal(b.tokens(i), t0[i])
        assert np.array_equal(bits(ctx_audio(pkg, b)), bits(a0))
        assert stats(b) == st0
        for i in range(2):
            assert np.array_equal(b.batch_tokens(i, 2), bt[i])
        assert L.bark_b200_batch_audio(b.ctx, 0, None, 0) == ba[0].size
        assert np.array_equal(bits(b.generate("Всё хорошо")), bits(r.generate("Всё хорошо")))     # same RNG state
        assert L.bark_b200_set_tokenizer(b.ctx, 2) == 0 and L.bark_b200_set_tokenizer(b.ctx, -1) == 0
        assert L.bark_b200_text_ids(b.ctx, 2, b"x", None, 0) == -1
        with pytest.raises(ValueError):
            b.set_tokenizer("wordpiece")
        assert b.tokenizer == "bert"
        assert np.array_equal(b.tokenize("Привет"), r.tokenize("Привет"))


def test_default_tokenizer_is_unchanged(pkg, orc, path, weights_file):
    """The default context and bark_b200_tokenize give the reference's ids (the C oracle's restatement of bark.cpp's tokenizer), on
    the standard tiny vocabulary and on the fixture's; text_ids under the reference kind are those ids uncapped."""
    for p in (weights_file("tiny", "f16"), path):
        o = orc.Oracle(p, seed=0, n_steps=4)
        with pkg.Bark(p) as b:
            for text in PARITY_TEXTS + [CASES[n][0] for n in ("lang_fr", "lang_ru", "pieces_300_plus")]:
                want = np.asarray(o.tokenize(text), np.int32)
                assert np.array_equal(b.tokenize(text), want), text
                n = int((want[:256] != 129595).sum())
                raw = b.text_ids(text)
                assert np.array_equal(raw[:n], want[:n] - 10048), text
                assert raw.size == n or (n == 255 and raw.size > 255), text
                assert np.array_equal(b.text_ids(text, tokenizer="reference"), raw)
