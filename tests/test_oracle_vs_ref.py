"""CPU: the C oracle against the unmodified reference, bit for bit.  The reference's outputs for exactly these inputs are stored in
tests/golden/ref_pairs/tiny_f16.npz (tests/golden/make_golden_ref_pairs.py), so the comparison needs no reference build."""
import hashlib
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR, assert_pinned, bits

G = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "tiny_f16.npz"))


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def pair(orc, weights_file):
    path = weights_file("tiny", "f16")
    assert hashlib.sha1(open(path, "rb").read()).hexdigest() == str(G["weights_sha1"]), "weight generator is not reproducible"
    return orc.Oracle(path, seed=0, n_steps=16), G


def test_gelu_table(orc, pair):
    o, _ = orc.gelu_tables()
    assert np.array_equal(o, np.load(os.path.join(GOLDEN_DIR, "gelu_table_f16.npz"))["table"])


def test_tokenizer(pair):
    o, r = pair
    for text, ids in zip(r["tokenizer_texts"], r["tokenizer_ids"]):
        assert np.array_equal(o.tokenize(str(text)), ids), text


def test_causal_eval_bit_exact(pair):
    o, r = pair
    rng = np.random.default_rng(1)
    for which, first, merge in ((0, None, True), (1, np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 37)]).astype(np.int32), False)):
        toks = o.tokenize("hello world") if first is None else first
        po = 0
        for step in range(len(r[f"causal{which}_sha1"])):
            lo, po = o.gpt_eval(which, toks, po, merge)
            assert po == r[f"causal{which}_n_past"][step], (which, step)
            assert np.array_equal(bits(lo[:64]), bits(r[f"causal{which}_head"][step])) and sha(lo) == str(r[f"causal{which}_sha1"][step]), (which, step)
            toks = np.array([int(np.argmax(lo[:10000])) if which == 0 else 10000 + int(np.argmax(lo[10000:12048]))], np.int32)


def test_fine_eval_bit_exact(pair):
    o, r = pair
    rng = np.random.default_rng(2)
    buf = rng.integers(0, 1024, (8, 1024)).astype(np.int32)
    for nn in (2, 7):
        x = buf.copy(); x[nn:, :] = 1024
        fl = o.fine_eval(x, nn)
        assert np.array_equal(bits(fl[:8, :64]), bits(r[f"fine{nn}_head"])) and sha(fl) == str(r[f"fine{nn}_sha1"]), nn


def test_sampler(pair):
    o, r = pair
    rng = np.random.default_rng(3)
    o.reseed(9)
    for i in range(150):
        lg = (rng.standard_normal((10048, 1024)[i % 2]) * 4).astype(np.float32)
        temp = (0.7, 0.5, 0.0)[i % 3]
        t, e = o.sample(lg, temp)
        assert t == r["sampler_tokens"][i] and bits(np.float32(e)) == bits(r["sampler_eos"][i]), i


def test_encodec_bit_exact(pair):
    o, r = pair
    rng = np.random.default_rng(4)
    for T in (7, 40):
        codes = rng.integers(0, 1024, (8, T)).astype(np.int32)
        assert_pinned(o.encodec_decode(codes), r, f"encodec{T}_audio")


def test_full_generate(pair):
    o, r = pair
    o.reseed(0)
    a = o.generate("hello world")
    for k in ("semantic", "coarse", "fine"):
        assert np.array_equal(a[k], r[f"generate_{k}"]), k
    assert_pinned(a["audio"], r, "generate_audio")


def test_long_context_bit_exact(orc, weights_file):
    """Steps up to n_kv 1024: semantic steps at n_past 1015 .. 1023 after the merged prompt and a 758-id continuation, coarse steps at
    n_past 887 .. 902 after a whole window prompt (the reference's logits in ref_pairs/long_context.npz)."""
    r = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "long_context.npz"))
    o = orc.Oracle(weights_file("tiny", "f16"))
    rng = np.random.default_rng(6)
    lg, n_past = o.gpt_eval(0, o.tokenize("hello world"), 0, True)
    lg, n_past = o.gpt_eval(0, rng.integers(0, 10000, 1015 - n_past).astype(np.int32), n_past, False)
    for i in range(9):
        lg, n_past = o.gpt_eval(0, np.array([int(np.argmax(lg[:10000]))], np.int32), n_past, False)
        assert_pinned(lg, r, f"semantic{i}", f"semantic step at n_past {n_past - 1}")
    assert n_past == 1024
    prompt = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 630)]).astype(np.int32)
    lg, n_past = o.gpt_eval(1, prompt, 0, False)
    for i in range(16):
        lg, n_past = o.gpt_eval(1, np.array([10000 + int(np.argmax(lg[10000:12048]))], np.int32), n_past, False)
        assert_pinned(lg, r, f"coarse{i}", f"coarse step at n_past {n_past - 1}")
