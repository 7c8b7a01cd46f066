"""CPU: upstream Bark's text tokenizer (bark_b200_bert_tokenize, DESIGN.md §17) against the oracle's ids in
tests/golden/tokenizer/bert_tokenizer.npz: every text case, every code point between two letters, the refusal of invalid UTF-8, and the generated
character-class header against what the oracle gives now."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import bert_fixture
from conftest import ROOT


@pytest.fixture(scope="module")
def golden():
    return bert_fixture.load()


def test_fixture_vocabulary_is_the_weights_writer_s(golden, weights_mod):
    """A weights file written with Config(extra_words=...) carries the fixture's vocabulary (what the GPU tests load)."""
    import dataclasses
    assert weights_mod.synth_vocab(dataclasses.replace(weights_mod.tiny(), extra_words=golden["extra_words"])) == golden["vocab"]
    assert golden["vocab"].count("Zürich") == 2


@pytest.mark.parametrize("i", range(33))
def test_text_cases_equal_the_oracle(pkg, golden, i):
    name, text, want = golden["cases"][i]
    got = pkg.bert_tokenize(golden["vocab"], text)
    assert np.array_equal(got, want), f"{name}: {got.tolist()} != {want.tolist()}"


def test_case_list_is_complete(golden):
    names = [n for n, _, _ in golden["cases"]]
    assert len(names) == 33 and sum(n.startswith("lang_") for n in names) == 13
    lengths = {n: len(ids) for n, _, ids in golden["cases"]}
    assert lengths["pieces_255"] == 255 and lengths["pieces_256"] == 256 and lengths["pieces_300_plus"] > 300
    assert lengths["word_100"] == 100 and lengths["word_101"] == 1


def test_prompts_follow_upstream_rule(golden):
    """The fixture's 513-id prompts: the first 256 ids plus the offset, text padding, an empty semantic history, the infer token."""
    for (name, _, ids), p in zip(golden["cases"], golden["prompt"]):
        n = min(len(ids), 256)
        assert np.array_equal(p[:n], ids[:n] + 10048), name
        assert (p[n:256] == 129595).all() and (p[256:512] == 10000).all() and p[512] == 129599, name


def test_every_code_point_equals_the_oracle(pkg, golden):
    """ "x" + c + "x" for every code point c but the surrogates and NUL (a C string ends there).  Checked 4096 at a time (the texts
    joined by spaces give the concatenation of their ids), and code point by code point inside a chunk that differs."""
    vocab = [v.encode() for v in golden["vocab"]]
    arr = (C.c_char_p * len(vocab))(*vocab)
    L = pkg.lib()

    def ids(text: str) -> np.ndarray:
        b = text.encode()
        out = np.zeros(4 * len(b) + 8, np.int32)
        n = L.bark_b200_bert_tokenize(arr, len(vocab), b, out.ctypes.data_as(C.c_void_p), out.size)
        assert 0 <= n <= out.size, text
        return out[:n]

    pairs = list(bert_fixture.code_point_ids(golden))
    assert len(pairs) == 0x110000 - 0x800 and pairs[0][0] == 0
    pairs = pairs[1:]
    bad = []
    for s in range(0, len(pairs), 4096):
        chunk = pairs[s:s + 4096]
        if np.array_equal(ids(" ".join("x" + chr(cp) + "x" for cp, _ in chunk)), np.concatenate([w for _, w in chunk])):
            continue
        bad += [(hex(cp), ids("x" + chr(cp) + "x").tolist(), w.tolist()) for cp, w in chunk if not np.array_equal(ids("x" + chr(cp) + "x"), w)]
        assert bad, "a chunk differs although each of its code points agrees"
        if len(bad) > 20:
            break
    assert not bad, bad[:20]


@pytest.mark.parametrize("raw", [
    b"\x80", b"a\xbfb",                                       # lone continuation bytes
    b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf",   # overlong forms
    b"\xed\xa0\x80", b"\xed\xbf\xbf", b"x\xed\xb2\x80y",       # UTF-16 surrogates
    b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8\x88\x80\x80\x80", b"\xff", b"\xfe",   # past U+10FFFF, bytes no UTF-8 uses
    b"\xe4\xbd", b"\xf0\x9f\x98", b"abc\xc3", b"\xe4\x41\xa0",   # truncated sequences
])
def test_invalid_utf8_is_refused(pkg, golden, raw, capfd):
    vocab = [v.encode() for v in golden["vocab"]]
    arr = (C.c_char_p * len(vocab))(*vocab)
    out = np.full(8, -7, np.int32)
    assert pkg.lib().bark_b200_bert_tokenize(arr, len(vocab), raw, out.ctypes.data_as(C.c_void_p), out.size) == -1
    assert (out == -7).all()
    assert "invalid UTF-8" in capfd.readouterr().err
    with pytest.raises(ValueError):
        pkg.bert_tokenize(golden["vocab"], raw)


def test_utf8_boundaries_are_accepted(pkg, golden):
    """The first and last code point of every UTF-8 length, and those around the surrogates, decode (their ids are checked above)."""
    for c in ("\x7f", "\x80", "\u07ff", "\u0800", "\ud7ff", "\ue000", "\uffff", "\U00010000", "\U0010ffff"):
        assert pkg.bert_tokenize(golden["vocab"], ("x" + c + "x").encode()).size >= 1


def test_hook_arguments(pkg, golden, capfd):
    L = pkg.lib()
    vocab = [v.encode() for v in golden["vocab"]]
    arr = (C.c_char_p * len(vocab))(*vocab)
    text = "Hello мир 你好".encode()
    n = L.bark_b200_bert_tokenize(arr, len(vocab), text, None, 0)
    full = pkg.bert_tokenize(golden["vocab"], text)
    assert n == full.size >= 4
    part = np.full(n, -7, np.int32)
    assert L.bark_b200_bert_tokenize(arr, len(vocab), text, part.ctypes.data_as(C.c_void_p), 2) == n
    assert np.array_equal(part[:2], full[:2]) and (part[2:] == -7).all()
    assert L.bark_b200_bert_tokenize(None, 3, text, None, 0) == -1
    assert L.bark_b200_bert_tokenize(arr, len(vocab), None, None, 0) == -1
    no_unk = [v for v in vocab if v != b"[UNK]"]
    arr2 = (C.c_char_p * len(no_unk))(*no_unk)
    assert L.bark_b200_bert_tokenize(arr2, len(no_unk), b"x", None, 0) == -1
    assert "[UNK]" in capfd.readouterr().err
    with pytest.raises(ValueError):
        pkg.bert_tokenize(golden["vocab"], "a\x00b")


def test_character_header_is_the_oracle_s():
    """bark.cpp_b200/csrc/bert_chars.h equals what tools/gen_bert_chars.py derives from the installed tokenizers now."""
    pytest.importorskip("tokenizers")
    spec = importlib.util.spec_from_file_location("gen_bert_chars", os.path.join(ROOT, "tools", "gen_bert_chars.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(gen.HEADER, encoding="utf-8") as f:
        committed = f.read()
    assert gen.strip_provenance(committed) == gen.strip_provenance(gen.generate())
