"""CPU: the long-form splitter (bark_b200_split_text, DESIGN.md §18, rules 1-4) against a Python restatement of the rules, on the 33
texts of tests/golden/tokenizer/bert_tokenizer.npz and constructed cases, under both tokenizers and at budgets 1, 2, 48 and 255; the
invariants every split keeps; and the refusals.

The restatement counts ids with the library's tested tokenizers: bark_cpp_b200.bert_tokenize for BERT, and for the reference kind the
C oracle's orc_tokenize (tests/test_bert_tokenizer_gpu.py checks it against the library), word by word: that tokenizer never joins
characters across a space, so a text's count is the sum of its words' counts, and a word stays below the oracle's 255-id cap."""
import ctypes as C
import dataclasses
import functools
import itertools
import os
import re

import numpy as np
import pytest

import bert_fixture
from conftest import FIXTURE_DIR

G = bert_fixture.load()
BUDGETS = (1, 2, 48, 255)
STRONG = set("。！？｡।॥")
WEAK = set(".!?…")
CLOSING = set("\"')]}»”’」』）")

CONSTRUCTED = {
    "decimals_eg_ellipsis": "Pi is 3.14 and e is 2.72. Use e.g. this, or e.g.x, or i.e.y… Really?! Yes... Mr. Smith went home.",
    "closing_marks": "He said \"stop.\" (Then he left.) [Fine.] {ok!} «Oui.» “Yes.” ‘No.’ "
                     "「はい。」『いいえ！』（完。） end",
    "cjk_marks_no_space": "今日は晴れ。明日は雨！本当？です｡"
                          "नमस्ते।ठीक॥end.。。done",
    "cues": "[laughs] Hello there. [music] ♪ la la la ♪ [sighs] okay... [clears throat] fine!",
    "whitespace_runs": "  one　　two.\u001c\u001c three \t\n four. five  six  ",
    "words_300": " ".join(w for _, w in zip(range(300), itertools.cycle(
        ["the", "quick", "brown", "fox", "Zürich", "straße", "café", "jumps", "over", "lazy", "dog", "hello", "world", "123"]))) + ".",
    "cjk_300": "".join(chr(0x4E00 + 37 * i) for i in range(300)) + "。",
    "kana_300": "".join(chr(0x3042 + (i * 7) % 80) for i in range(300)),
    "long_word": "Before " + "x" * 150 + " after. " + "Zürich" * 20 + "!",
    "mixed_budget": "Short. " + " ".join(["antidisestablishmentarianism"] * 40) + " ok. 你好世界。 Hi!",
}


def cases():
    return [(n, t) for n, t, _ in G["cases"]] + list(CONSTRUCTED.items())


@pytest.fixture(scope="module")
def oracle(orc, weights_mod):
    """The C oracle on a tiny model written with the fixture's vocabulary (the reference tokenizer's ids over it)."""
    p = os.path.join(FIXTURE_DIR, "tiny_f16_1234_bert_vocab.bin")
    if not os.path.exists(p):
        os.makedirs(FIXTURE_DIR, exist_ok=True)
        weights_mod.write_weights(p + ".tmp", dataclasses.replace(weights_mod.tiny(), extra_words=G["extra_words"]), seed=1234)
        os.replace(p + ".tmp", p)
    return orc.Oracle(p, seed=0, n_steps=4)


@pytest.fixture(scope="module")
def counters(pkg, oracle):
    @functools.lru_cache(maxsize=None)
    def ref_word(w: str) -> int:
        n = int((oracle.tokenize(w)[:256] != 129595).sum())
        assert n < 255, f"a word at the oracle's cap: {w!r}"
        return n

    @functools.lru_cache(maxsize=None)
    def bert(t: str) -> int:
        return int(pkg.bert_tokenize(G["vocab"], t).size)

    return {"reference": lambda t: sum(ref_word(w) for w in t.split(" ") if w), "bert": bert}


def restate(text: str, budget: int, count) -> list:
    """Rules 1-4 in Python: the chunk texts."""
    s = re.sub(r"\s+", " ", text).strip()
    sentences, start, i = [], 0, 0
    while i < len(s):
        if s[i] not in STRONG and s[i] not in WEAK:
            i += 1
            continue
        j, strong = i, False
        while j < len(s) and (s[j] in STRONG or s[j] in WEAK):
            strong |= s[j] in STRONG
            j += 1
        while j < len(s) and s[j] in CLOSING:
            j += 1
        if strong or j == len(s) or s[j] == " ":
            sentences.append(s[start:j])
            if j < len(s) and s[j] == " ":
                j += 1
            start = j
        i = j
    if start < len(s):
        sentences.append(s[start:])
    chunks = []
    for sen in sentences:
        if count(sen) <= budget:
            chunks.append(sen)
            continue
        rest = sen
        while rest:
            words = rest.split(" ")
            if count(words[0]) > budget:
                q = 1
                while q < len(words[0]) and count(words[0][:q + 1]) <= budget:
                    q += 1
                chunks.append(words[0][:q])
                rest = rest[q:]
                continue
            k = 1
            while k < len(words) and count(" ".join(words[:k + 1])) <= budget:
                k += 1
            chunks.append(" ".join(words[:k]))
            rest = " ".join(words[k:])
    chunks = [c for c in chunks if count(c) > 0]
    return chunks if 1 <= len(chunks) <= 1024 else None          # refused: no chunk left, or more than 1024


def hook(pkg, text, kind, budget):
    """bark_b200_split_text: (bounds [n][2], normalised bytes), or -1."""
    vocab = [v.encode() for v in G["vocab"]]
    arr = (C.c_char_p * len(vocab))(*vocab)
    b = text if isinstance(text, bytes) else text.encode()
    L = pkg.lib()
    n = L.bark_b200_split_text(arr, len(vocab), pkg.TOKENIZERS[kind], b, budget, None, 0)
    if n < 0:
        return n
    out = np.full((n + 1, 2), -7, np.int32)
    assert L.bark_b200_split_text(arr, len(vocab), pkg.TOKENIZERS[kind], b, budget, out.ctypes.data_as(C.c_void_p), n) == n
    assert (out[n] == -7).all(), "wrote past cap"
    return out[:n], re.sub(r"\s+", " ", b.decode()).strip().encode()


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("kind", ["reference", "bert"])
@pytest.mark.parametrize("name", [n for n, _ in cases()])
def test_split_equals_the_restatement(pkg, counters, name, kind, budget):
    text = dict(cases())[name]
    count = counters[kind]
    want = restate(text, budget, count)
    if want is None:
        assert hook(pkg, text, kind, budget) == -1
        return
    bounds, norm = hook(pkg, text, kind, budget)
    got = [norm[s:e].decode() for s, e in bounds]
    assert got == want
    assert pkg.split_text(G["vocab"], text, tokenizer=kind, max_chunk_ids=budget) == want
    # invariants: within the budget, bounds at code point starts, in order, and what lies between chunks is a dropped separator or
    # text without ids
    for c in got:
        assert 1 <= count(c) <= budget, c
    prev = 0
    for s, e in bounds:
        assert prev <= s < e <= len(norm)
        for x in (s, e):
            assert x == len(norm) or norm[x] & 0xC0 != 0x80, "a bound inside a UTF-8 sequence"
        gap = norm[prev:s].decode()
        assert gap in ("", " ") or count(gap) == 0, gap
        prev = e
    assert count(norm[prev:].decode()) == 0


def test_constructed_cases_split_where_the_rules_say(pkg):
    t = "Pi is 3.14. Use e.g.x here. Mr. Smith said \"hi.\" Then… ok?! 日本。中文！end"
    assert pkg.split_text(G["vocab"], t, tokenizer="bert", max_chunk_ids=255) == [
        "Pi is 3.14.", "Use e.g.x here.", "Mr.", "Smith said \"hi.\"", "Then…", "ok?!", "日本。", "中文！", "end"]
    # the reference tokenizer has no ids for CJK text: those chunks are dropped
    assert pkg.split_text(G["vocab"], t, tokenizer="reference", max_chunk_ids=255)[-2:] == ["ok?!", "end"]
    # budgets split long sentences into pieces, never merging short sentences
    assert len(pkg.split_text(G["vocab"], CONSTRUCTED["words_300"], max_chunk_ids=48)) > 1
    assert pkg.split_text(G["vocab"], "a. b. c.", tokenizer="bert") == ["a.", "b.", "c."]


@pytest.mark.parametrize("raw", [b"\x80", b"caf\xc3 \xff", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"abc\xc3", b"\xc0\x80"])
@pytest.mark.parametrize("kind", ["reference", "bert"])
def test_invalid_utf8_is_refused(pkg, raw, kind, capfd):
    assert hook(pkg, raw, kind, 48) == -1
    assert "invalid UTF-8" in capfd.readouterr().err
    with pytest.raises(ValueError):
        pkg.split_text(G["vocab"], raw, tokenizer=kind)


def test_refusals(pkg, capfd):
    L = pkg.lib()
    vocab = [v.encode() for v in G["vocab"]]
    arr = (C.c_char_p * len(vocab))(*vocab)
    assert L.bark_b200_split_text(None, 3, 0, b"Hello.", 48, None, 0) == -1
    assert L.bark_b200_split_text(arr, len(vocab), 0, None, 48, None, 0) == -1
    assert L.bark_b200_split_text(arr, len(vocab), 2, b"Hello.", 48, None, 0) == -1
    for budget in (0, 256, -1):
        for kind in (0, 1):
            assert L.bark_b200_split_text(arr, len(vocab), kind, b"Hello.", budget, None, 0) == -1
    assert L.bark_b200_split_text(arr, len(vocab), 0, b"Hello.", 1, None, 0) >= 1
    assert L.bark_b200_split_text(arr, len(vocab), 0, b"Hello.", 255, None, 0) == 1
    # no chunk left: empty, whitespace only, or no ids under the tokenizer
    for text, kind in ((b"", 1), (b" \t\n", 0), ("日本語。".encode(), 0)):
        assert L.bark_b200_split_text(arr, len(vocab), kind, text, 48, None, 0) == -1
    assert L.bark_b200_split_text(arr, len(vocab), 1, "日本語。".encode(), 48, None, 0) == 1
    # at most 1024 chunks
    for kind in (0, 1):
        assert L.bark_b200_split_text(arr, len(vocab), kind, b"a. " * 1024, 48, None, 0) == 1024
        assert L.bark_b200_split_text(arr, len(vocab), kind, b"a. " * 1025, 48, None, 0) == -1
    assert "more than 1024 chunks" in capfd.readouterr().err
