"""Writes tests/golden/tokenizer/bert_tokenizer.npz: upstream Bark's text ids, computed by the oracle, for tests/test_bert_tokenizer.py and
tests/test_bert_tokenizer_gpu.py (DESIGN.md §17).

The oracle is upstream Bark's rule (bark/generation.py):

    BertTokenizer(vocab, do_lower_case=False).encode(re.sub(r"\\s+", " ", text).strip(), add_special_tokens=False)

with transformers 5 (the tokenizers-backed BertTokenizer; both versions are recorded in the file).  It needs transformers, so it runs
only where the fixture is made; rerunning it gives identical bytes.  Contents:

  vocab_*        the vocabulary: weights.synth_vocab of a Config whose extra_words (extra_*) hold pieces of sample sentences in Bark's
                 13 languages (whole words, single characters, ## pieces, multi-character pieces) and one duplicated entry, so a
                 weights file written with weights.Config(extra_words=...) carries the same vocabulary
  text_*         the text cases (UTF-8), ids_* their oracle ids (before truncation), prompt [n][513] the prompts upstream builds
                 from them without a history prompt (first 256 ids + text_encoding_offset, text_pad_token, 256 semantic_pad_token,
                 semantic_infer_token)
  cp_*           every code point's ids for "x" + c + "x", run-length coded: run r covers the code points from cp_first[r] up to the
                 next run's first (surrogates skipped), each with ids cp_ids[r] (-1 padded)

Strings are stored as UTF-8 bytes with offsets (numpy's unicode arrays drop trailing NULs).

    python tests/golden/make_golden_bert_tokenizer.py
"""
import dataclasses
import io
import os
import re
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

graft.load_package()

OUT = os.path.join(HERE, "tokenizer", "bert_tokenizer.npz")
TEXT_ENCODING_OFFSET, TEXT_PAD, SEMANTIC_PAD, SEMANTIC_INFER = 10048, 129595, 10000, 129599     # bark_context_default_params

SENTENCES = [
    ("en", "Hello, my name is Suno. And, uh — and I like pizza. [laughs] But I also have other interests such as playing tic tac toe."),
    ("de", "Guten Tag! Die Straße in Zürich ist heute sehr schön, oder?"),
    ("es", "¿Dónde está la biblioteca? Mañana será otro día."),
    ("fr", "Bonjour, je m'appelle Élodie et j'adore les crêpes à Noël."),
    ("hi", "नमस्ते, आप कैसे हैं? मैं ठीक हूँ।"),
    ("it", "Però la città è bellissima, perché no?"),
    ("ja", "こんにちは、元気ですか？今日は良い天気です。"),
    ("ko", "안녕하세요, 만나서 반갑습니다. 감사합니다!"),
    ("pl", "Zażółć gęślą jaźń, proszę pana."),
    ("pt", "Não sei, mas a lição é óbvia: coração."),
    ("ru", "Привет, как дела? Всё хорошо, спасибо."),
    ("tr", "Günaydın, nasılsın? Işık ğüzel değil mi?"),
    ("zh", "你好，我叫小明。今天天气很好！"),
]
DUPLICATE = "Zürich"             # in the vocabulary twice: the later id wins

CASES = [(f"lang_{k}", t) for k, t in SENTENCES] + [
    ("mixed_scripts", "Hello мир, 你好 world: Straße café 123 नमस्ते 안녕"),
    ("cjk_ext_b", "𠀀𠀁 𪚥 x𠀂y 你𠀀好"),
    ("emoji_zwj", "I \u2764\ufe0f you \U0001f468\u200d\U0001f469\u200d\U0001f467 family \U0001f389! \U0001f44d\U0001f3fd"),
    ("combining", "x\u0303x a\u0301 Zu\u0308rich Z\u00fcrich"),
    ("decomposed_e", "caf\u00e9 cafe\u0301"),   # NFC and decomposed: the oracle applies no NFC, so the two differ
    ("spaces_controls", "a\u00a0b\u3000c\u0085d\u2028e\x1cf\tg\nh\ue000i\x7fj\u200bk\ufffdl\x0bm\x01n"),
    ("empty", ""),
    ("whitespace_only", " \t\n\u3000\u00a0\x1c "),
    ("word_100", "a" * 100),
    ("word_101", "a" * 101),
    ("word_100_cjk_tail", "b" * 99 + "你"),
    ("fails_halfway", "hello helloΩ Ωhello hel"),
    ("abc123", "abc123 123abc a1b2c3"),
    ("specials", "[PAD] [UNK] [CLS] [SEP] [MASK]"),
    ("specials_in_words", "un[MASK]known x[SEP]y[CLS]z [[MASK]] [mask] [MASK [PAD[UNK]"),
    ("laughs", "[laughs] Hello [laughs] there [music] ♪ la la ♪"),
    ("duplicate", f"{DUPLICATE} {DUPLICATE}!"),
    ("pieces_255", " ".join(["a"] * 255)),
    ("pieces_256", " ".join(["a"] * 256)),
    ("pieces_300_plus", "x, " * 160 + "Привет мир"),
]


def _tokenizer(vocab):
    from transformers import BertTokenizer
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "vocab.txt")
        with open(path, "w", encoding="utf-8") as f:
            f.write("".join(v + "\n" for v in vocab))
        return BertTokenizer(path, do_lower_case=False)


def upstream_ids(tok, texts):
    """Upstream Bark's rule: _normalize_whitespace, then encode without special tokens."""
    texts = [re.sub(r"\s+", " ", t).strip() for t in texts]
    return tok(texts, add_special_tokens=False)["input_ids"]


def extra_words(weights):
    """Deterministic pieces of the sample sentences' words: whole words, character pieces, multi-character pieces, or nothing."""
    from tokenizers import normalizers, pre_tokenizers
    norm = normalizers.BertNormalizer(clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=False)
    pre = pre_tokenizers.BertPreTokenizer()
    base = set(weights.synth_vocab(dataclasses.replace(weights.tiny(), extra_words=[])))
    out, seen = [], set(base)

    def add(p):
        if p not in seen:
            seen.add(p)
            out.append(p)

    i = 0
    for _, s in SENTENCES:
        for w, _ in pre.pre_tokenize_str(norm.normalize_str(s)):
            if w.isascii():
                continue
            rule = i % 4
            i += 1
            if rule == 0 or len(w) == 1:
                add(w)
            elif rule == 1:
                add(w[0])
                for c in w[1:]:
                    add("##" + c)
            elif rule == 2:
                add(w[:2])
                add("##" + w[2:] if len(w) > 2 else w)
                for c in w:
                    add(c)
                    add("##" + c)
    for p in ("Str", "##aße", "##ße", "##ß", "При", "##вет", "мир", "你好", "天气", "##\u0301", "\U0001f600", "\u2764", "\U0001f389", "##s",
              DUPLICATE):
        add(p)
    out.append(DUPLICATE)
    return out


def _blob(strings):
    data = [s.encode("utf-8") for s in strings]
    off = np.zeros(len(data) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in data])
    return np.frombuffer(b"".join(data), np.uint8).copy(), off


def _write_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps, so the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w") as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue(), compresslevel=9)


def main():
    import tokenizers
    import transformers
    weights = graft.importlib.import_module("bark_cpp_b200.weights")      # plain Python: no library needed
    extra = extra_words(weights)
    vocab = weights.synth_vocab(dataclasses.replace(weights.tiny(), extra_words=extra))
    tok = _tokenizer(vocab)
    v = tok.get_vocab()
    later = max(i for i, t in enumerate(vocab) if t == DUPLICATE)
    assert vocab.count(DUPLICATE) == 2 and v[DUPLICATE] == later, "the oracle does not let the later duplicate win"

    names = [n for n, _ in CASES]
    texts = [t for _, t in CASES]
    ids = upstream_ids(tok, texts)
    prompt = np.zeros((len(CASES), 513), np.int32)
    for i, x in enumerate(ids):
        p = [t + TEXT_ENCODING_OFFSET for t in x[:256]]
        p += [TEXT_PAD] * (256 - len(p)) + [SEMANTIC_PAD] * 256 + [SEMANTIC_INFER]
        prompt[i] = p

    cps = [cp for cp in range(0x110000) if not 0xD800 <= cp <= 0xDFFF]
    first, run_ids, prev = [], [], None
    for s in range(0, len(cps), 65536):
        chunk = cps[s:s + 65536]
        for cp, x in zip(chunk, upstream_ids(tok, ["x" + chr(cp) + "x" for cp in chunk])):
            assert 1 <= len(x) <= 3, (hex(cp), x)
            t = tuple(x) + (-1,) * (3 - len(x))
            if t != prev:
                first.append(cp)
                run_ids.append(t)
                prev = t

    vb, vo = _blob(vocab)
    eb, eo = _blob(extra)
    nb, no = _blob(names)
    tb, to = _blob(texts)
    flat = np.array([t for x in ids for t in x], np.int32)
    io_ = np.zeros(len(ids) + 1, np.int64)
    io_[1:] = np.cumsum([len(x) for x in ids])
    vb2, vo2 = _blob([f"transformers {transformers.__version__}", f"tokenizers {tokenizers.__version__}"])
    _write_npz(OUT, dict(vocab_bytes=vb, vocab_offsets=vo, extra_bytes=eb, extra_offsets=eo, name_bytes=nb, name_offsets=no,
                         text_bytes=tb, text_offsets=to, ids=flat, ids_offsets=io_, prompt=prompt,
                         cp_first=np.array(first, np.int32), cp_ids=np.array(run_ids, np.int32),
                         versions_bytes=vb2, versions_offsets=vo2))
    print(f"wrote {OUT}: {len(vocab)} vocabulary entries, {len(CASES)} texts, {len(first)} code point runs "
          f"(transformers {transformers.__version__}, tokenizers {tokenizers.__version__})")


if __name__ == "__main__":
    main()
