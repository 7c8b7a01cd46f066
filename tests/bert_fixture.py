"""Reads tests/golden/tokenizer/bert_tokenizer.npz (written by tests/golden/make_golden_bert_tokenizer.py): upstream Bark's text ids from the
oracle, for tests/test_bert_tokenizer.py and tests/test_bert_tokenizer_gpu.py."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tokenizer", "bert_tokenizer.npz")


def _strings(f, key):
    b, off = f[key + "_bytes"].tobytes(), f[key + "_offsets"]
    return [b[off[i]:off[i + 1]].decode("utf-8") for i in range(len(off) - 1)]


def load() -> dict:
    """vocab, extra_words, cases [(name, text, ids)], prompt [n][513], cp_first [R], cp_ids [R][3] (-1 padded), versions."""
    with np.load(PATH) as f:
        names, texts = _strings(f, "name"), _strings(f, "text")
        ids, off = f["ids"], f["ids_offsets"]
        return dict(vocab=_strings(f, "vocab"), extra_words=_strings(f, "extra"), versions=_strings(f, "versions"),
                    cases=[(n, t, ids[off[i]:off[i + 1]].copy()) for i, (n, t) in enumerate(zip(names, texts))],
                    prompt=f["prompt"].copy(), cp_first=f["cp_first"].copy(), cp_ids=f["cp_ids"].copy())


def code_point_ids(g: dict):
    """(code point, its oracle ids for "x" + c + "x") for every code point but the surrogates, in order."""
    first, rows = g["cp_first"], g["cp_ids"]
    for r in range(len(first)):
        end = int(first[r + 1]) if r + 1 < len(first) else 0x110000
        want = rows[r][rows[r] >= 0]
        for cp in range(int(first[r]), end):
            if not 0xD800 <= cp <= 0xDFFF:
                yield cp, want
