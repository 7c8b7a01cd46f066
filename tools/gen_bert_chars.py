"""Writes bark.cpp_b200/csrc/bert_chars.h: the character classes of upstream Bark's text tokenizer (DESIGN.md §17).

Upstream Bark tokenizes with transformers' BertTokenizer for bert-base-multilingual-cased, which runs the `tokenizers` pipeline
BertNormalizer(clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=False) -> BertPreTokenizer() -> WordPiece.
Both of the first two act on each code point alone, so every code point falls in one of five classes, read off the oracle here:

  removed  normalize_str(c) == ""         (NUL, U+FFFD, controls, format, unassigned and private-use code points)
  space    normalize_str(c) == " "        (replaced by a space: a word boundary)
  cjk      normalize_str(c) == " c "      (padded with spaces: a word of its own)
  punct    normalize_str(c) == c and pre_tokenize_str("x" + c + "x") gives 3 pieces   (a word of one character)
  word     normalize_str(c) == c and it gives 1 piece

Any other outcome stops the script.  Upstream first applies re.sub(r"\\s+", " ", text).strip(); the set of that \\s (str.isspace) is
written too.  Surrogates never come out of the UTF-8 decoder; they are listed as removed.

    python tools/gen_bert_chars.py            # rewrites the header
"""
from __future__ import annotations

import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "bark.cpp_b200", "csrc", "bert_chars.h")
CLASSES = ("word", "punct", "cjk", "space", "removed")
MAX_CP = 0x10FFFF


def _pipeline():
    from tokenizers import normalizers, pre_tokenizers
    norm = normalizers.BertNormalizer(clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=False)
    pre = pre_tokenizers.BertPreTokenizer()
    try:                                           # the oracle's own pipeline, where transformers is installed: it must be this one
        import tempfile
        from transformers import BertTokenizer
        with tempfile.TemporaryDirectory() as d:
            v = os.path.join(d, "vocab.txt")
            with open(v, "w") as f:
                f.write("[PAD]\n[UNK]\n[CLS]\n[SEP]\n[MASK]\n")
            bt = BertTokenizer(v, do_lower_case=False).backend_tokenizer
        assert repr(bt.normalizer) == repr(norm) and repr(bt.pre_tokenizer) == repr(pre), (bt.normalizer, bt.pre_tokenizer)
    except ImportError:
        pass
    return norm, pre


def classify() -> list:
    """Class index (CLASSES) of every code point 0 .. 0x10FFFF."""
    norm, pre = _pipeline()
    cls = [CLASSES.index("removed")] * (MAX_CP + 1)
    for cp in range(MAX_CP + 1):
        if 0xD800 <= cp <= 0xDFFF:
            continue
        c = chr(cp)
        n = norm.normalize_str(c)
        if n == "":
            k = "removed"
        elif n == " ":
            k = "space"
        elif n == " " + c + " ":
            k = "cjk"
        elif n == c:
            pieces = [p for p, _ in pre.pre_tokenize_str("x" + c + "x")]
            if pieces == ["x", c, "x"]:
                k = "punct"
            elif pieces == ["x" + c + "x"]:
                k = "word"
            else:
                raise SystemExit(f"U+{cp:04X}: pre-tokenized to {pieces!r}, neither punctuation nor a word character")
        else:
            raise SystemExit(f"U+{cp:04X}: normalized to {n!r}, none of the five classes")
        cls[cp] = CLASSES.index(k)
    return cls


def py_space() -> list:
    """[lo, hi] ranges of the code points Python's str.isspace (and so re's \\s) accepts."""
    cps = [cp for cp in range(MAX_CP + 1) if not 0xD800 <= cp <= 0xDFFF and chr(cp).isspace()]
    for cp in range(MAX_CP + 1):
        if not 0xD800 <= cp <= 0xDFFF:
            assert bool(re.fullmatch(r"\s", chr(cp))) == chr(cp).isspace(), f"U+{cp:04X}"
    out = []
    for cp in cps:
        if out and out[-1][1] == cp - 1:
            out[-1][1] = cp
        else:
            out.append([cp, cp])
    return out


def body(cls: list, spaces: list) -> str:
    """The header without its provenance comment."""
    runs = [(0, cls[0])]
    for cp in range(1, MAX_CP + 1):
        if cls[cp] != runs[-1][1]:
            runs.append((cp, cls[cp]))
    counts = {k: sum(1 for cp in range(MAX_CP + 1) if cls[cp] == i and not 0xD800 <= cp <= 0xDFFF) for i, k in enumerate(CLASSES)}
    lines = ["#pragma once", "#include <cstdint>", "", "namespace bark {", "namespace bert_chars {", "",
             "// " + ", ".join(f"{k} {v}" for k, v in counts.items()) + " code points (surrogates aside)",
             "enum Class : uint8_t { kWord = 0, kPunct = 1, kCJK = 2, kSpace = 3, kRemoved = 4 };",
             "// code points [first, the next run's first) are of class cls; the last run ends at U+10FFFF",
             "struct Run { uint32_t first; uint8_t cls; };",
             f"constexpr int kNumRuns = {len(runs)};",
             "constexpr Run kRuns[kNumRuns] = {"]
    for i in range(0, len(runs), 8):
        lines.append("    " + " ".join(f"{{0x{a:X}, {c}}}," for a, c in runs[i:i + 8]))
    lines += ["};", "", "// Python's str.isspace, the \\s of upstream's whitespace rule: [lo, hi]",
              "struct Range { uint32_t lo, hi; };", f"constexpr int kNumPySpace = {len(spaces)};", "constexpr Range kPySpace[kNumPySpace] = {"]
    lines.append("    " + " ".join(f"{{0x{a:X}, 0x{b:X}}}," for a, b in spaces))
    lines += ["};", "", "}  // namespace bert_chars", "}  // namespace bark", ""]
    return "\n".join(lines)


def generate() -> str:
    """The whole header, as derived from the installed tokenizers now."""
    import tokenizers
    try:
        import transformers
        tv = f"transformers {transformers.__version__}, "
    except ImportError:
        tv = ""
    head = (f"// Generated by tools/gen_bert_chars.py from {tv}tokenizers {tokenizers.__version__}, Python "
            f"{sys.version_info.major}.{sys.version_info.minor}: do not edit.\n"
            "// Character classes of upstream Bark's BERT tokenizer (DESIGN.md §17), read off the oracle for every code point.\n")
    return head + body(classify(), py_space())


def strip_provenance(text: str) -> str:
    return "\n".join(l for l in text.split("\n") if not l.startswith("// Generated by"))


if __name__ == "__main__":
    text = generate()
    with open(HEADER, "w") as f:
        f.write(text)
    print(f"wrote {HEADER} ({len(text)} bytes)")
