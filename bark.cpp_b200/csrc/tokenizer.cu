// The text tokenizers of a bark_context (bark_b200_set_tokenizer, BARK_B200_TOKENIZER).  Host code only: a prompt is at most 256 pieces.
// The reference's, the default (bark.cpp:480-662): 52 Latin-1 accents folded, [[:punct:]]|[[:alpha:]]+|[[:digit:]]+, greedy WordPiece.
// Upstream Bark's (bark/generation.py): BertTokenizer("bert-base-multilingual-cased").encode(_normalize_whitespace(text),
// add_special_tokens=False), restated on the host (DESIGN.md §17):
//   1. whitespace   every run of Python's \s (str.isspace) becomes one space, both ends stripped
//   2. UTF-8        decoded strictly; invalid input is refused
//   3. specials     [PAD] [UNK] [CLS] [SEP] [MASK] found literally are whole tokens (before normalisation, as tokenizers' added tokens)
//   4. classes      per code point (bert_chars.h, generated from the oracle): removed, space, CJK (a word of its own), punctuation
//                   (a word of one character), word character
//   5. WordPiece    greedy longest match with ## continuations; a word of more than 100 code points, or one with a position that
//                   matches nothing, is one [UNK]
#include "context.h"
#include "bert_chars.h"

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace {

// ---------------------------------------------------------------------------------------------
// the reference's tokenizer (bark.cpp:480-620)
// ---------------------------------------------------------------------------------------------
inline bool is_alpha(unsigned char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
inline bool is_digit(unsigned char c) { return c >= '0' && c <= '9'; }
inline bool is_punct(unsigned char c) { return c > 32 && c < 127 && !is_alpha(c) && !is_digit(c); }

// Latin-1 letters with diacritics (two-byte UTF-8, lead 0xC3) -> base ASCII letter; 0 if not mapped.
// Same 52 code points as the reference's table (bark.cpp:488-541).
char fold_accent(unsigned char second) {
    const unsigned cp = 0xC0u + (second - 0x80u);          // U+00C0 .. U+00FF
    const bool lower = cp >= 0xE0;
    const unsigned up = lower ? cp - 0x20 : cp;
    char base = 0;
    if (up >= 0xC0 && up <= 0xC5) base = 'A';
    else if (up == 0xC7) base = 'C';
    else if (up >= 0xC8 && up <= 0xCB) base = 'E';
    else if (up >= 0xCC && up <= 0xCF) base = 'I';
    else if (up == 0xD1) base = 'N';
    else if (up >= 0xD2 && up <= 0xD6) base = 'O';
    else if (up >= 0xD9 && up <= 0xDC) base = 'U';
    else if (up == 0xDD) base = 'Y';
    if (!base) return 0;
    return lower ? (char)(base + 32) : base;
}

std::string strip_accents_utf8(const std::string & in) {
    std::string out;
    for (size_t i = 0; i < in.size();) {
        const unsigned char c = (unsigned char) in[i];
        const unsigned hi = c >> 4;
        size_t len = hi < 12 ? 1 : hi < 14 ? 2 : hi == 14 ? 3 : 4;      // lead-byte length table, bark.cpp:480-484
        len = std::min(len, in.size() - i);
        char folded = 0;
        if (len == 2 && c == 0xC3) { const unsigned char d = (unsigned char) in[i + 1]; if (d >= 0x80 && d <= 0xBF) folded = fold_accent(d); }
        if (folded) out.push_back(folded); else out.append(in, i, len);
        i += len;
    }
    return out;
}

// bert_tokenize (bark.cpp:558-620); warn: the reference's message for a character no entry matches
void wordpiece(const std::map<std::string, int32_t> & vocab, const std::string & text, std::vector<int32_t> & out, int n_max_tokens, bool warn = true) {
    const std::string s = strip_accents_utf8(text);
    out.clear();
    size_t i = 0;
    while (i < s.size()) {
        const unsigned char c = (unsigned char) s[i];
        size_t j = i;
        if (is_punct(c)) j = i + 1;
        else if (is_alpha(c)) { while (j < s.size() && is_alpha((unsigned char) s[j])) j++; }
        else if (is_digit(c)) { while (j < s.size() && is_digit((unsigned char) s[j])) j++; }
        else { i++; continue; }
        const std::string word = s.substr(i, j - i);
        i = j;
        size_t p = 0; bool cont = false;
        while (p < word.size()) {
            if ((int) out.size() >= n_max_tokens - 1) break;
            size_t e = word.size(); bool hit = false;
            for (; e > p; e--) {
                auto it = vocab.find((cont ? "##" : "") + word.substr(p, e - p));
                if (it != vocab.end()) { out.push_back(it->second); p = e; cont = true; hit = true; break; }
            }
            if (!hit) { if (warn) fprintf(stderr, "%s: unknown token '%c'\n", "bert_tokenize", word[p]); cont = true; p++; }
        }
    }
}

using namespace bark::bert_chars;

Class char_class(uint32_t cp) {
    const Run * r = std::upper_bound(kRuns, kRuns + kNumRuns, cp, [](uint32_t c, const Run & x) { return c < x.first; });
    return (Class) r[-1].cls;
}

}  // namespace

// shared with the long-form splitter (long_form.cu)
namespace bark {

bool py_space(uint32_t cp) {
    for (const bert_chars::Range & r : bert_chars::kPySpace) if (cp >= r.lo && cp <= r.hi) return true;
    return false;
}

// Strict UTF-8 (RFC 3629): no overlong forms, no surrogates, nothing past U+10FFFF.  false with the offending byte's offset.
bool decode_utf8(const std::string & s, std::vector<uint32_t> & out, size_t * bad) {
    out.clear();
    for (size_t i = 0; i < s.size();) {
        const unsigned char c = (unsigned char) s[i];
        int len; uint32_t cp, min;
        if (c < 0x80) { out.push_back(c); i++; continue; }
        else if (c >= 0xC2 && c <= 0xDF) { len = 2; cp = c & 0x1F; min = 0x80; }
        else if (c >= 0xE0 && c <= 0xEF) { len = 3; cp = c & 0x0F; min = 0x800; }
        else if (c >= 0xF0 && c <= 0xF4) { len = 4; cp = c & 0x07; min = 0x10000; }
        else { *bad = i; return false; }                              // a continuation byte, an overlong lead (C0, C1) or F5..FF
        if (i + (size_t) len > s.size()) { *bad = i; return false; }
        for (int k = 1; k < len; k++) {
            const unsigned char d = (unsigned char) s[i + (size_t) k];
            if ((d & 0xC0) != 0x80) { *bad = i; return false; }
            cp = cp << 6 | (d & 0x3F);
        }
        if (cp < min || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) { *bad = i; return false; }
        out.push_back(cp);
        i += (size_t) len;
    }
    return true;
}

void append_utf8(std::string & s, uint32_t cp) {
    if (cp < 0x80) s.push_back((char) cp);
    else if (cp < 0x800) { s.push_back((char)(0xC0 | cp >> 6)); s.push_back((char)(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) { s.push_back((char)(0xE0 | cp >> 12)); s.push_back((char)(0x80 | (cp >> 6 & 0x3F))); s.push_back((char)(0x80 | (cp & 0x3F))); }
    else { s.push_back((char)(0xF0 | cp >> 18)); s.push_back((char)(0x80 | (cp >> 12 & 0x3F))); s.push_back((char)(0x80 | (cp >> 6 & 0x3F))); s.push_back((char)(0x80 | (cp & 0x3F))); }
}

}  // namespace bark

namespace {

using bark::append_utf8;

// WordPiece of one word (tokenizers' WordPiece::tokenize): at each position the longest vocabulary entry, "##" after the first piece,
// shortened one code point at a time
void wordpiece_word(const std::map<std::string, int32_t> & vocab, const std::vector<uint32_t> & word, int32_t unk, std::vector<int32_t> & out) {
    if (word.size() > 100) { out.push_back(unk); return; }                       // max_input_chars_per_word
    const size_t n0 = out.size();
    std::string piece;
    for (size_t start = 0; start < word.size();) {
        size_t end = word.size();
        for (; end > start; end--) {
            piece.assign(start > 0 ? "##" : "");
            for (size_t k = start; k < end; k++) append_utf8(piece, word[k]);
            const auto it = vocab.find(piece);
            if (it != vocab.end()) { out.push_back(it->second); break; }
        }
        if (end == start) { out.resize(n0); out.push_back(unk); return; }       // no piece at this position: the whole word is [UNK]
        start = end;
    }
}

// Normalisation, pre-tokenisation and WordPiece of a stretch of text between specials
void tokenize_span(const std::map<std::string, int32_t> & vocab, const uint32_t * cp, size_t n, int32_t unk, std::vector<int32_t> & out) {
    std::vector<uint32_t> word;
    auto flush = [&] { if (!word.empty()) { wordpiece_word(vocab, word, unk, out); word.clear(); } };
    for (size_t i = 0; i < n; i++) {
        switch (char_class(cp[i])) {
            case kRemoved: break;
            case kSpace: flush(); break;
            case kCJK: case kPunct: flush(); word.push_back(cp[i]); flush(); break;
            case kWord: word.push_back(cp[i]); break;
        }
    }
    flush();
}

}  // namespace

namespace bark {

bool bert_tokenize(const std::map<std::string, int32_t> & vocab, const std::string & text, std::vector<int32_t> & out, const char * fn) {
    out.clear();
    std::vector<uint32_t> raw, cp;
    size_t bad = 0;
    if (!decode_utf8(text, raw, &bad)) { fprintf(stderr, "%s: invalid UTF-8 at byte %zu of the text\n", fn, bad); return false; }
    const auto unk_it = vocab.find("[UNK]");
    if (unk_it == vocab.end()) { fprintf(stderr, "%s: the vocabulary has no [UNK] entry\n", fn); return false; }
    // upstream's _normalize_whitespace: re.sub(r"\s+", " ", text).strip()
    for (uint32_t c : raw) {
        if (!py_space(c)) cp.push_back(c);
        else if (!cp.empty() && cp.back() != ' ') cp.push_back(' ');
    }
    if (!cp.empty() && cp.back() == ' ') cp.pop_back();
    // the five specials, matched literally before normalisation; one that the vocabulary lacks is ordinary text
    static const char * const kSpecials[] = {"[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"};
    size_t span = 0;
    for (size_t i = 0; i < cp.size(); i++) {
        if (cp[i] != '[') continue;
        for (const char * sp : kSpecials) {
            const size_t len = strlen(sp);
            if (i + len > cp.size() || !std::equal(sp, sp + len, cp.begin() + (std::ptrdiff_t) i)) continue;
            const auto it = vocab.find(sp);
            if (it == vocab.end()) continue;
            tokenize_span(vocab, cp.data() + span, i - span, unk_it->second, out);
            out.push_back(it->second);
            span = i + len;
            i = span - 1;
            break;
        }
    }
    tokenize_span(vocab, cp.data() + span, cp.size() - span, unk_it->second, out);
    return true;
}

bool tokenizer_known(int kind, const char * fn) {
    if (kind == BARK_B200_TOKENIZER_REFERENCE || kind == BARK_B200_TOKENIZER_BERT) return true;
    fprintf(stderr, "%s: unknown tokenizer %d (0 reference, 1 bert)\n", fn, kind);
    return false;
}

int tokenizer_from_env(const char * fn) {
    const char * e = getenv("BARK_B200_TOKENIZER");
    if (!e || !*e || !strcmp(e, "reference")) return BARK_B200_TOKENIZER_REFERENCE;
    if (!strcmp(e, "bert")) return BARK_B200_TOKENIZER_BERT;
    fprintf(stderr, "%s: BARK_B200_TOKENIZER=%s is neither 'reference' nor 'bert'\n", fn, e);
    return -1;
}

bool text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, int cap, std::vector<int32_t> & ids, const char * fn,
              bool warn) {
    if (!tokenizer_known(kind, fn)) return false;
    if (kind == BARK_B200_TOKENIZER_REFERENCE) { wordpiece(vocab, text, ids, cap, warn); return true; }
    if (!bert_tokenize(vocab, text, ids, fn)) return false;
    ids.resize(std::min(ids.size(), (size_t) cap));
    return true;
}

int count_text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, const char * fn) {
    std::vector<int32_t> ids;
    return text_ids(vocab, kind, text, INT_MAX, ids, fn, false) ? (int) ids.size() : -1;
}

}  // namespace bark
