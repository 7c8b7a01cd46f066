// Long-form generation (DESIGN.md §18): upstream Bark's long-form recipe behind bark_generate_audio.  The text is split into sentences,
// over-long sentences into pieces the prompt can hold, and each chunk is one ordinary generation on the context, prompted so that the
// voice stays the same; the waveforms are joined with silence.  Host code only: every chunk runs the existing device stages.
//
//   1. normalise  strict UTF-8 (tokenizer.cu decode_utf8); every run of Python's \s one space, both ends stripped (upstream's
//                 _normalize_whitespace)
//   2. sentences  a run of end marks, with the closing marks directly after it, ends a sentence when the run holds a mark that needs no
//                 space (。！？｡।॥) or a space or the end of the text follows; that space is dropped.  No abbreviation list.
//   3. pieces     a sentence over the id budget: greedy by words, a word over the budget alone greedy by code points
//   4. drop, cap  chunks without ids dropped; none left or more than kLongFormMaxChunks refused
//   5. voice      chain: chunk k > 0 prompted by chunk k - 1's own ids when they are a valid prompt, else by chunk k - 1's prompt;
//                 fixed: every chunk by the context's prompt
#include "context.h"

#include <algorithm>
#include <cstdio>

namespace {

// ends a sentence without a space after it
bool strong_end(uint32_t c) { return c == 0x3002 || c == 0xFF01 || c == 0xFF1F || c == 0xFF61 || c == 0x0964 || c == 0x0965; }
// ends a sentence when a space or the end of the text follows
bool weak_end(uint32_t c) { return c == '.' || c == '!' || c == '?' || c == 0x2026; }
// a closing mark that stays with the sentence before it
bool closing(uint32_t c) {
    static const uint32_t k[] = {'"', '\'', ')', ']', '}', 0x00BB, 0x201D, 0x2019, 0x300D, 0x300F, 0xFF09};
    return std::find(std::begin(k), std::end(k), c) != std::end(k);
}

// Chunk k - 1's own ids as a history prompt, codebook-major as upstream's voice files hold them; false (with make_history_prompt's message)
// when they are not a valid one
bool own_prompt(const bark_context_params & P, const Generation & g, HistoryPrompt & h) {
    const int n_c = (int) g.coarse_tokens.size() / 2, n_f = (int) g.fine_tokens.size() / 8;
    std::vector<int32_t> c((size_t) 2 * n_c), f((size_t) 8 * n_f);
    for (int t = 0; t < n_c; t++) for (int k = 0; k < 2; k++) c[(size_t) k * n_c + t] = g.coarse_tokens[(size_t) t * 2 + k];
    for (int t = 0; t < n_f; t++) for (int q = 0; q < 8; q++) f[(size_t) q * n_f + t] = g.fine_tokens[(size_t) t * 8 + q];
    const bark_b200_history_prompt p{g.semantic_tokens.data(), (int) g.semantic_tokens.size(), c.data(), n_c, f.data(), n_f};
    return bark::make_history_prompt(P, p, h);
}

}  // namespace

namespace bark {

int split_text(const std::string & text, int max_ids, const std::function<int(const std::string &)> & count, std::string & norm,
               std::vector<std::pair<size_t, size_t>> & bounds, const char * fn) {
    if (max_ids < 1 || max_ids > 255) { fprintf(stderr, "%s: max_chunk_ids %d (1 to 255)\n", fn, max_ids); return -1; }
    std::vector<uint32_t> raw, cp;
    size_t bad = 0;
    if (!decode_utf8(text, raw, &bad)) { fprintf(stderr, "%s: invalid UTF-8 at byte %zu of the text\n", fn, bad); return -1; }
    for (uint32_t c : raw) {
        if (!py_space(c)) cp.push_back(c);
        else if (!cp.empty() && cp.back() != ' ') cp.push_back(' ');
    }
    if (!cp.empty() && cp.back() == ' ') cp.pop_back();
    const size_t n = cp.size();
    std::vector<size_t> off(n + 1);                          // byte offset of code point i in norm
    norm.clear();
    for (size_t i = 0; i < n; i++) { off[i] = norm.size(); append_utf8(norm, cp[i]); }
    off[n] = norm.size();
    bounds.clear();
    auto ids = [&](size_t a, size_t b) { return count(norm.substr(off[a], off[b] - off[a])); };
    // A chunk of code points [a, b): kept when it has ids.  False for a failed count or one chunk too many.
    bool failed = false;
    auto emit = [&](size_t a, size_t b, int c) {
        if (c < 0) { failed = true; return false; }
        if (c > 0) bounds.emplace_back(off[a], off[b]);
        if ((int) bounds.size() > kLongFormMaxChunks) { fprintf(stderr, "%s: more than %d chunks\n", fn, kLongFormMaxChunks); failed = true; }
        return !failed;
    };
    auto word_end = [&](size_t p, size_t b) { while (p < b && cp[p] != ' ') p++; return p; };
    // Rule 3 on the sentence [a, b): greedy by words, a first word over the budget alone greedy by code points (at least one)
    auto sentence = [&](size_t a, size_t b) {
        const int whole = ids(a, b);
        if (whole <= max_ids) return emit(a, b, whole);
        for (size_t p = a; p < b;) {
            size_t e = word_end(p, b);
            int c = ids(p, e);
            if (c < 0) return emit(p, e, c);
            if (c > max_ids) {
                size_t q = p + 1;
                for (int cq; q < e && (cq = ids(p, q + 1)) <= max_ids; q++) if (cq < 0) return emit(p, q + 1, cq);
                if (!emit(p, q, ids(p, q))) return false;
                p = q;                                        // the rest of the word begins the rest of the sentence
                continue;
            }
            while (e < b) {
                const size_t next = word_end(e + 1, b);
                const int cn = ids(p, next);
                if (cn < 0) return emit(p, next, cn);
                if (cn > max_ids) break;
                e = next; c = cn;
            }
            if (!emit(p, e, c)) return false;
            p = e < b ? e + 1 : b;                            // the space at the split is dropped
        }
        return true;
    };
    size_t start = 0;
    for (size_t i = 0; i < n && !failed;) {
        if (!strong_end(cp[i]) && !weak_end(cp[i])) { i++; continue; }
        size_t j = i; bool strong = false;
        while (j < n && (strong_end(cp[j]) || weak_end(cp[j]))) strong |= strong_end(cp[j++]);
        while (j < n && closing(cp[j])) j++;
        if (strong || j == n || cp[j] == ' ') {
            if (j > start && !sentence(start, j)) break;
            if (j < n && cp[j] == ' ') j++;
            start = j;
        }
        i = j;
    }
    if (!failed && start < n) sentence(start, n);
    if (failed) return -1;
    if (bounds.empty()) { fprintf(stderr, "%s: the text leaves no chunk with text ids\n", fn); return -1; }
    return (int) bounds.size();
}

bool generate_long(bark_context * ctx, const std::string & text) {
    const char * fn = "bark_generate_audio";
    const bark_b200_long_form lf = ctx->long_form.settings;
    if (ctx->shard.on) { fprintf(stderr, "%s: long-form generation is not available on a context whose fine stage is sharded over GPUs\n", fn); return false; }
    std::string norm;
    std::vector<std::pair<size_t, size_t>> bounds;
    const auto count = [&](const std::string & t) { return count_text_ids(ctx->token_to_id, ctx->tokenizer, t, fn); };
    if (split_text(text, lf.max_chunk_ids, count, norm, bounds, fn) < 0) return false;     // refused: nothing has changed

    const int64_t t0 = now_us();
    Generation & g = ctx->gen;
    struct RestorePrompt {                                    // the context's prompt is back on every way out
        Generation & g; HistoryPrompt saved;
        ~RestorePrompt() { g.prompt = std::move(saved); }
    } restore{g, g.prompt};
    GPTModel * const models[3] = {&ctx->semantic, &ctx->coarse, &ctx->fine};
    int64_t samples0[3];
    for (int i = 0; i < 3; i++) samples0[i] = models[i]->n_sample;
    bark_statistics sum{};
    std::vector<LongFormChunk> chunks;
    std::vector<float> audio;
    ctx->long_form.chunks.clear();
    for (size_t k = 0; k < bounds.size(); k++) {
        if (k > 0 && lf.voice == BARK_B200_VOICE_CHAIN) {
            HistoryPrompt h;
            if (own_prompt(ctx->params, g, h)) g.prompt = std::move(h);
            else fprintf(stderr, "%s: chunk %zu's ids are not a valid prompt; chunk %zu keeps its prompt\n", fn, k - 1, k);
        }
        const std::string chunk = norm.substr(bounds[k].first, bounds[k].second - bounds[k].first);
        if (!generate_one(ctx, chunk)) { fprintf(stderr, "%s: chunk %zu of %zu failed\n", fn, k, bounds.size()); return false; }
        sum.t_semantic_us += ctx->stats.t_semantic_us; sum.t_coarse_us += ctx->stats.t_coarse_us; sum.t_fine_us += ctx->stats.t_fine_us;
        if (k > 0) audio.insert(audio.end(), (size_t) lf.gap_samples, 0.0f);
        audio.insert(audio.end(), g.audio.begin(), g.audio.end());
        chunks.push_back({chunk, g.tokens, g.semantic_tokens, g.coarse_tokens, g.fine_tokens});
    }
    g.audio.swap(audio);
    sum.t_load_us = ctx->stats.t_load_us;
    sum.n_sample_semantic = (int32_t)(models[0]->n_sample - samples0[0]);
    sum.n_sample_coarse = (int32_t)(models[1]->n_sample - samples0[1]);
    sum.n_sample_fine = (int32_t)(models[2]->n_sample - samples0[2]);
    sum.t_eval_us = now_us() - t0;
    ctx->stats = sum;
    ctx->long_form.chunks.swap(chunks);
    return true;
}

}  // namespace bark
