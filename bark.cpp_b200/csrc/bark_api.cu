// The bark.h C API (include/bark.h) and the host control plane behind it: tokenizer, the three
// stage loops, statistics.  Semantics follow the reference's bark.cpp — including
// its quirks (SURVEY.md App. D) — because token parity depends on them; the code is new.
//
//   tokenizer ............ bark.cpp:480-662   (accent strip, [[:punct:]]|[[:alpha:]]+|[[:digit:]]+, greedy WordPiece)
//   semantic loop ........ bark.cpp:1645-1743
//   coarse loop .......... bark.cpp:1745-1905
//   fine loop ............ bark.cpp:1961-2104
//   generate / lifecycle . bark.cpp:1165-1184, 2125-2232, 2379-2407
#include "../../include/bark_b200.h"
#include "context.h"
#include "codec_kernels.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <stdexcept>

using namespace bark;

namespace {

thread_local int g_device_override = -1;   // bark_b200_set_device applies to the calling thread's next bark_load_model
bool quiet() { static const bool q = [] { const char * e = getenv("BARK_B200_QUIET"); return e && *e && *e != '0'; }(); return q; }

// ---------------------------------------------------------------------------------------------
// tokenizer
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

// bark.cpp:622-662, on the context's tokenizer: the reference's, or upstream Bark's (bert_tokenizer.cu), whose prompt keeps the first
// max_ctx ids.  false (message naming fn) for a text the BERT tokenizer refuses; g is then untouched.
bool tokenize_input(bark_context * ctx, Generation & g, const std::string & text, const char * fn) {
    const bark_context_params & P = ctx->params;
    const int max_ctx = std::min(ctx->semantic.block_size, 256);
    std::vector<int32_t> pieces;
    if (ctx->tokenizer == BARK_B200_TOKENIZER_BERT) {
        if (!bert_tokenize(ctx->token_to_id, text, pieces, fn)) return false;
        pieces.resize(std::min(pieces.size(), (size_t) max_ctx));
    } else {
        wordpiece(ctx->token_to_id, text, pieces, max_ctx);
    }
    std::vector<int32_t> t((size_t) max_ctx, 0);
    std::copy(pieces.begin(), pieces.end(), t.begin());
    for (auto & v : t) v += P.text_encoding_offset;                               // offset applied to every slot before padding (quirk D.4)
    for (size_t k = pieces.size(); k < t.size(); k++) t[k] = P.text_pad_token;
    const size_t hist0 = t.size();
    t.insert(t.end(), 256, P.semantic_pad_token);                                 // semantic history: empty without a prompt,
    const std::vector<int32_t> & S = g.prompt.semantic;                           // else the prompt's last 256 ids, right-padded
    const size_t n_hist = std::min<size_t>(S.size(), 256);
    std::copy(S.end() - (std::ptrdiff_t) n_hist, S.end(), t.begin() + (std::ptrdiff_t) hist0);
    t.push_back(P.semantic_infer_token);
    g.tokens = t;
    if (!quiet()) {
        printf("%s: prompt: '%s'\n", "bark_tokenize_input", text.c_str());
        printf("%s: number of tokens in prompt = %zu, first 8 tokens: ", "bark_tokenize_input", g.tokens.size());
        for (size_t k = 0; k < std::min<size_t>(8, g.tokens.size()); k++) printf("%d ", g.tokens[k]);
        printf("\n\n");
    }
    return true;
}

// The end of a stage: its sample count and time in the statistics (n_sample, t_us: the stage's fields), and the reference's printout
// (bark_print_statistics, bark.cpp:176-182).
void end_stage(GPTModel & m, int64_t t_start, int32_t & n_sample, int64_t & t_us) {
    n_sample = (int32_t) m.n_sample;
    m.t_main_us = now_us() - t_start;
    t_us = m.t_main_us;
    if (quiet()) return;
    printf("\n\n");
    printf("%s:   sample time = %8.2f ms / %lld tokens\n", "bark_print_statistics", m.t_sample_us / 1000.0f, (long long) m.n_sample);
    printf("%s:  predict time = %8.2f ms / %.2f ms per token\n", "bark_print_statistics", m.t_predict_us / 1000.0f,
           m.n_sample ? m.t_predict_us / (double) m.n_sample / 1000.0 : 0.0);
    printf("%s:    total time = %8.2f ms\n", "bark_print_statistics", m.t_main_us / 1000.0f);
    printf("\n");
}

// ---------------------------------------------------------------------------------------------
// stage loops
// ---------------------------------------------------------------------------------------------
// Runs `n` consecutive sampling steps of one causal stream with the sampler on the device (sampling.cu).  Step 0 evaluates
// `first_in` (a prompt or the single token the host already knows); every later step reads its input token from device
// memory, where the previous step's sampler left it — so all n decode + sample launches are enqueued without a host round
// trip and there is one synchronisation at the end.  lo_of(j) is the offset of step j's logit window in the vocabulary
// (samp_n logits wide); tokens come back with that offset added.  A step the kernel flags as too close to call (see
// sampling.cu) is replayed on the host with the reference's arithmetic and the same uniform draw, and the chain restarts
// behind it; tokens and RNG state are those of the reference's step-by-step loop either way.  Semantic and coarse run here, so
// the limits of the sampler (kSampleMaxLogits) and of the uniform / token buffers (1024 steps) are checked here.
template <typename LoOf>
bool run_chain(bark_context * ctx, std::mt19937 & rng, GPTModel & m, const std::vector<int32_t> & first_in, bool merge_ctx, int * n_past, int n, LoOf lo_of, int samp_n, float temp,
               const bark_b200_sampling & filt, int32_t * out_tok, float * out_eos) {
    if (n < 1 || n > 1024) { fprintf(stderr, "%s: %d steps in one chain (1 to 1024)\n", __func__, n); return false; }
    if (samp_n > kSampleMaxLogits) { fprintf(stderr, "%s: %d logits per sample exceed the device sampler's row of %d\n", __func__, samp_n, kSampleMaxLogits); return false; }
    const int64_t t_begin = now_us();
    cudaStream_t s = ctx->stream;
    if (temp != 0.0f) {
        for (int j = 0; j < n; j++) ctx->h_u[j] = std::generate_canonical<double, 53>(rng);     // one draw per sample, as the discrete distribution's operator() makes
        BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->d_u, ctx->h_u, (size_t) n * sizeof(double), cudaMemcpyHostToDevice, s)); bark::g_h2d_bytes += (size_t) n * sizeof(double);
    }
    const bool chain = ctx->use_decode_kernel && m.decode_ok, filtered = filter_on(filt);
    std::vector<int> past_before((size_t) n);
    std::vector<int32_t> cur_in = first_in;
    std::vector<float> host_logits;
    int start = 0;
    while (start < n) {
        const int stop = chain ? n : start + 1;
        for (int j = start; j < stop; j++) {
            const int lo = lo_of(j);
            past_before[(size_t) j] = *n_past;
            if (j == start) { if (!gpt_eval(ctx, m, cur_in.data(), (int) cur_in.size(), n_past, merge_ctx && *n_past == 0, nullptr, lo, lo + samp_n)) return false; }
            const int force = ctx->debug_flag_every > 0 && (ctx->n_sample_calls++ % ctx->debug_flag_every) == 0;
            if (j > start && !gpt_decode_chained(ctx, m, ctx->d_feed, n_past, lo, lo + samp_n)) return false;
            if (filtered) {                              // the filter's row, then the sampler on it: still no host round trip
                filter_rows(ctx->last_logits + lo, m.n_out_vocab, samp_n, 1, filt, ctx->d_frow, nullptr, ctx->d_fflags + j, 0, s);
                sample_rows(ctx->d_frow, samp_n, samp_n, 1, temp, ctx->d_u + j, ctx->d_stok + j, lo, ctx->d_feed, ctx->d_seos + j, ctx->d_sflags + j, force, 0, s);
            } else {
                sample_rows(ctx->last_logits + lo, m.n_out_vocab, samp_n, 1, temp, ctx->d_u + j, ctx->d_stok + j, lo, ctx->d_feed, ctx->d_seos + j, ctx->d_sflags + j, force, 0, s);
            }
        }
        read_back_samples(ctx, start, stop, true, filtered);
        int f = start;
        while (f < stop && !sample_flagged(ctx, f, filtered)) f++;
        if (f == stop) { start = stop; if (start < n) cur_in.assign(1, ctx->h_stok[start - 1]); continue; }
        // step f must be decided on the host: re-evaluate it with its logits read back (steps before f stand)
        if (f > start) cur_in.assign(1, ctx->h_stok[f - 1]);
        *n_past = past_before[(size_t) f];
        const int lo = lo_of(f);
        host_logits.resize((size_t) m.n_out_vocab);
        if (!gpt_eval(ctx, m, cur_in.data(), (int) cur_in.size(), n_past, merge_ctx && *n_past == 0, host_logits.data(), lo, lo + samp_n)) return false;
        if (filtered) filter_row_host(host_logits.data() + lo, samp_n, filt);
        ctx->h_stok[f] = lo + sample_token_given_u(host_logits.data() + lo, samp_n, temp, ctx->h_u[f], &ctx->h_seos[f]);
        ctx->n_sample_host_replays++;
        start = f + 1;
        cur_in.assign(1, ctx->h_stok[f]);
    }
    for (int j = 0; j < n; j++) { out_tok[j] = ctx->h_stok[j]; if (out_eos) out_eos[j] = ctx->h_seos[j]; }
    m.n_sample += n;
    m.t_predict_us += now_us() - t_begin;      // evaluation and sampling overlap on the device: the split the reference prints does not exist here
    return true;
}

// Bark's semantic stop rule (bark.cpp:1675-1677) for one sampled id and the probability of the last logit: the id is appended to
// `out` unless it stops the stage.  True when another step follows; the stage also ends with n_steps_text_encoder ids.
bool semantic_accept(const bark_context_params & P, std::vector<int32_t> & out, int32_t tok, float eos) {
    if (tok == P.semantic_vocab_size || eos >= P.min_eos_p) return false;
    out.push_back(tok);
    return (int) out.size() < P.n_steps_text_encoder;
}

bool run_semantic(bark_context * ctx, Generation & g) {
    const int64_t t_start = now_us();
    GPTModel & m = ctx->semantic;
    const bark_context_params & P = ctx->params;
    std::vector<int32_t> input = g.tokens, output;
    int n_past = 0;
    // batches of kBatch steps run ahead of the stop test; if the stop falls inside a batch, the RNG is wound back to
    // where the step-by-step loop would have left it and the surplus steps are dropped (their KV rows are never read)
    constexpr int kBatch = 64;
    std::vector<int32_t> tok(kBatch); std::vector<float> eos(kBatch);
    bool more = P.n_steps_text_encoder > 0;
    for (int i = 0; more; i += kBatch) {
        const int nb = std::min(kBatch, P.n_steps_text_encoder - i);
        const std::mt19937 saved = g.rng;
        // the reference samples over ALL n_out_vocab logits, not the 10001 "relevant" ones (quirk D.1)
        if (!run_chain(ctx, g.rng, m, input, true, &n_past, nb, [](int) { return 0; }, m.n_out_vocab, P.temp, ctx->sampling[0], tok.data(), eos.data())) { fprintf(stderr, "%s: Could not generate token\n", __func__); return false; }
        int used = 0;
        for (; more && used < nb; used++) {
            if (P.progress_callback) P.progress_callback(ctx, SEMANTIC, 100 * (i + used + 1) / P.n_steps_text_encoder, P.progress_callback_user_data);
            more = semantic_accept(P, output, tok[(size_t) used], eos[(size_t) used]);
        }
        if (used < nb) {                             // stopped inside the batch
            if (P.temp != 0.0f) { g.rng = saved; for (int k = 0; k < used; k++) (void) std::generate_canonical<double, 53>(g.rng); }
            m.n_sample -= nb - used;
        }
        if (more) input.assign(1, tok[(size_t) nb - 1]);
    }
    g.semantic_tokens = output;
    end_stage(m, t_start, ctx->stats.n_sample_semantic, ctx->stats.t_semantic_us);
    return true;
}

// The coarse stage of one generation (bark.cpp:1745-1905): its prompt history, the ids sampled so far and what its KV cache holds, and
// the stage's rules on them.  run_coarse drives one; the batch (batch_coarse) one per item, with every item's window w in one step.
struct CoarseStage {
    const bark_context_params * P = nullptr;
    std::vector<int32_t> sem;                        // the prompt's semantic history (n_sh ids), then the generation's semantic ids
    std::vector<int32_t> out;                        // the prompt's coarse history (n_ch ids), then the coarse ids sampled so far
    std::vector<int32_t> kv_ids;                     // ids whose K/V rows the cache holds, by position
    int n_sh = 0; size_t n_ch = 0;
    size_t kv_canon = 0;                             // leading rows of the cache known to be canonical (window)
    int n_steps = 0;                                 // coarse ids to sample

    float stc_ratio() const { return P->coarse_rate_hz / P->semantic_rate_hz * P->n_coarse_codebooks; }
    int max_semantic_history() const { return (int) floorf(P->max_coarse_history / stc_ratio()); }
    int n_windows() const { return (int) ceilf((float) n_steps / P->sliding_window_size); }
    int first_step(int w) const { return w * P->sliding_window_size; }
    int window_len(int w) const { return std::min(P->sliding_window_size, n_steps - first_step(w)); }
    // only logits [lo, lo + codebook_size) are ever looked at in this stage (bark.cpp:1829-1833): the window alternates with the codebook
    int lo(int step) const { return P->semantic_vocab_size + ((step % P->n_coarse_codebooks == 0) ? 0 : 1) * P->codebook_size; }

    // The step count (from the generated semantic ids only) and the prompt's history; false with a message naming `fn` for a model
    // whose logits do not hold the two codebook windows after the semantic ids, or for nothing to generate.
    bool setup(const bark_context_params & params, const GPTModel & m, const Generation & g, const char * fn) {
        P = &params;
        if (P->n_coarse_codebooks != 2 || P->semantic_vocab_size + 2 * P->codebook_size > m.n_out_vocab) {
            fprintf(stderr, "bark_b200: unsupported coarse codebook configuration (%d codebooks of %d after %d semantic ids, %d logits)\n",
                    P->n_coarse_codebooks, P->codebook_size, P->semantic_vocab_size, m.n_out_vocab);
            return false;
        }
        n_steps = (int)(floorf(g.semantic_tokens.size() * stc_ratio() / P->n_coarse_codebooks) * P->n_coarse_codebooks);
        if (n_steps <= 0) { fprintf(stderr, "%s: nothing to generate (%zu semantic tokens)\n", fn, g.semantic_tokens.size()); return false; }
        // The history (upstream Bark's generate_coarse): in sem the last n_sh semantic ids of the prompt, in out the last n_ch of its
        // coarse codes flattened the way the stage's ids are (c0[0], c1[0], c0[1], ..., codebook k offset by semantic_vocab_size +
        // k codebook_size) with the last two dropped (upstream's time alignment).  Both empty without a prompt.
        const HistoryPrompt & h = g.prompt;
        if (!h.empty()) {
            const int n_s = (int) h.semantic.size(), n_c = (int) h.coarse.size() / P->n_coarse_codebooks;
            n_sh = std::min({max_semantic_history(), n_s - n_s % 2, (int) floorf(2 * n_c / stc_ratio())});
            if (n_sh < 1) throw std::logic_error("CoarseStage: a validated prompt leaves no semantic history");   // ruled out by the alignment check
            const int ch = (int) roundf(n_sh * stc_ratio());
            sem.assign(h.semantic.end() - n_sh, h.semantic.end());
            for (int f = n_c * P->n_coarse_codebooks - ch; f < n_c * P->n_coarse_codebooks - 2; f++) {
                const int t = f / P->n_coarse_codebooks, k = f % P->n_coarse_codebooks;
                out.push_back(h.coarse[(size_t) k * n_c + t] + P->semantic_vocab_size + k * P->codebook_size);
            }
            n_ch = out.size();                       // ch less the two dropped
        }
        sem.insert(sem.end(), g.semantic_tokens.begin(), g.semantic_tokens.end());
        out.reserve(n_ch + (size_t) n_steps);
        return true;
    }

    // The prompt of window w and the part of it to evaluate: returns the ids from position *n_past on.  kv_ids / kv_canon are updated
    // to this prompt.
    std::vector<int32_t> window(bark_context * ctx, int w, int * n_past) {
        const int semantic_idx = n_sh + (int) roundf(first_step(w) / stc_ratio());
        // window input: semantic tokens from the history start TO THE END, cut/padded to 256 (quirk D.5), infer token, coarse history
        std::vector<int32_t> in(sem.begin() + std::max(semantic_idx - max_semantic_history(), 0), sem.end());
        in.resize(256, P->coarse_semantic_pad_token);
        in.push_back(P->coarse_infer_token);
        const size_t hist = std::min<size_t>((size_t) P->max_coarse_history, out.size());
        in.insert(in.end(), out.end() - (std::ptrdiff_t) hist, out.end());
        // Prefix reuse.  The reference re-evaluates the whole window prompt from n_past = 0 (bark.cpp:1795-1812).  Row p of
        // that evaluation depends on the ids at positions <= p and on the call's n_kv — but only through WHERE the summation
        // structure is cut: soft_max switches from the 8-wide polynomial to libm expf at column n_kv & ~7 and the P.V dot
        // from lane chains to the scalar leftovers at column n_kv & ~31 (ggml.c:2845-2888, 2144-2170).  For p < (n_kv & ~31)
        // every column beyond the cut is masked (an exact zero), so the row has ONE value whatever the call's n_kv:
        // "canonical".  Rows [0, n_kv & ~31) of every evaluation here are canonical (by induction over the layers), so a
        // window whose prompt starts with the ids the cache holds re-uses the canonical rows and evaluates the rest in one
        // call with the reference's own n_kv — bit-identical K/V rows and logits, 60-91 rows instead of 257-887.
        *n_past = 0;
        if (ctx->kv_reuse) {
            size_t common = 0;
            while (common < kv_ids.size() && common < in.size() && kv_ids[common] == in[common]) common++;
            *n_past = (int) std::min({common, kv_canon, in.size() & ~(size_t) 31, in.size() - 1});       // keep >= 1 id to evaluate
            ctx->n_kv_reused += (unsigned long long) *n_past;
        }
        kv_canon = std::max((size_t) *n_past, in.size() & ~(size_t) 31);
        std::vector<int32_t> in_eval(in.begin() + *n_past, in.end());
        kv_ids = in;
        return in_eval;
    }

    // The id sampled at step j of window w; true when another step of the window follows.  The window's last sample is never
    // evaluated, so it does not enter the cache.
    bool accept(int w, int j, int32_t tok) {
        out.push_back(tok);
        if (j + 1 >= window_len(w)) return false;
        kv_ids.push_back(tok);
        return true;
    }

    // the stage's flat ids (two interleaved codebook windows of the vocabulary) -> [T][2] codes
    void store(std::vector<int32_t> & coarse) const {
        coarse.resize(out.size() - n_ch);
        for (size_t i = 0; i + 1 < coarse.size(); i += 2) {
            coarse[i] = out[n_ch + i] - P->semantic_vocab_size;
            coarse[i + 1] = out[n_ch + i + 1] - P->semantic_vocab_size - P->codebook_size;
        }
    }
};

bool run_coarse(bark_context * ctx, Generation & g) {
    const int64_t t_start = now_us();
    GPTModel & m = ctx->coarse;
    const bark_context_params & P = ctx->params;
    CoarseStage cs;
    if (!cs.setup(P, m, g, __func__)) return false;
    for (int w = 0; w < cs.n_windows(); w++) {
        int n_past = 0;
        std::vector<int32_t> in_eval = cs.window(ctx, w, &n_past);
        const int nw = cs.window_len(w), step0 = cs.first_step(w);
        std::vector<int32_t> tok((size_t) nw);
        if (!run_chain(ctx, g.rng, m, in_eval, false, &n_past, nw, [&](int j) { return cs.lo(step0 + j); }, P.codebook_size, P.temp, ctx->sampling[1], tok.data(), nullptr)) { fprintf(stderr, "%s: Could not generate token\n", __func__); return false; }
        for (int j = 0; j < nw; j++) {
            if (P.progress_callback) P.progress_callback(ctx, COARSE, 100 * (step0 + j + 1) / cs.n_steps, P.progress_callback_user_data);
            cs.accept(w, j, tok[(size_t) j]);
        }
    }
    cs.store(g.coarse_tokens);
    end_stage(m, t_start, ctx->stats.n_sample_coarse, ctx->stats.t_coarse_us);
    return true;
}

// progress: call the progress callback (not during a batch)
bool run_fine(bark_context * ctx, Generation & g, bool progress = true) {
    const int64_t t_start = now_us();
    GPTModel & m = ctx->fine;
    const bark_context_params & P = ctx->params;
    const int n_coarse = P.n_coarse_codebooks, n_cb = P.n_fine_codebooks, cb_size = P.codebook_size;
    if (n_cb != 8 || n_coarse != 2 || cb_size != 1024) { fprintf(stderr, "%s: unsupported codebook configuration\n", __func__); return false; }
    const int T = (int) g.coarse_tokens.size() / 2;
    // history: the last H <= 512 frames of the prompt's fine codes come first (upstream Bark's generate_fine); H = 0 without a prompt
    const std::vector<int32_t> & F = g.prompt.fine;
    const int n_f = (int) F.size() / 8, H = std::min(n_f, 512);
    const int len = std::max(H + T, 1024);
    std::vector<int32_t> arr((size_t) len * 8, cb_size);                          // [len][8], padded with codebook_size (bark.cpp:1982-1996)
    for (int t = 0; t < H; t++) for (int c = 0; c < 8; c++) arr[(size_t) t * 8 + c] = F[(size_t) c * n_f + (n_f - H + t)];
    for (int t = 0; t < T; t++) { arr[(size_t)(H + t) * 8] = g.coarse_tokens[(size_t) t * 2]; arr[(size_t)(H + t) * 8 + 1] = g.coarse_tokens[(size_t) t * 2 + 1]; }
    const int n_loops = std::max(0, (int) ceilf((len - 1024) / 512.f)) + 1;      // = max(0, ceil((T - (1024 - H)) / 512)) + 1
    std::vector<int32_t> buf((size_t) 8 * 1024), sampled(1024);
    for (int n = 0; n < n_loops; n++) {
        const int start = std::min(n * 512, len - 1024), fill = std::min(H + n * 512, len - 512), rel = fill - start;
        for (int c = 0; c < 8; c++) for (int j = 0; j < 1024; j++) buf[(size_t) c * 1024 + j] = arr[(size_t)(start + j) * 8 + c];
        for (int nn = n_coarse; nn < n_cb; nn++) {
            if (progress && P.progress_callback) P.progress_callback(ctx, FINE, 100 * (n * (n_cb - n_coarse) + (nn - n_coarse + 1)) / (n_loops * (n_cb - n_coarse)), P.progress_callback_user_data);
            const bool ok = ctx->shard.on                     // rows of the window split over the GPUs of the job (shard.cu)
                ? fine_eval_shard(ctx, buf.data(), nn) && sample_shard(ctx, g.rng, cb_size, P.fine_temp, sampled.data())
                : fine_eval(ctx, buf.data(), nn, nullptr) && sample_device(ctx, m, g.rng, ctx->last_logits, m.n_out_vocab, cb_size, 1024, P.fine_temp, sampled.data(), nullptr);
            if (!ok) { fprintf(stderr, "%s: Could not generate token\n", __func__); return false; }
            // For unprompted clips <= 1024 frames (rel == 0) this is the reference's write (bark.cpp:2037).  For longer clips the
            // reference indexes buf[nn*1024 + rel + i] and runs off the buffer (SURVEY finding 5); there, and under a fine
            // history, we keep the original Bark semantics: every row is sampled (same RNG consumption) and rows >= rel are written in place.
            for (int i = rel; i < 1024; i++) buf[(size_t) nn * 1024 + i] = sampled[(size_t) i];
        }
        for (int nn = n_coarse; nn < n_cb; nn++) for (int j = 0; j < 1024 - rel; j++) arr[(size_t)(fill + j) * 8 + nn] = buf[(size_t) nn * 1024 + rel + j];
    }
    g.fine_tokens.assign(arr.begin() + (std::ptrdiff_t) H * 8, arr.begin() + (std::ptrdiff_t)(H + T) * 8);   // the generated frames
    end_stage(m, t_start, ctx->stats.n_sample_fine, ctx->stats.t_fine_us);
    return true;
}

// fine ids -> waveform (bark.cpp:2151-2159 + EnCodec) of n generations, decoded together by one batched codec_decode
bool decode_audio(bark_context * ctx, Generation * const * gens, int n) {
    if (ctx->params.target_bandwidth != 6 || ctx->params.sample_rate != 24000) {
        fprintf(stderr, "%s: only target_bandwidth 6 / 24 kHz is implemented\n", __func__); return false;
    }
    std::vector<std::vector<int32_t>> codes((size_t) n);
    std::vector<const int32_t *> ptrs((size_t) n);
    std::vector<int> T((size_t) n);
    for (int i = 0; i < n; i++) {
        // [T][8] -> [8][T]: EnCodec wants one contiguous time series per codebook
        const std::vector<int32_t> & fine = gens[i]->fine_tokens;
        const int Ti = (int) fine.size() / 8;
        std::vector<int32_t> & c = codes[(size_t) i];
        c.resize((size_t) 8 * Ti);
        for (int q = 0; q < 8; q++) for (int t = 0; t < Ti; t++) c[(size_t) q * Ti + t] = fine[(size_t) t * 8 + q];
        ptrs[(size_t) i] = c.data(); T[(size_t) i] = Ti;
    }
    std::vector<std::vector<float>> audio((size_t) n);
    if (!codec_decode(ctx->codec, ctx->codec_scratch, ctx->stream, n, ptrs.data(), T.data(), 8, audio.data(), n > 1 ? "bark_b200_generate_batch" : nullptr)) { printf("%s: Could not generate waveform from tokens with Encodec\n", __func__); return false; }
    for (int i = 0; i < n; i++) gens[i]->audio.swap(audio[(size_t) i]);
    return true;
}

// ---------------------------------------------------------------------------------------------
// batched generation (bark_b200_generate_batch)
//
// Up to 8 prompts share each semantic / coarse decode step: the step's rows go through the per-op kernels with rows = B, so
// every weight is read once per step for all of them (8 is the row tile of the few-row mat-mul kernels).  Each row's arithmetic
// is the single run's, so every item is bit-identical to its own single run: prefills, fine passes and the codec run per item.
// ---------------------------------------------------------------------------------------------
constexpr int kMaxBatch = 8;

// KV caches for `n` slots (semantic and coarse), the step's logits and id / position buffers.  Out of device memory: a message and
// false; the slots completed so far stay (bark_free frees them), a slot is only counted once all four of its slabs exist.
bool ensure_batch_slots(bark_context * ctx, int n) {
    BatchSlots & S = ctx->batch;
    auto fail = [&](const char * what) { (void) cudaGetLastError(); fprintf(stderr, "bark_b200: out of device memory for %s\n", what); return false; };
    if (!S.d_logits) {
        const size_t n_out = (size_t) std::max(ctx->semantic.n_out_vocab, ctx->coarse.n_out_vocab);
        float * l = nullptr; int32_t * d = nullptr, * h = nullptr;
        if (cudaMalloc(&l, kMaxBatch * n_out * 4) != cudaSuccess) return fail("the batch logits");
        if (cudaMalloc(&d, 16 * 4) != cudaSuccess) { cudaFree(l); return fail("the batch logits"); }
        if (cudaMallocHost(&h, 16 * 4) != cudaSuccess) { cudaFree(l); cudaFree(d); return fail("the batch logits"); }
        S.d_logits = l; S.d_step = d; S.h_step = h;
    }
    for (; S.cap < n; S.cap++) {
        float * slab[4] = {nullptr, nullptr, nullptr, nullptr};                   // semantic k, v, coarse k, v
        size_t bytes[4];
        for (int j = 0; j < 4; j++) {
            const GPTModel & m = j < 2 ? ctx->semantic : ctx->coarse;
            bytes[j] = (size_t) m.n_layer * m.block_size * m.n_embd * 4;
            if (cudaMalloc(&slab[j], bytes[j]) != cudaSuccess) {
                for (int q = 0; q < j; q++) cudaFree(slab[q]);
                return fail("a batch item's KV cache");
            }
        }
        for (int j = 0; j < 4; j++) BARK_CUDA_CHECK(cudaMemsetAsync(slab[j], 0, bytes[j], ctx->stream));
        S.k[0][S.cap] = slab[0]; S.v[0][S.cap] = slab[1]; S.k[1][S.cap] = slab[2]; S.v[1][S.cap] = slab[3];
    }
    return true;
}

struct BatchItem {
    Generation g;
    int n_past = 0;                                  // of the item's cache in the stage running
    CoarseStage coarse;
};

// Prefill of item b on its own cache (the existing kernels); its last-row logits become row `row` of the batch logits.
bool batch_prefill(bark_context * ctx, GPTModel & m, int which, BatchItem & it, int b, int row, const std::vector<int32_t> & in, bool merge, int lo, int hi) {
    BatchSlots & S = ctx->batch;
    if (!gpt_eval(ctx, m, in.data(), (int) in.size(), &it.n_past, merge, nullptr, lo, hi, S.k[which][b], S.v[which][b])) return false;
    BARK_CUDA_CHECK(cudaMemcpyAsync(S.d_logits + (size_t) row * m.n_out_vocab, ctx->last_logits, (size_t) m.n_out_vocab * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    BARK_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));        // gpt_eval stages the ids in one pinned buffer: the next prefill overwrites it
    return true;
}

// Samples row r of the batch logits (window [lo, lo + n)) for item act[r], with one uniform from that item's RNG, as run_chain draws
// it.  The one host synchronisation of the step; rows the device kernel flags are replayed on the host from the same logits and
// uniform.  tok[r] = lo + the sampled index, eos[r] = probability of the window's last logit.
bool batch_sample(bark_context * ctx, GPTModel & m, std::vector<BatchItem> & items, const std::vector<int> & act, int lo, int n, float temp,
                  const bark_b200_sampling & filt, int32_t * tok, float * eos) {
    const int64_t t0 = now_us();
    const int B = (int) act.size();
    if (n > kSampleMaxLogits) { fprintf(stderr, "%s: %d logits per row exceed the device sampler's row of %d\n", __func__, n, kSampleMaxLogits); return false; }
    if (temp != 0.0f) for (int r = 0; r < B; r++) ctx->h_u[r] = std::generate_canonical<double, 53>(items[(size_t) act[(size_t) r]].g.rng);
    sample_and_replay(ctx, ctx->batch.d_logits, m.n_out_vocab, lo, n, B, temp, true, &filt);
    for (int r = 0; r < B; r++) { tok[r] = ctx->h_stok[r]; eos[r] = ctx->h_seos[r]; }
    m.n_sample += B;
    m.t_sample_us += now_us() - t0;
    return true;
}

// The batched step of the rows act[r] with input ids tok[r]; advances their n_past.
bool batch_step(bark_context * ctx, GPTModel & m, int which, std::vector<BatchItem> & items, const std::vector<int> & act, const int32_t * tok, int lo, int hi) {
    float * sk[kMaxBatch], * sv[kMaxBatch]; int pos[kMaxBatch];
    for (size_t r = 0; r < act.size(); r++) { sk[r] = ctx->batch.k[which][act[r]]; sv[r] = ctx->batch.v[which][act[r]]; pos[r] = items[(size_t) act[r]].n_past; }
    if (!gpt_step_batch(ctx, m, (int) act.size(), sk, sv, tok, pos, lo, hi, ctx->batch.d_logits)) return false;
    for (int b : act) items[(size_t) b].n_past++;
    return true;
}

// semantic stage of every item (run_semantic's loop): an item leaves the step at its own stop or after n_steps_text_encoder ids
bool batch_semantic(bark_context * ctx, std::vector<BatchItem> & items) {
    GPTModel & m = ctx->semantic;
    const bark_context_params & P = ctx->params;
    std::vector<int> act;
    for (int b = 0; b < (int) items.size() && P.n_steps_text_encoder > 0; b++) {
        items[(size_t) b].n_past = 0;
        if (!batch_prefill(ctx, m, 0, items[(size_t) b], b, b, items[(size_t) b].g.tokens, true, 0, 0)) return false;
        act.push_back(b);
    }
    int32_t tok[kMaxBatch]; float eos[kMaxBatch];
    while (!act.empty()) {
        if (!batch_sample(ctx, m, items, act, 0, m.n_out_vocab, P.temp, ctx->sampling[0], tok, eos)) return false;     // all n_out logits (quirk D.1)
        std::vector<int> next; int32_t next_tok[kMaxBatch];
        for (size_t r = 0; r < act.size(); r++) {
            if (semantic_accept(P, items[(size_t) act[r]].g.semantic_tokens, tok[r], eos[r])) { next_tok[next.size()] = tok[r]; next.push_back(act[r]); }
        }
        act.swap(next);
        if (!act.empty() && !batch_step(ctx, m, 0, items, act, next_tok, 0, 0)) return false;
    }
    return true;
}

// coarse stage of every item (run_coarse): window w starts at step 60 w for every item, so the logit window alternates alike
bool batch_coarse(bark_context * ctx, std::vector<BatchItem> & items) {
    GPTModel & m = ctx->coarse;
    const bark_context_params & P = ctx->params;
    int n_windows = 0;
    for (BatchItem & it : items) {
        if (!it.coarse.setup(P, m, it.g, __func__)) return false;
        n_windows = std::max(n_windows, it.coarse.n_windows());
    }
    const CoarseStage & rule = items.front().coarse;          // window starts and codebook windows depend on the parameters alone
    int32_t tok[kMaxBatch]; float eos[kMaxBatch];
    for (int w = 0; w < n_windows; w++) {
        const int step0 = rule.first_step(w), lo0 = rule.lo(step0);
        std::vector<int> act;
        for (int b = 0; b < (int) items.size(); b++) {
            BatchItem & it = items[(size_t) b];
            if (w >= it.coarse.n_windows()) continue;
            const std::vector<int32_t> in_eval = it.coarse.window(ctx, w, &it.n_past);
            if (!batch_prefill(ctx, m, 1, it, b, (int) act.size(), in_eval, false, lo0, lo0 + P.codebook_size)) return false;
            act.push_back(b);
        }
        for (int j = 0; !act.empty(); j++) {
            const int lo = rule.lo(step0 + j);
            if (!batch_sample(ctx, m, items, act, lo, P.codebook_size, P.temp, ctx->sampling[1], tok, eos)) return false;
            std::vector<int> next; int32_t next_tok[kMaxBatch];
            for (size_t r = 0; r < act.size(); r++)
                if (items[(size_t) act[r]].coarse.accept(w, j, tok[r])) { next_tok[next.size()] = tok[r]; next.push_back(act[r]); }
            act.swap(next);
            const int lo_next = rule.lo(step0 + j + 1);
            if (!act.empty() && !batch_step(ctx, m, 1, items, act, next_tok, lo_next, lo_next + P.codebook_size)) return false;
        }
    }
    for (BatchItem & it : items) it.coarse.store(it.g.coarse_tokens);
    return true;
}

// What a batch must leave as it was: the models' counters (they belong to the context's own runs) always, the context's statistics
// unless the batch succeeds.  Restored on every way out, a thrown CUDA failure included.
struct BatchGuard {
    bark_context * ctx; bark_statistics stats; int64_t counters[3][4]; bool keep_stats = false;
    GPTModel * model(int i) const { return i == 0 ? &ctx->semantic : i == 1 ? &ctx->coarse : &ctx->fine; }
    explicit BatchGuard(bark_context * c) : ctx(c), stats(c->stats) {
        for (int i = 0; i < 3; i++) { const GPTModel & m = *model(i); counters[i][0] = m.n_sample; counters[i][1] = m.t_sample_us; counters[i][2] = m.t_predict_us; counters[i][3] = m.t_main_us; }
    }
    int32_t samples(int i) const { return (int32_t)(model(i)->n_sample - counters[i][0]); }
    ~BatchGuard() {
        for (int i = 0; i < 3; i++) { GPTModel & m = *model(i); m.n_sample = counters[i][0]; m.t_sample_us = counters[i][1]; m.t_predict_us = counters[i][2]; m.t_main_us = counters[i][3]; }
        if (!keep_stats) ctx->stats = stats;
    }
};

}  // namespace

// Validates a history prompt by upstream Bark's rules and copies it into h; false with a message on stderr (h untouched).  The
// alignment check is upstream's round(n_c / n_s, 1) == round(stc / n_coarse_codebooks, 1), stc = coarse_rate_hz / semantic_rate_hz *
// n_coarse_codebooks; for the default rates (75 / 49.9 Hz, 2 codebooks: 1.503 -> 1.5) it is the exact 29 n_s < 20 n_c < 31 n_s.
bool bark::make_history_prompt(const bark_context_params & P, const bark_b200_history_prompt & p, HistoryPrompt & h) {
    const char * fn = "bark_b200_set_history_prompt";
    const long long n_s = p.n_semantic, n_c = p.n_coarse_frames, n_f = p.n_fine_frames;
    if (n_s < 1 || !p.semantic) { fprintf(stderr, "%s: %lld semantic ids (at least 1)\n", fn, n_s); return false; }
    if (n_c < 1 || !p.coarse) { fprintf(stderr, "%s: %lld coarse frames (at least 1)\n", fn, n_c); return false; }
    if (n_f < 0 || (n_f > 0 && !p.fine)) { fprintf(stderr, "%s: %lld fine frames (0 or more)\n", fn, n_f); return false; }
    if (P.n_coarse_codebooks != 2 || P.n_fine_codebooks != 8) { fprintf(stderr, "%s: unsupported codebook configuration\n", fn); return false; }
    auto in_range = [](const int32_t * a, long long n, int hi, const char * what) {
        for (long long i = 0; i < n; i++)
            if (a[i] < 0 || a[i] >= hi) { fprintf(stderr, "bark_b200_set_history_prompt: %s id %d at %lld is outside [0, %d)\n", what, a[i], i, hi); return false; }
        return true;
    };
    if (!in_range(p.semantic, n_s, P.semantic_vocab_size, "semantic") || !in_range(p.coarse, 2 * n_c, P.codebook_size, "coarse") ||
        !in_range(p.fine, 8 * n_f, P.codebook_size, "fine")) return false;
    bool aligned;
    if (P.coarse_rate_hz == 75.0f && P.semantic_rate_hz == 49.9f) aligned = 29 * n_s < 20 * n_c && 20 * n_c < 31 * n_s;
    else {
        const double stc = (double)(P.coarse_rate_hz / P.semantic_rate_hz * P.n_coarse_codebooks);
        aligned = std::round(10.0 * n_c / n_s) == std::round(10.0 * stc / P.n_coarse_codebooks);
    }
    if (!aligned) { fprintf(stderr, "%s: %lld coarse frames do not align with %lld semantic ids (29 n_s < 20 n_c < 31 n_s)\n", fn, n_c, n_s); return false; }
    h.semantic.assign(p.semantic, p.semantic + n_s);
    h.coarse.assign(p.coarse, p.coarse + 2 * n_c);
    h.fine.assign(p.fine, p.fine + 8 * n_f);
    return true;
}

namespace {

// A failed batch changes nothing a caller can read: bark_b200_batch_* still return the last successful batch.  prompts (may be null,
// and so may any entry): item i's history prompt.
bool generate_batch(bark_context * ctx, const char * const * texts, const uint32_t * seeds, const bark_b200_history_prompt * const * prompts, int n) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return false; }
    if (n < 1 || n > kMaxBatch) { fprintf(stderr, "%s: %d prompts (1 to %d per batch)\n", __func__, n, kMaxBatch); return false; }
    if (!texts || !seeds) { fprintf(stderr, "%s: null prompts or seeds\n", __func__); return false; }
    for (int i = 0; i < n; i++) if (!texts[i]) { fprintf(stderr, "%s: prompt %d is null\n", __func__, i); return false; }
    if (ctx->shard.on) { fprintf(stderr, "%s: not available on a context whose fine stage is sharded over GPUs\n", __func__); return false; }
    std::vector<BatchItem> items((size_t) n);
    for (int i = 0; i < n; i++)
        if (prompts && prompts[i] && !make_history_prompt(ctx->params, *prompts[i], items[(size_t) i].g.prompt)) {
            fprintf(stderr, "%s: history prompt %d rejected\n", __func__, i); return false;
        }
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (!ensure_batch_slots(ctx, n)) return false;
    BatchGuard guard(ctx);
    bark_statistics st{};
    st.t_load_us = ctx->stats.t_load_us;
    const int64_t t0 = now_us();
    for (int i = 0; i < n; i++) {
        items[(size_t) i].g.rng = std::mt19937(seeds[i]);
        if (!tokenize_input(ctx, items[(size_t) i].g, texts[i], "bark_b200_generate_batch")) { fprintf(stderr, "%s: text %d refused\n", __func__, i); return false; }
    }
    bool ok = batch_semantic(ctx, items);
    const int64_t t1 = now_us();
    ok = ok && batch_coarse(ctx, items);
    const int64_t t2 = now_us();
    st.n_sample_semantic = guard.samples(0);
    st.n_sample_coarse = guard.samples(1);
    int64_t t_fine = 0;
    std::vector<Generation *> gens;
    for (int i = 0; ok && i < n; i++) {
        const int64_t tf = now_us();
        ok = run_fine(ctx, items[(size_t) i].g, false);
        t_fine += now_us() - tf;
        gens.push_back(&items[(size_t) i].g);
    }
    ok = ok && decode_audio(ctx, gens.data(), n);
    st.n_sample_fine = guard.samples(2);
    if (!ok) return false;
    st.t_semantic_us = t1 - t0; st.t_coarse_us = t2 - t1; st.t_fine_us = t_fine; st.t_eval_us = now_us() - t0;
    ctx->stats = st; guard.keep_stats = true;
    ctx->batch.results.clear();
    for (BatchItem & it : items) ctx->batch.results.push_back(std::move(it.g));
    return true;
}

void alloc_workspace(bark_context * ctx) {
    int E = 0, H = 0, max_block = 0; size_t kp_bytes = 0, n_logits = 0;
    for (GPTModel * m : {&ctx->semantic, &ctx->coarse, &ctx->fine}) {
        E = std::max(E, (int) m->n_embd); H = std::max(H, (int) m->n_head); max_block = std::max(max_block, (int) m->block_size);
        const size_t es = m->wtype == W_F16 ? 2 : 4;
        kp_bytes = std::max(kp_bytes, (size_t) li_padded_k(4 * m->n_embd, (int) es) * es);
    }
    n_logits = std::max<size_t>({(size_t) ctx->semantic.n_out_vocab, (size_t) ctx->coarse.n_out_vocab, (size_t) 1024 * ctx->fine.n_out_vocab});
    Workspace & ws = ctx->ws;
    const size_t R = 1024;
    ws.max_rows = (int) R; ws.E = E;
    ws.x    = (float *) ctx_alloc(ctx, R * E * 4);
    ws.act  = ctx_alloc(ctx, R * kp_bytes);
    ws.act2 = ctx_alloc(ctx, R * kp_bytes);
    ws.q    = (float *) ctx_alloc(ctx, R * E * 4);
    ws.kbuf = (float *) ctx_alloc(ctx, R * E * 4);
    ws.vbuf = (float *) ctx_alloc(ctx, R * E * 4);
    // scores of the batched decode step (<= 8 rows x H heads x max_kv) and of the three-kernel attention for few rows (gpt_kernels.h)
    ws.scores = (float *) ctx_alloc(ctx, std::max((size_t) 8 * max_block, (size_t) attn_tiled_max_rows(H, ctx->n_sm_total) * 1024) * H * 4);
    ws.logits = (float *) ctx_alloc(ctx, n_logits * 4);
    ws.tok  = (int32_t *) ctx_alloc(ctx, 8 * 1024 * 4);
    if (is_quant(ctx->semantic.wtype) || is_quant(ctx->coarse.wtype) || is_quant(ctx->fine.wtype)) {
        ctx->q8.q = (int8_t *) ctx_alloc(ctx, R * (size_t) 4 * E); ctx->q8.d = (float *) ctx_alloc(ctx, R * (size_t)(4 * E / 32) * 4);
        ctx->q8.s = (float *) ctx_alloc(ctx, R * (size_t)(4 * E / 32) * 4);
    }
    if (ctx->fast_mode) {
        const GPTModel & fm = ctx->fine;
        if (fm.n_embd / fm.n_head != 64 || fm.n_embd % 64 != 0 || fm.n_embd > 1024) {
            fprintf(stderr, "bark_b200: BARK_B200_MODE=fast needs a fine model with 64-wide heads; using the parity path\n");
            ctx->fast_mode = false;
        } else {
            const size_t FE = (size_t) fm.n_embd;
            ctx->f_a16 = (__half *) ctx_alloc(ctx, R * FE * 2); ctx->f_h16 = (__half *) ctx_alloc(ctx, R * 4 * FE * 2);
            ctx->f_qk16 = (__half *) ctx_alloc(ctx, R * 2 * FE * 2); ctx->f_vt16 = (__half *) ctx_alloc(ctx, FE * R * 2); ctx->f_att16 = (__half *) ctx_alloc(ctx, R * FE * 2);
        }
    }
    BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_logits, n_logits * 4));
    BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_tok, 8 * 1024 * 4));
    ctx->d_u = (double *) ctx_alloc(ctx, 1024 * 8); ctx->d_stok = (int32_t *) ctx_alloc(ctx, 1024 * 4);
    ctx->d_sflags = (int32_t *) ctx_alloc(ctx, 1024 * 4); ctx->d_seos = (float *) ctx_alloc(ctx, 1024 * 4);
    ctx->d_feed = (int32_t *) ctx_alloc(ctx, 64); BARK_CUDA_CHECK(cudaMemset(ctx->d_feed, 0, 64));
    ctx->d_frow = (float *) ctx_alloc(ctx, (size_t) kMaxFilterRows * kSampleMaxLogits * 4); ctx->d_fflags = (int32_t *) ctx_alloc(ctx, 1024 * 4);
    BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_fflags, 1024 * 4));
    BARK_CUDA_CHECK(cudaMemset(ctx->d_u, 0, 1024 * 8));
    BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_u, 1024 * 8)); BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_stok, 1024 * 4));
    BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_sflags, 1024 * 4)); BARK_CUDA_CHECK(cudaMallocHost(&ctx->h_seos, 1024 * 4));
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// ggml.h shim
// ---------------------------------------------------------------------------------------------
extern "C" struct ggml_context * ggml_init(struct ggml_init_params) { static int token; return reinterpret_cast<struct ggml_context *>(&token); }   // nothing to initialise: f16 conversions are hardware instructions here
extern "C" void    ggml_free(struct ggml_context *) {}
extern "C" void    ggml_time_init(void) {}
extern "C" int64_t ggml_time_us(void) { return now_us(); }
extern "C" int64_t ggml_time_ms(void) { return now_us() / 1000; }

// ---------------------------------------------------------------------------------------------
// bark.h
// ---------------------------------------------------------------------------------------------
extern "C" struct bark_context_params bark_context_default_params(void) {
    bark_context_params p;
    memset(&p, 0, sizeof(p));
    p.verbosity = LOW;
    p.temp = 0.7f; p.fine_temp = 0.5f; p.min_eos_p = 0.2f;
    p.sliding_window_size = 60; p.max_coarse_history = 630;
    p.sample_rate = 24000; p.target_bandwidth = 6;
    p.cls_token_id = 101; p.sep_token_id = 102;
    p.n_steps_text_encoder = 768;
    p.text_pad_token = 129595; p.text_encoding_offset = 10048;
    p.semantic_rate_hz = 49.9f; p.semantic_pad_token = 10000; p.semantic_vocab_size = 10000; p.semantic_infer_token = 129599;
    p.coarse_rate_hz = 75.0f; p.coarse_infer_token = 12050; p.coarse_semantic_pad_token = 12048;
    p.n_coarse_codebooks = 2; p.n_fine_codebooks = 8; p.codebook_size = 1024;
    p.progress_callback = nullptr; p.progress_callback_user_data = nullptr;
    return p;
}

extern "C" void bark_b200_set_device(int device) { g_device_override = device; }

int bark::select_device(const char * caller, cudaDeviceProp * prop) {
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        fprintf(stderr, "%s: no CUDA device available — this library has no CPU path\n", caller);
        return -1;
    }
    int dev = g_device_override;
    if (dev < 0) { const char * e = getenv("BARK_B200_DEVICE"); dev = e ? atoi(e) : 0; }
    if (dev < 0 || dev >= n_dev) { fprintf(stderr, "%s: CUDA device %d out of range (%d present)\n", caller, dev, n_dev); return -1; }
    if (cudaSetDevice(dev) != cudaSuccess || cudaGetDeviceProperties(prop, dev) != cudaSuccess) { fprintf(stderr, "%s: cannot use CUDA device %d: %s\n", caller, dev, cudaGetErrorString(cudaGetLastError())); return -1; }
    if (prop->major != 9 || prop->minor != 0) {
        fprintf(stderr, "%s: device %d is sm_%d%d; this library is built for sm_90a (H100) only\n", caller, dev, prop->major, prop->minor);
        return -1;
    }
    return dev;
}

extern "C" struct bark_context * bark_load_model(const char * model_path, struct bark_context_params params, uint32_t seed) {
    const int64_t t0 = now_us();
    if (!model_path) { fprintf(stderr, "%s: null model path\n", __func__); return nullptr; }
    int tokenizer = BARK_B200_TOKENIZER_REFERENCE;            // BARK_B200_TOKENIZER: the context's initial tokenizer (include/bark_b200.h)
    if (const char * e = getenv("BARK_B200_TOKENIZER"); e && *e) {
        if (!strcmp(e, "bert")) tokenizer = BARK_B200_TOKENIZER_BERT;
        else if (strcmp(e, "reference")) { fprintf(stderr, "%s: BARK_B200_TOKENIZER=%s is neither 'reference' nor 'bert'\n", __func__, e); return nullptr; }
    }
    int long_form = -1;                                       // BARK_B200_LONG_FORM: long form on with this voice and the defaults (-1: off)
    if (const char * e = getenv("BARK_B200_LONG_FORM"); e && *e && strcmp(e, "off")) {
        if (!strcmp(e, "chain")) long_form = BARK_B200_VOICE_CHAIN;
        else if (!strcmp(e, "fixed")) long_form = BARK_B200_VOICE_FIXED;
        else { fprintf(stderr, "%s: BARK_B200_LONG_FORM=%s is none of 'chain', 'fixed', 'off'\n", __func__, e); return nullptr; }
    }
    cudaDeviceProp prop;
    const int dev = select_device(__func__, &prop);
    if (dev < 0) return nullptr;
    bark_context * ctx = new bark_context();
    ctx->device = dev;
    ctx->tokenizer = tokenizer;
    ctx->long_form.on = long_form >= 0;
    if (long_form >= 0) ctx->long_form.settings.voice = long_form;
    ctx->n_sm = ctx->n_sm_total = prop.multiProcessorCount;
    if (ctx->n_sm >= 132) ctx->n_sm = 128;                    // CTAs of the persistent decode step: a power of two below the SM count (fewer pollers per exchange)
    { const char * e = getenv("BARK_B200_MODE"); ctx->fast_mode = e && !strcmp(e, "fast"); }             // "fast": tensor-core fine passes (fast_kernels.cu), not bit-identical
    { const char * e = getenv("BARK_B200_DECODE_CTAS"); if (e && atoi(e) >= 64 && atoi(e) <= ctx->n_sm) ctx->n_sm = atoi(e); }   // experiment knob: CTAs of the persistent decode kernel
    { const char * e = getenv("BARK_B200_SAMPLE_FLAG_EVERY"); ctx->debug_flag_every = e ? atoi(e) : 0; }
    { const char * e = getenv("BARK_B200_KV_REUSE"); ctx->kv_reuse = !(e && !strcmp(e, "0")); }              // "0": re-prefill every coarse window like the reference (A-B)
    { const char * e = getenv("BARK_B200_DECODE"); ctx->use_decode_kernel = !(e && !strcmp(e, "multi")); }   // "multi": one kernel per op (debug / A-B)
    { const char * e = getenv("BARK_B200_DECODE_TIMING_TID"); if (e && atoi(e) >= 0 && atoi(e) < 512) ctx->timing_tid = atoi(e) & ~31; }
    { const char * e = getenv("BARK_B200_POLL_NS"); if (e && atoi(e) >= 0 && atoi(e) <= 100000) ctx->poll_ns = (unsigned) atoi(e); }
    { const char * e = getenv("BARK_B200_HEADSTART"); if (e) { unsigned v[6]; if (sscanf(e, "%u:%u:%u:%u:%u:%u", &v[0], &v[1], &v[2], &v[3], &v[4], &v[5]) == 6) for (int i = 0; i < 6; i++) ctx->headstart[i] = std::min(v[i], 100000u); } }
    ctx->params = params;
    const bool loaded = guarded(false, [&] {                  // a CUDA failure while loading (out of memory, ...) is a failed load, not an abort
    BARK_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    if (!load_model_file(model_path, ctx)) return false;
    alloc_workspace(ctx);
    { const char * e = getenv("BARK_B200_TAG_BASE"); if (e) ctx->tag_base = (unsigned) strtoul(e, nullptr, 0); }      // tests: start the exchange epochs near the 32-bit wrap
    if (getenv("BARK_B200_DECODE_TIMING")) { ctx->d_timing = (unsigned long long *) ctx_alloc(ctx, 256 * 32 * 8); BARK_CUDA_CHECK(cudaMemset(ctx->d_timing, 0, 256 * 32 * 8)); }
    BARK_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return true;
    });
    if (!loaded) {
        fprintf(stderr, "%s: failed to load model weights from '%s'\n", __func__, model_path);
        bark_free(ctx);
        return nullptr;
    }
    ctx->gen.rng = std::mt19937(seed);
    ctx->stats.t_load_us = now_us() - t0;
    return ctx;
}

extern "C" void bark_reset_statistics(struct bark_context * ctx) {
    if (!ctx) return;
    const int64_t load = ctx->stats.t_load_us;
    memset(&ctx->stats, 0, sizeof(ctx->stats));
    ctx->stats.t_load_us = load;          // the reference zeroes the whole struct (bark.cpp:2403-2407) and so reports load time 0 after
                                          // the first generate; keeping it is the useful reading of "load time of the model"
}

extern "C" bool bark_b200_forward_text_encoder(struct bark_context * ctx, int) { return guarded(false, [&] { return ctx && run_semantic(ctx, ctx->gen); }); }
extern "C" bool bark_b200_forward_coarse_encoder(struct bark_context * ctx, int) { return guarded(false, [&] { return ctx && run_coarse(ctx, ctx->gen); }); }
extern "C" bool bark_b200_forward_fine_encoder(struct bark_context * ctx, int) { return guarded(false, [&] { return ctx && run_fine(ctx, ctx->gen); }); }
// the reference also exports these three as C++ symbols without a header (bark.cpp:1703,1865,2061)
BARK_API bool bark_forward_text_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_text_encoder(ctx, n); }
BARK_API bool bark_forward_coarse_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_coarse_encoder(ctx, n); }
BARK_API bool bark_forward_fine_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_fine_encoder(ctx, n); }

bool bark::generate_one(bark_context * ctx, const std::string & text) {
    const char * fn = "bark_generate_audio_impl";
    const int64_t t0 = now_us();
    Generation & g = ctx->gen;
    if (!tokenize_input(ctx, g, text, "bark_generate_audio")) return false;      // a refused text changes nothing
    bark_reset_statistics(ctx);
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (!run_semantic(ctx, g)) { fprintf(stderr, "%s: failed to forward text encoder\n", fn); return false; }
    if (!run_coarse(ctx, g))   { fprintf(stderr, "%s: failed to forward coarse encoder\n", fn); return false; }
    if (!run_fine(ctx, g))     { fprintf(stderr, "%s: failed to forward fine encoder\n", fn); return false; }
    Generation * gp = &g;
    if (!decode_audio(ctx, &gp, 1)) return false;
    ctx->stats.t_eval_us = now_us() - t0;
    return true;
}

static bool bark_generate_audio_impl(struct bark_context * ctx, const char * text, int n_threads) {
    (void) n_threads;                      // CPU thread count of the reference's backend; nothing to size here
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return false; }
    if (!text) { fprintf(stderr, "%s: null prompt\n", __func__); return false; }
    if (ctx->long_form.on) return generate_long(ctx, text);
    if (!generate_one(ctx, text)) return false;
    ctx->long_form.chunks.clear();         // the chunk getters describe the last generation only
    return true;
}
extern "C" bool bark_generate_audio(struct bark_context * ctx, const char * text, int n_threads) { return guarded((bool) false, [&] { return bark_generate_audio_impl(ctx, text, n_threads); }); }

extern "C" float * bark_get_audio_data(struct bark_context * ctx) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return nullptr; }
    return ctx->gen.audio.empty() ? nullptr : ctx->gen.audio.data();
}
extern "C" int bark_get_audio_data_size(struct bark_context * ctx) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return 0; }
    return (int) ctx->gen.audio.size();
}
extern "C" int64_t bark_get_load_time(struct bark_context * ctx) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return 0; }
    return ctx->stats.t_load_us;
}
extern "C" int64_t bark_get_eval_time(struct bark_context * ctx) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", __func__); return 0; }
    return ctx->stats.t_eval_us;
}

extern "C" void bark_free(struct bark_context * ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    ctx->arena.release();
    for (int p = 0; p < ctx->shard.world; p++) if (p != ctx->shard.rank && ctx->shard.peer[p]) cudaIpcCloseMemHandle(ctx->shard.peer[p]);
    if (ctx->shard.local) cudaFree(ctx->shard.local);
    ctx->codec_scratch.release();
    if (ctx->h_logits) cudaFreeHost(ctx->h_logits);
    if (ctx->h_tok) cudaFreeHost(ctx->h_tok);
    if (ctx->h_u) cudaFreeHost(ctx->h_u);
    if (ctx->h_stok) cudaFreeHost(ctx->h_stok);
    if (ctx->h_sflags) cudaFreeHost(ctx->h_sflags);
    if (ctx->h_seos) cudaFreeHost(ctx->h_seos);
    if (ctx->h_fflags) cudaFreeHost(ctx->h_fflags);
    for (int w = 0; w < 2; w++) for (int b = 0; b < ctx->batch.cap; b++) { cudaFree(ctx->batch.k[w][b]); cudaFree(ctx->batch.v[w][b]); }
    if (ctx->batch.d_logits) cudaFree(ctx->batch.d_logits);
    if (ctx->batch.d_step) cudaFree(ctx->batch.d_step);
    if (ctx->batch.h_step) cudaFreeHost(ctx->batch.h_step);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

// ---------------------------------------------------------------------------------------------
// additive entry points (include/bark_b200.h): per-call hooks for parity tests and the benchmark
// ---------------------------------------------------------------------------------------------
static GPTModel * pick(bark_context * ctx, int which) { return which == 0 ? &ctx->semantic : which == 1 ? &ctx->coarse : which == 2 ? &ctx->fine : nullptr; }

static int bark_b200_gpt_eval_impl(struct bark_context * ctx, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) {
    if (!ctx || which < 0 || which > 1 || !tokens || !logits_out) return 0;
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    return gpt_eval(ctx, *pick(ctx, which), tokens, n, n_past, merge_ctx != 0, logits_out) ? 1 : 0;
}
extern "C" int bark_b200_gpt_eval(struct bark_context * ctx, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) { return guarded((int) 0, [&] { return bark_b200_gpt_eval_impl(ctx, which, tokens, n, n_past, merge_ctx, logits_out); }); }
static int bark_b200_fine_eval_impl(struct bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_out) {
    if (!ctx || !in_buffer || !logits_out) return 0;
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    return fine_eval(ctx, in_buffer, nn, logits_out) ? 1 : 0;
}
extern "C" int bark_b200_fine_eval(struct bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_out) { return guarded((int) 0, [&] { return bark_b200_fine_eval_impl(ctx, in_buffer, nn, logits_out); }); }
static int bark_b200_encodec_decode_impl(struct bark_context * ctx, const int32_t * codes, int n_frames, float * out, int out_cap) {
    if (!ctx || !codes) return -1;
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (!codec_decode(ctx->codec, ctx->codec_scratch, ctx->stream, 1, &codes, &n_frames, 8, &ctx->gen.audio)) return -1;
    const int n = (int) ctx->gen.audio.size();
    if (out) memcpy(out, ctx->gen.audio.data(), sizeof(float) * (size_t) std::min(n, out_cap));
    return n;
}
extern "C" int bark_b200_encodec_decode(struct bark_context * ctx, const int32_t * codes, int n_frames, float * out, int out_cap) { return guarded((int) -1, [&] { return bark_b200_encodec_decode_impl(ctx, codes, n_frames, out, out_cap); }); }
static int bark_b200_encodec_encode_impl(struct bark_context * ctx, const float * audio, int n_samples, int32_t * codes, int codes_cap, float * latent,
                                         int latent_cap, const AudioFormat * fmt = nullptr) {
    const char * fn = fmt ? "bark_b200_encodec_encode_resampled" : "bark_b200_encodec_encode";
    if (!ctx || !audio) { fprintf(stderr, "%s: null %s\n", fn, ctx ? "audio" : "context"); return -1; }
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    std::vector<int32_t> c; std::vector<float> l;
    if (!codec_encode(ctx->codec, ctx->codec_scratch, ctx->stream, 1, &audio, &n_samples, 8, {&c, &l}, nullptr, fmt)) return -1;
    if (codes) memcpy(codes, c.data(), sizeof(int32_t) * std::min(c.size(), (size_t) std::max(codes_cap, 0)));
    if (latent) memcpy(latent, l.data(), sizeof(float) * std::min(l.size(), (size_t) std::max(latent_cap, 0)));
    return (int)(c.size() / 8);
}
extern "C" int bark_b200_encodec_encode(struct bark_context * ctx, const float * audio, int n_samples, int32_t * codes, int codes_cap, float * latent,
                                        int latent_cap) {
    return guarded((int) -1, [&] { return bark_b200_encodec_encode_impl(ctx, audio, n_samples, codes, codes_cap, latent, latent_cap); });
}
extern "C" int bark_b200_encodec_encode_resampled(struct bark_context * ctx, const float * audio, int n_frames, int channels, int sample_rate, int32_t * codes,
                                                  int codes_cap, float * latent, int latent_cap) {
    const AudioFormat f{channels, sample_rate};
    return guarded((int) -1, [&] { return bark_b200_encodec_encode_impl(ctx, audio, n_frames, codes, codes_cap, latent, latent_cap, &f); });
}
extern "C" int bark_b200_sample(struct bark_context * ctx, int which, const float * logits, int n, float temp, float * eos_p) {
    if (!ctx || !logits || n < 1) return -1;
    GPTModel & m = *pick(ctx, which < 0 || which > 2 ? 0 : which);
    const int64_t t0 = now_us();
    // what libstdc++'s discrete distribution takes: one draw, none on the argmax path or for a single logit
    const double u = temp != 0.0f && n > 1 ? std::generate_canonical<double, 53>(ctx->gen.rng) : 0.0;
    const int32_t next = sample_token_given_u(logits, n, temp, u, eos_p);
    m.t_sample_us += now_us() - t0;
    m.n_sample += 1;
    return next;
}
static int bark_b200_sample_rows_impl(struct bark_context * ctx, const float * logits, int n, int rows, float temp, int32_t * tokens_out, float * eos_p_out) {
    if (!ctx || !logits || !tokens_out || rows < 1 || rows > 1024 || n < 2 || n > kSampleMaxLogits) return -1;
    const size_t cap = std::max<size_t>({(size_t) ctx->semantic.n_out_vocab, (size_t) ctx->coarse.n_out_vocab, (size_t) 1024 * ctx->fine.n_out_vocab});
    if ((size_t) rows * n > cap) return -1;
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->ws.logits, logits, (size_t) rows * n * 4, cudaMemcpyHostToDevice, ctx->stream));
    const long long before = ctx->n_sample_host_replays;
    if (!sample_device(ctx, ctx->fine, ctx->gen.rng, ctx->ws.logits, n, n, rows, temp, tokens_out, eos_p_out)) return -1;
    return (int)(ctx->n_sample_host_replays - before);
}
extern "C" int bark_b200_sample_rows(struct bark_context * ctx, const float * logits, int n, int rows, float temp, int32_t * tokens_out, float * eos_p_out) { return guarded((int) -1, [&] { return bark_b200_sample_rows_impl(ctx, logits, n, rows, temp, tokens_out, eos_p_out); }); }
extern "C" void bark_b200_reseed(struct bark_context * ctx, uint32_t seed) { if (ctx) ctx->gen.rng = std::mt19937(seed); }
extern "C" void bark_b200_tokenize(struct bark_context * ctx, const char * text, int32_t * out513) {
    if (!ctx || !text || !out513) return;
    if (!tokenize_input(ctx, ctx->gen, text, "bark_b200_tokenize")) return;
    memcpy(out513, ctx->gen.tokens.data(), sizeof(int32_t) * 513);
}
template <class G>       // a Generation or a LongFormChunk
static int copy_tokens(const G & g, int stage, int32_t * out, int cap) {
    const std::vector<int32_t> * v = stage == 0 ? &g.semantic_tokens : stage == 1 ? &g.coarse_tokens : stage == 2 ? &g.fine_tokens : stage == 3 ? &g.tokens : nullptr;
    if (!v) return -1;
    if (out) memcpy(out, v->data(), sizeof(int32_t) * std::min(v->size(), (size_t) std::max(cap, 0)));
    return (int) v->size();
}
extern "C" int bark_b200_get_tokens(struct bark_context * ctx, int stage, int32_t * out, int cap) { return ctx ? copy_tokens(ctx->gen, stage, out, cap) : -1; }
extern "C" void bark_b200_set_tokens(struct bark_context * ctx, int stage, const int32_t * in, int n) {
    if (!ctx || !in || n < 0) return;
    Generation & g = ctx->gen;
    if (stage == 0) g.semantic_tokens.assign(in, in + n); else if (stage == 1) g.coarse_tokens.assign(in, in + n); else if (stage == 3) g.tokens.assign(in, in + n);
}
extern "C" void bark_b200_get_stats(struct bark_context * ctx, struct bark_statistics * out, int64_t * per_model9) {
    if (!ctx) return;
    if (out) *out = ctx->stats;
    if (per_model9) { const GPTModel * m[3] = {&ctx->semantic, &ctx->coarse, &ctx->fine}; for (int i = 0; i < 3; i++) { per_model9[3 * i] = m[i]->t_predict_us; per_model9[3 * i + 1] = m[i]->t_sample_us; per_model9[3 * i + 2] = m[i]->n_sample; } }
}
extern "C" void bark_b200_get_hparams(struct bark_context * ctx, int which, int32_t * out10) {
    if (!ctx || !out10) return;
    const GPTModel * m = pick(ctx, which); if (!m) return;
    const int32_t v[10] = {m->n_layer, m->n_head, m->n_embd, m->block_size, m->bias, m->n_in_vocab, m->n_out_vocab, m->n_lm_heads, m->n_wtes, m->ftype};
    memcpy(out10, v, sizeof(v));
}
extern "C" unsigned long long bark_b200_kernel_launches(void) { return g_kernel_launches.load(); }
static unsigned bark_b200_layernorm_fallbacks_impl(struct bark_context * ctx) {
    if (!ctx) return 0;
    unsigned v = 0; BARK_CUDA_CHECK(cudaMemcpy(&v, ctx->d_ln_fallbacks, sizeof(v), cudaMemcpyDeviceToHost)); return v;
}
extern "C" unsigned bark_b200_layernorm_fallbacks(struct bark_context * ctx) { return guarded((unsigned) 0, [&] { return bark_b200_layernorm_fallbacks_impl(ctx); }); }
static int bark_b200_decode_timing_impl(struct bark_context * ctx, unsigned long long * out, int n) {
    if (!ctx || !ctx->d_timing || !out) return 0;
    BARK_CUDA_CHECK(cudaMemcpy(out, ctx->d_timing, sizeof(unsigned long long) * (size_t) std::min(n, 256 * 32), cudaMemcpyDeviceToHost));
    return std::min(n, 256 * 32);
}
extern "C" int bark_b200_decode_timing(struct bark_context * ctx, unsigned long long * out, int n) { return guarded((int) 0, [&] { return bark_b200_decode_timing_impl(ctx, out, n); }); }
extern "C" int bark_b200_fast_mode(struct bark_context * ctx) { return ctx && ctx->fast_mode ? 1 : 0; }

extern "C" int bark_b200_set_sampling(struct bark_context * ctx, int stage, const struct bark_b200_sampling * s) {
    const char * fn = "bark_b200_set_sampling";
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", fn); return 0; }
    if (stage != 0 && stage != 1) { fprintf(stderr, "%s: stage %d (0 semantic, 1 coarse; the fine stage has no filter)\n", fn, stage); return 0; }
    if (s && !sampling_valid(fn, *s)) return 0;
    ctx->sampling[stage] = s ? *s : bark_b200_sampling{0, 0, 1.0f};
    return 1;
}

// text tokenizers (include/bark_b200.h)
extern "C" int bark_b200_set_tokenizer(struct bark_context * ctx, int kind) {
    const char * fn = "bark_b200_set_tokenizer";
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", fn); return 0; }
    if (kind != BARK_B200_TOKENIZER_REFERENCE && kind != BARK_B200_TOKENIZER_BERT) { fprintf(stderr, "%s: unknown tokenizer %d (0 reference, 1 bert)\n", fn, kind); return 0; }
    ctx->tokenizer = kind;
    return 1;
}
static int copy_ids(const std::vector<int32_t> & ids, int32_t * out, int cap) {
    if (out) memcpy(out, ids.data(), sizeof(int32_t) * std::min(ids.size(), (size_t) std::max(cap, 0)));
    return (int) ids.size();
}
// The uncapped ids of text under kind; false with a message naming fn for a text the tokenizer refuses or an unknown kind.  warn: the
// reference tokenizer's message for a character it skips.
static bool text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, std::vector<int32_t> & ids, const char * fn,
                     bool warn) {
    if (kind == BARK_B200_TOKENIZER_REFERENCE) { wordpiece(vocab, text, ids, INT_MAX, warn); return true; }
    if (kind == BARK_B200_TOKENIZER_BERT) return bert_tokenize(vocab, text, ids, fn);
    fprintf(stderr, "%s: unknown tokenizer %d (0 reference, 1 bert)\n", fn, kind);
    return false;
}
int bark::count_text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, const char * fn) {
    std::vector<int32_t> ids;
    return text_ids(vocab, kind, text, ids, fn, false) ? (int) ids.size() : -1;
}
extern "C" int bark_b200_text_ids(struct bark_context * ctx, int kind, const char * text, int32_t * out, int cap) {
    const char * fn = "bark_b200_text_ids";
    if (!ctx || !text) { fprintf(stderr, "%s: null %s\n", fn, ctx ? "text" : "context"); return -1; }
    return guarded((int) -1, [&] {
        std::vector<int32_t> ids;
        if (!text_ids(ctx->token_to_id, kind, text, ids, fn, true)) return -1;
        return copy_ids(ids, out, cap);
    });
}
// vocab[0..n) as the loader's token_to_id holds a file's vocabulary (id = index, later duplicates win); false with a message for a null entry
static bool vocab_map(const char * const * vocab, int n, std::map<std::string, int32_t> & v, const char * fn) {
    for (int i = 0; i < n; i++) {
        if (!vocab[i]) { fprintf(stderr, "%s: vocabulary entry %d is null\n", fn, i); return false; }
        v[vocab[i]] = i;
    }
    return true;
}
extern "C" int bark_b200_bert_tokenize(const char * const * vocab, int n_vocab, const char * text, int32_t * out, int cap) {
    const char * fn = "bark_b200_bert_tokenize";
    if (!vocab || n_vocab < 0 || !text) { fprintf(stderr, "%s: null vocabulary or text\n", fn); return -1; }
    return guarded((int) -1, [&] {
        std::map<std::string, int32_t> v;
        if (!vocab_map(vocab, n_vocab, v, fn)) return -1;
        std::vector<int32_t> ids;
        if (!bert_tokenize(v, text, ids, fn)) return -1;
        return copy_ids(ids, out, cap);
    });
}

// long-form generation (include/bark_b200.h, long_form.cu)
extern "C" int bark_b200_set_long_form(struct bark_context * ctx, const struct bark_b200_long_form * lf) {
    const char * fn = "bark_b200_set_long_form";
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", fn); return 0; }
    if (!lf) { ctx->long_form.on = false; return 1; }
    if (lf->voice != BARK_B200_VOICE_CHAIN && lf->voice != BARK_B200_VOICE_FIXED) { fprintf(stderr, "%s: unknown voice %d (0 chain, 1 fixed)\n", fn, lf->voice); return 0; }
    if (lf->max_chunk_ids < 1 || lf->max_chunk_ids > 255) { fprintf(stderr, "%s: max_chunk_ids %d (1 to 255)\n", fn, lf->max_chunk_ids); return 0; }
    if (lf->gap_samples < 0 || lf->gap_samples > 240000) { fprintf(stderr, "%s: gap_samples %d (0 to 240000)\n", fn, lf->gap_samples); return 0; }
    ctx->long_form.settings = *lf;
    ctx->long_form.on = true;
    return 1;
}
extern "C" int bark_b200_long_chunks(struct bark_context * ctx) { return ctx ? (int) ctx->long_form.chunks.size() : -1; }
extern "C" int bark_b200_long_chunk_text(struct bark_context * ctx, int k, char * out, int cap) {
    if (!ctx || k < 0 || k >= (int) ctx->long_form.chunks.size()) return -1;
    const std::string & t = ctx->long_form.chunks[(size_t) k].text;
    if (out) memcpy(out, t.data(), std::min(t.size(), (size_t) std::max(cap, 0)));
    return (int) t.size();
}
extern "C" int bark_b200_long_chunk_tokens(struct bark_context * ctx, int k, int stage, int32_t * out, int cap) {
    if (!ctx || k < 0 || k >= (int) ctx->long_form.chunks.size()) return -1;
    return copy_tokens(ctx->long_form.chunks[(size_t) k], stage, out, cap);
}
extern "C" int bark_b200_split_text(const char * const * vocab, int n_vocab, int kind, const char * text, int max_chunk_ids, int32_t * bounds, int cap) {
    const char * fn = "bark_b200_split_text";
    if (!vocab || n_vocab < 0 || !text) { fprintf(stderr, "%s: null vocabulary or text\n", fn); return -1; }
    if (kind != BARK_B200_TOKENIZER_REFERENCE && kind != BARK_B200_TOKENIZER_BERT) { fprintf(stderr, "%s: unknown tokenizer %d (0 reference, 1 bert)\n", fn, kind); return -1; }
    return guarded((int) -1, [&] {
        std::map<std::string, int32_t> v;
        if (!vocab_map(vocab, n_vocab, v, fn)) return -1;
        std::string norm;
        std::vector<std::pair<size_t, size_t>> b;
        const int n = split_text(text, max_chunk_ids, [&](const std::string & t) { return count_text_ids(v, kind, t, fn); }, norm, b, fn);
        for (int i = 0; bounds && i < std::min(n, cap); i++) { bounds[2 * i] = (int32_t) b[(size_t) i].first; bounds[2 * i + 1] = (int32_t) b[(size_t) i].second; }
        return n;
    });
}

// batched generation (include/bark_b200.h)
extern "C" bool bark_b200_generate_batch(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds, int n, int n_threads) {
    (void) n_threads;
    return guarded(false, [&] { return generate_batch(ctx, texts, seeds, nullptr, n); });
}
extern "C" bool bark_b200_generate_batch_prompted(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds,
                                                  const struct bark_b200_history_prompt * const * prompts, int n, int n_threads) {
    (void) n_threads;
    return guarded(false, [&] { return generate_batch(ctx, texts, seeds, prompts, n); });
}
// speaker history prompt of the context's own generations (include/bark_b200.h)
extern "C" int bark_b200_set_history_prompt(struct bark_context * ctx, const struct bark_b200_history_prompt * prompt) {
    if (!ctx) { fprintf(stderr, "bark_b200_set_history_prompt: invalid bark context\n"); return 0; }
    return guarded((int) 0, [&] {
        HistoryPrompt h;                                      // empty: no prompt
        if (prompt && !make_history_prompt(ctx->params, *prompt, h)) return 0;
        ctx->gen.prompt = std::move(h);
        return 1;
    });
}
extern "C" int bark_b200_batch_audio(struct bark_context * ctx, int i, float * out, int cap) {
    if (!ctx || i < 0 || i >= (int) ctx->batch.results.size()) return -1;
    const std::vector<float> & a = ctx->batch.results[(size_t) i].audio;
    if (out) memcpy(out, a.data(), sizeof(float) * std::min(a.size(), (size_t) std::max(cap, 0)));
    return (int) a.size();
}
extern "C" int bark_b200_batch_tokens(struct bark_context * ctx, int i, int stage, int32_t * out, int cap) {
    if (!ctx || i < 0 || i >= (int) ctx->batch.results.size()) return -1;
    return copy_tokens(ctx->batch.results[(size_t) i], stage, out, cap);
}
static int bark_b200_gpt_eval_slot_impl(struct bark_context * ctx, int which, int slot, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) {
    if (!ctx || which < 0 || which > 1 || slot < 0 || slot >= kMaxBatch || !tokens || !n_past || !logits_out) return 0;
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (!ensure_batch_slots(ctx, slot + 1)) return 0;
    return gpt_eval(ctx, *pick(ctx, which), tokens, n, n_past, merge_ctx != 0, logits_out, 0, 0, ctx->batch.k[which][slot], ctx->batch.v[which][slot]) ? 1 : 0;
}
extern "C" int bark_b200_gpt_eval_slot(struct bark_context * ctx, int which, int slot, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) {
    return guarded((int) 0, [&] { return bark_b200_gpt_eval_slot_impl(ctx, which, slot, tokens, n, n_past, merge_ctx, logits_out); });
}
static int bark_b200_gpt_step_batch_impl(struct bark_context * ctx, int which, int B, const int32_t * slots, const int32_t * tokens, int * n_past, float * logits_out) {
    if (!ctx || which < 0 || which > 1 || B < 1 || B > kMaxBatch || !slots || !tokens || !n_past || !logits_out) return 0;
    int top = 0;
    for (int r = 0; r < B; r++) {
        if (slots[r] < 0 || slots[r] >= kMaxBatch) return 0;
        for (int q = 0; q < r; q++) if (slots[q] == slots[r]) { fprintf(stderr, "%s: slot %d appears twice\n", __func__, slots[r]); return 0; }
        top = std::max(top, slots[r] + 1);
    }
    BARK_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (!ensure_batch_slots(ctx, top)) return 0;
    GPTModel & m = *pick(ctx, which);
    float * sk[kMaxBatch], * sv[kMaxBatch];
    for (int r = 0; r < B; r++) { sk[r] = ctx->batch.k[which][slots[r]]; sv[r] = ctx->batch.v[which][slots[r]]; }
    if (!gpt_step_batch(ctx, m, B, sk, sv, tokens, n_past, 0, 0, ctx->batch.d_logits)) return 0;
    const size_t nb = (size_t) B * m.n_out_vocab * 4;
    BARK_CUDA_CHECK(cudaMemcpyAsync(logits_out, ctx->batch.d_logits, nb, cudaMemcpyDeviceToHost, ctx->stream)); g_d2h_bytes += nb;
    BARK_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    for (int r = 0; r < B; r++) n_past[r]++;
    return 1;
}
extern "C" int bark_b200_gpt_step_batch(struct bark_context * ctx, int which, int B, const int32_t * slots, const int32_t * tokens, int * n_past, float * logits_out) {
    return guarded((int) 0, [&] { return bark_b200_gpt_step_batch_impl(ctx, which, B, slots, tokens, n_past, logits_out); });
}

extern "C" const char * bark_b200_version(void) { return "bark_b200 r3 (sm_90a; parity path + opt-in wgmma fast mode)"; }
