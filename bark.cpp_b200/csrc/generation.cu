// The generation drivers (bark.cpp:622-662, 1645-2159): the prompt, the semantic, coarse and fine loops, the codec, and batched generation.
// Semantics follow the reference's, including its quirks (SURVEY.md App. D), because token parity depends on them; the code is new.
#include "context.h"
#include "codec_kernels.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>

using namespace bark;

namespace bark {

bool quiet() { static const bool q = [] { const char * e = getenv("BARK_B200_QUIET"); return e && *e && *e != '0'; }(); return q; }

// bark.cpp:622-662, on the context's tokenizer (tokenizer.cu), its ids cut to a prompt of max_ctx.  false (message naming fn) for a text
// the tokenizer refuses; g is then untouched.
bool tokenize_input(bark_context * ctx, Generation & g, const std::string & text, const char * fn) {
    const bark_context_params & P = ctx->params;
    const int max_ctx = std::min(ctx->semantic.block_size, 256);
    std::vector<int32_t> pieces;
    if (!text_ids(ctx->token_to_id, ctx->tokenizer, text, max_ctx, pieces, fn, true)) return false;
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
bool run_fine(bark_context * ctx, Generation & g, bool progress) {
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

// A failed batch changes nothing a caller can read: bark_b200_batch_* still return the last successful batch.  prompts (may be null,
// and so may any entry): item i's history prompt.
bool generate_batch(bark_context * ctx, const char * const * texts, const uint32_t * seeds, const bark_b200_history_prompt * const * prompts, int n) {
    if (n < 1 || n > kMaxBatch) { fprintf(stderr, "%s: %d prompts (1 to %d per batch)\n", __func__, n, kMaxBatch); return false; }
    if (!texts || !seeds) { fprintf(stderr, "%s: null prompts or seeds\n", __func__); return false; }
    for (int i = 0; i < n; i++) if (!texts[i]) { fprintf(stderr, "%s: prompt %d is null\n", __func__, i); return false; }
    if (ctx->shard.on) { fprintf(stderr, "%s: not available on a context whose fine stage is sharded over GPUs\n", __func__); return false; }
    std::vector<BatchItem> items((size_t) n);
    for (int i = 0; i < n; i++)
        if (prompts && prompts[i] && !make_history_prompt(ctx->params, *prompts[i], items[(size_t) i].g.prompt)) {
            fprintf(stderr, "%s: history prompt %d rejected\n", __func__, i); return false;
        }
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

}  // namespace bark

// One bark_generate_audio on the context's generation state (text tokenized, three stages, codec, statistics); false with a message, and
// nothing changed when the tokenizer refuses the text
bool bark::generate_one(bark_context * ctx, const std::string & text) {
    const char * fn = "bark_generate_audio_impl";
    const int64_t t0 = now_us();
    Generation & g = ctx->gen;
    if (!tokenize_input(ctx, g, text, "bark_generate_audio")) return false;      // a refused text changes nothing
    bark_reset_statistics(ctx);
    if (!run_semantic(ctx, g)) { fprintf(stderr, "%s: failed to forward text encoder\n", fn); return false; }
    if (!run_coarse(ctx, g))   { fprintf(stderr, "%s: failed to forward coarse encoder\n", fn); return false; }
    if (!run_fine(ctx, g))     { fprintf(stderr, "%s: failed to forward fine encoder\n", fn); return false; }
    Generation * gp = &g;
    if (!decode_audio(ctx, &gp, 1)) return false;
    ctx->stats.t_eval_us = now_us() - t0;
    return true;
}

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
