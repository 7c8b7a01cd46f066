// The bark.h C API (include/bark.h) and the additive entry points of include/bark_b200.h: context lifecycle (bark.cpp:1165-1184,
// 2189-2232, 2379-2407) and one call path, with_context, behind every call on a context.
#include "../../include/bark_b200.h"
#include "context.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <climits>
#include <cstring>

using namespace bark;

namespace {

thread_local int g_device_override = -1;   // bark_b200_set_device applies to the calling thread's next bark_load_model

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
    const int tokenizer = tokenizer_from_env(__func__);       // BARK_B200_TOKENIZER: the context's initial tokenizer (include/bark_b200.h)
    if (tokenizer < 0) return nullptr;
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

extern "C" bool bark_b200_forward_text_encoder(struct bark_context * ctx, int) { return with_context(ctx, __func__, false, [&] { return run_semantic(ctx, ctx->gen); }); }
extern "C" bool bark_b200_forward_coarse_encoder(struct bark_context * ctx, int) { return with_context(ctx, __func__, false, [&] { return run_coarse(ctx, ctx->gen); }); }
extern "C" bool bark_b200_forward_fine_encoder(struct bark_context * ctx, int) { return with_context(ctx, __func__, false, [&] { return run_fine(ctx, ctx->gen); }); }
// the reference also exports these three as C++ symbols without a header (bark.cpp:1703,1865,2061)
BARK_API bool bark_forward_text_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_text_encoder(ctx, n); }
BARK_API bool bark_forward_coarse_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_coarse_encoder(ctx, n); }
BARK_API bool bark_forward_fine_encoder(struct bark_context * ctx, int n) { return bark_b200_forward_fine_encoder(ctx, n); }

extern "C" bool bark_generate_audio(struct bark_context * ctx, const char * text, int n_threads) {
    (void) n_threads;                      // CPU thread count of the reference's backend; nothing to size here
    return with_context(ctx, __func__, false, [&] {
        if (!text) { fprintf(stderr, "%s: null prompt\n", "bark_generate_audio"); return false; }
        if (ctx->long_form.on) return generate_long(ctx, text);
        if (!generate_one(ctx, text)) return false;
        ctx->long_form.chunks.clear();     // the chunk getters describe the last generation only
        return true;
    });
}

extern "C" float * bark_get_audio_data(struct bark_context * ctx) { return with_context<float *>(ctx, __func__, nullptr, [&] { return ctx->gen.audio.empty() ? nullptr : ctx->gen.audio.data(); }); }
extern "C" int bark_get_audio_data_size(struct bark_context * ctx) { return with_context(ctx, __func__, 0, [&] { return (int) ctx->gen.audio.size(); }); }
extern "C" int64_t bark_get_load_time(struct bark_context * ctx) { return with_context<int64_t>(ctx, __func__, 0, [&] { return ctx->stats.t_load_us; }); }
extern "C" int64_t bark_get_eval_time(struct bark_context * ctx) { return with_context<int64_t>(ctx, __func__, 0, [&] { return ctx->stats.t_eval_us; }); }

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

extern "C" int bark_b200_gpt_eval(struct bark_context * ctx, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) {
    return with_context(ctx, __func__, 0, [&] {
        if (which < 0 || which > 1 || !tokens || !logits_out) return 0;
        return gpt_eval(ctx, *pick(ctx, which), tokens, n, n_past, merge_ctx != 0, logits_out) ? 1 : 0;
    });
}
extern "C" int bark_b200_fine_eval(struct bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_out) { return with_context(ctx, __func__, 0, [&] { return in_buffer && logits_out && fine_eval(ctx, in_buffer, nn, logits_out) ? 1 : 0; }); }
extern "C" int bark_b200_encodec_decode(struct bark_context * ctx, const int32_t * codes, int n_frames, float * out, int out_cap) {
    return with_context(ctx, __func__, -1, [&] {
        if (!codes || !codec_decode(ctx->codec, ctx->codec_scratch, ctx->stream, 1, &codes, &n_frames, 8, &ctx->gen.audio)) return -1;
        return copy_out(ctx->gen.audio, out, out_cap);
    });
}
// the two encoder hooks, named fn: the clip's codes [8][T] and latent [128][T] copied out, T returned; fmt: the resampled call's format
static int encode_hook(bark_context * ctx, const char * fn, const float * audio, int n_samples, int32_t * codes, int codes_cap, float * latent, int latent_cap,
                       const AudioFormat * fmt) {
    return with_context(ctx, fn, -1, [&] {
        if (!audio) { fprintf(stderr, "%s: null audio\n", fn); return -1; }
        std::vector<int32_t> c; std::vector<float> l;
        if (!codec_encode(ctx->codec, ctx->codec_scratch, ctx->stream, 1, &audio, &n_samples, 8, {&c, &l}, nullptr, fmt)) return -1;
        copy_out(c, codes, codes_cap); copy_out(l, latent, latent_cap);
        return (int)(c.size() / 8);
    });
}
extern "C" int bark_b200_encodec_encode(struct bark_context * ctx, const float * audio, int n_samples, int32_t * codes, int codes_cap, float * latent,
                                        int latent_cap) {
    return encode_hook(ctx, __func__, audio, n_samples, codes, codes_cap, latent, latent_cap, nullptr);
}
extern "C" int bark_b200_encodec_encode_resampled(struct bark_context * ctx, const float * audio, int n_frames, int channels, int sample_rate, int32_t * codes,
                                                  int codes_cap, float * latent, int latent_cap) {
    const AudioFormat f{channels, sample_rate};
    return encode_hook(ctx, __func__, audio, n_frames, codes, codes_cap, latent, latent_cap, &f);
}
extern "C" int bark_b200_sample(struct bark_context * ctx, int which, const float * logits, int n, float temp, float * eos_p) {
    return with_context(ctx, __func__, -1, [&] {
        if (!logits || n < 1) return -1;
        GPTModel & m = *pick(ctx, which < 0 || which > 2 ? 0 : which);
        const int64_t t0 = now_us();
        // what libstdc++'s discrete distribution takes: one draw, none on the argmax path or for a single logit
        const double u = temp != 0.0f && n > 1 ? std::generate_canonical<double, 53>(ctx->gen.rng) : 0.0;
        const int32_t next = sample_token_given_u(logits, n, temp, u, eos_p);
        m.t_sample_us += now_us() - t0;
        m.n_sample += 1;
        return next;
    });
}
extern "C" int bark_b200_sample_rows(struct bark_context * ctx, const float * logits, int n, int rows, float temp, int32_t * tokens_out, float * eos_p_out) {
    return with_context(ctx, __func__, -1, [&] {
        if (!logits || !tokens_out || rows < 1 || rows > 1024 || n < 2 || n > kSampleMaxLogits) return -1;
        const size_t cap = std::max<size_t>({(size_t) ctx->semantic.n_out_vocab, (size_t) ctx->coarse.n_out_vocab, (size_t) 1024 * ctx->fine.n_out_vocab});
        if ((size_t) rows * n > cap) return -1;
        BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->ws.logits, logits, (size_t) rows * n * 4, cudaMemcpyHostToDevice, ctx->stream));
        const long long before = ctx->n_sample_host_replays;
        if (!sample_device(ctx, ctx->fine, ctx->gen.rng, ctx->ws.logits, n, n, rows, temp, tokens_out, eos_p_out)) return -1;
        return (int)(ctx->n_sample_host_replays - before);
    });
}
extern "C" void bark_b200_reseed(struct bark_context * ctx, uint32_t seed) { with_context(ctx, __func__, false, [&] { ctx->gen.rng = std::mt19937(seed); return true; }); }
extern "C" void bark_b200_tokenize(struct bark_context * ctx, const char * text, int32_t * out513) {
    with_context(ctx, __func__, false, [&] {
        if (!text || !out513 || !tokenize_input(ctx, ctx->gen, text, "bark_b200_tokenize")) return false;
        memcpy(out513, ctx->gen.tokens.data(), sizeof(int32_t) * 513);
        return true;
    });
}
template <class G>       // a Generation or a LongFormChunk
static int copy_tokens(const G & g, int stage, int32_t * out, int cap) {
    const std::vector<int32_t> * v = stage == 0 ? &g.semantic_tokens : stage == 1 ? &g.coarse_tokens : stage == 2 ? &g.fine_tokens : stage == 3 ? &g.tokens : nullptr;
    return v ? copy_out(*v, out, cap) : -1;
}
extern "C" int bark_b200_get_tokens(struct bark_context * ctx, int stage, int32_t * out, int cap) { return with_context(ctx, __func__, -1, [&] { return copy_tokens(ctx->gen, stage, out, cap); }); }
extern "C" void bark_b200_set_tokens(struct bark_context * ctx, int stage, const int32_t * in, int n) {
    with_context(ctx, __func__, false, [&] {
        if (!in || n < 0) return false;
        Generation & g = ctx->gen;
        if (stage == 0) g.semantic_tokens.assign(in, in + n); else if (stage == 1) g.coarse_tokens.assign(in, in + n); else if (stage == 3) g.tokens.assign(in, in + n);
        return true;
    });
}
extern "C" void bark_b200_get_stats(struct bark_context * ctx, struct bark_statistics * out, int64_t * per_model9) {
    with_context(ctx, __func__, false, [&] {
        if (out) *out = ctx->stats;
        if (per_model9) { const GPTModel * m[3] = {&ctx->semantic, &ctx->coarse, &ctx->fine}; for (int i = 0; i < 3; i++) { per_model9[3 * i] = m[i]->t_predict_us; per_model9[3 * i + 1] = m[i]->t_sample_us; per_model9[3 * i + 2] = m[i]->n_sample; } }
        return true;
    });
}
extern "C" void bark_b200_get_hparams(struct bark_context * ctx, int which, int32_t * out10) {
    with_context(ctx, __func__, false, [&] {
        const GPTModel * m = pick(ctx, which); if (!out10 || !m) return false;
        const int32_t v[10] = {m->n_layer, m->n_head, m->n_embd, m->block_size, m->bias, m->n_in_vocab, m->n_out_vocab, m->n_lm_heads, m->n_wtes, m->ftype};
        memcpy(out10, v, sizeof(v));
        return true;
    });
}
extern "C" unsigned long long bark_b200_kernel_launches(void) { return g_kernel_launches.load(); }
extern "C" unsigned bark_b200_layernorm_fallbacks(struct bark_context * ctx) {
    return with_context(ctx, __func__, 0u, [&] { unsigned v = 0; BARK_CUDA_CHECK(cudaMemcpy(&v, ctx->d_ln_fallbacks, sizeof(v), cudaMemcpyDeviceToHost)); return v; });
}
extern "C" int bark_b200_decode_timing(struct bark_context * ctx, unsigned long long * out, int n) {
    return with_context(ctx, __func__, 0, [&] {
        if (!ctx->d_timing || !out) return 0;
        BARK_CUDA_CHECK(cudaMemcpy(out, ctx->d_timing, sizeof(unsigned long long) * (size_t) std::min(n, 256 * 32), cudaMemcpyDeviceToHost));
        return std::min(n, 256 * 32);
    });
}
extern "C" int bark_b200_fast_mode(struct bark_context * ctx) { return with_context(ctx, __func__, 0, [&] { return ctx->fast_mode ? 1 : 0; }); }

extern "C" int bark_b200_set_sampling(struct bark_context * ctx, int stage, const struct bark_b200_sampling * s) {
    const char * fn = "bark_b200_set_sampling";
    return with_context(ctx, fn, 0, [&] {
        if (stage != 0 && stage != 1) { fprintf(stderr, "%s: stage %d (0 semantic, 1 coarse; the fine stage has no filter)\n", fn, stage); return 0; }
        if (s && !sampling_valid(fn, *s)) return 0;
        ctx->sampling[stage] = s ? *s : bark_b200_sampling{0, 0, 1.0f};
        return 1;
    });
}

// text tokenizers (include/bark_b200.h, tokenizer.cu)
extern "C" int bark_b200_set_tokenizer(struct bark_context * ctx, int kind) {
    const char * fn = "bark_b200_set_tokenizer";
    return with_context(ctx, fn, 0, [&] {
        if (!tokenizer_known(kind, fn)) return 0;
        ctx->tokenizer = kind;
        return 1;
    });
}
extern "C" int bark_b200_text_ids(struct bark_context * ctx, int kind, const char * text, int32_t * out, int cap) {
    const char * fn = "bark_b200_text_ids";
    return with_context(ctx, fn, -1, [&] {
        if (!text) { fprintf(stderr, "%s: null text\n", fn); return -1; }
        std::vector<int32_t> ids;
        return text_ids(ctx->token_to_id, kind, text, INT_MAX, ids, fn, true) ? copy_out(ids, out, cap) : -1;
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
        return copy_out(ids, out, cap);
    });
}

// long-form generation (include/bark_b200.h, long_form.cu)
extern "C" int bark_b200_set_long_form(struct bark_context * ctx, const struct bark_b200_long_form * lf) {
    const char * fn = "bark_b200_set_long_form";
    return with_context(ctx, fn, 0, [&] {
        if (!lf) { ctx->long_form.on = false; return 1; }
        if (lf->voice != BARK_B200_VOICE_CHAIN && lf->voice != BARK_B200_VOICE_FIXED) { fprintf(stderr, "%s: unknown voice %d (0 chain, 1 fixed)\n", fn, lf->voice); return 0; }
        if (lf->max_chunk_ids < 1 || lf->max_chunk_ids > 255) { fprintf(stderr, "%s: max_chunk_ids %d (1 to 255)\n", fn, lf->max_chunk_ids); return 0; }
        if (lf->gap_samples < 0 || lf->gap_samples > 240000) { fprintf(stderr, "%s: gap_samples %d (0 to 240000)\n", fn, lf->gap_samples); return 0; }
        ctx->long_form.settings = *lf;
        ctx->long_form.on = true;
        return 1;
    });
}
extern "C" int bark_b200_long_chunks(struct bark_context * ctx) { return with_context(ctx, __func__, -1, [&] { return (int) ctx->long_form.chunks.size(); }); }
extern "C" int bark_b200_long_chunk_text(struct bark_context * ctx, int k, char * out, int cap) {
    return with_context(ctx, __func__, -1, [&] { return k < 0 || k >= (int) ctx->long_form.chunks.size() ? -1 : copy_out(ctx->long_form.chunks[(size_t) k].text, out, cap); });
}
extern "C" int bark_b200_long_chunk_tokens(struct bark_context * ctx, int k, int stage, int32_t * out, int cap) {
    return with_context(ctx, __func__, -1, [&] { return k < 0 || k >= (int) ctx->long_form.chunks.size() ? -1 : copy_tokens(ctx->long_form.chunks[(size_t) k], stage, out, cap); });
}
extern "C" int bark_b200_split_text(const char * const * vocab, int n_vocab, int kind, const char * text, int max_chunk_ids, int32_t * bounds, int cap) {
    const char * fn = "bark_b200_split_text";
    if (!vocab || n_vocab < 0 || !text) { fprintf(stderr, "%s: null vocabulary or text\n", fn); return -1; }
    if (!tokenizer_known(kind, fn)) return -1;
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

// batched generation (include/bark_b200.h, generation.cu)
extern "C" bool bark_b200_generate_batch(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds, int n, int /*n_threads*/) {
    return with_context(ctx, __func__, false, [&] { return generate_batch(ctx, texts, seeds, nullptr, n); });
}
extern "C" bool bark_b200_generate_batch_prompted(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds,
                                                  const struct bark_b200_history_prompt * const * prompts, int n, int /*n_threads*/) {
    return with_context(ctx, __func__, false, [&] { return generate_batch(ctx, texts, seeds, prompts, n); });
}
// speaker history prompt of the context's own generations (include/bark_b200.h)
extern "C" int bark_b200_set_history_prompt(struct bark_context * ctx, const struct bark_b200_history_prompt * prompt) {
    return with_context(ctx, __func__, 0, [&] {
        HistoryPrompt h;                                      // empty: no prompt
        if (prompt && !make_history_prompt(ctx->params, *prompt, h)) return 0;
        ctx->gen.prompt = std::move(h);
        return 1;
    });
}
extern "C" int bark_b200_batch_audio(struct bark_context * ctx, int i, float * out, int cap) {
    return with_context(ctx, __func__, -1, [&] { return i < 0 || i >= (int) ctx->batch.results.size() ? -1 : copy_out(ctx->batch.results[(size_t) i].audio, out, cap); });
}
extern "C" int bark_b200_batch_tokens(struct bark_context * ctx, int i, int stage, int32_t * out, int cap) {
    return with_context(ctx, __func__, -1, [&] { return i < 0 || i >= (int) ctx->batch.results.size() ? -1 : copy_tokens(ctx->batch.results[(size_t) i], stage, out, cap); });
}
extern "C" int bark_b200_gpt_eval_slot(struct bark_context * ctx, int which, int slot, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out) {
    return with_context(ctx, __func__, 0, [&] {
        if (which < 0 || which > 1 || slot < 0 || slot >= kMaxBatch || !tokens || !n_past || !logits_out) return 0;
        if (!ensure_batch_slots(ctx, slot + 1)) return 0;
        return gpt_eval(ctx, *pick(ctx, which), tokens, n, n_past, merge_ctx != 0, logits_out, 0, 0, ctx->batch.k[which][slot], ctx->batch.v[which][slot]) ? 1 : 0;
    });
}
extern "C" int bark_b200_gpt_step_batch(struct bark_context * ctx, int which, int B, const int32_t * slots, const int32_t * tokens, int * n_past, float * logits_out) {
    return with_context(ctx, __func__, 0, [&] {
        if (which < 0 || which > 1 || B < 1 || B > kMaxBatch || !slots || !tokens || !n_past || !logits_out) return 0;
        int top = 0;
        for (int r = 0; r < B; r++) {
            if (slots[r] < 0 || slots[r] >= kMaxBatch) return 0;
            for (int q = 0; q < r; q++) if (slots[q] == slots[r]) { fprintf(stderr, "%s: slot %d appears twice\n", "bark_b200_gpt_step_batch", slots[r]); return 0; }
            top = std::max(top, slots[r] + 1);
        }
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
    });
}

extern "C" const char * bark_b200_version(void) { return "bark_b200 r3 (sm_90a; parity path + opt-in wgmma fast mode)"; }
