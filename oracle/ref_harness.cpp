// TEST INFRASTRUCTURE — not product code.
//
// Thin C-ABI shim around the UNMODIFIED reference (PABannier/bark.cpp).  It is compiled by
// oracle/Makefile from the sources where they lie under $(REF) (make ref REF=...); nothing from
// the reference is copied into this repository.  The single-TU include below is only there to
// reach the reference's file-static stage functions and bark_context fields so that tests can
//   (a) read the token streams the reference produced (bark.cpp:147-151),
//   (b) teacher-force single GPT evaluations (bark.cpp:1586 bark_eval_encoder_internal,
//       bark.cpp:1907 bark_eval_fine_encoder_internal) and read back the raw logits,
//   (c) run the EnCodec decoder alone (encodec.cpp:902 encodec_decompress_audio).
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load the resulting oracle/_ref/libbark_ref.so.
#include "bark.cpp"   // resolved through -I$(REF)

#include <cstring>

extern "C" {

struct bark_context * ref_load(const char * path, uint32_t seed, int n_steps_text_encoder, int verbosity) {
    bark_context_params p = bark_context_default_params();
    p.verbosity = (bark_verbosity_level) verbosity;
    if (n_steps_text_encoder > 0) p.n_steps_text_encoder = n_steps_text_encoder;
    return bark_load_model(path, p, seed);
}

void ref_set_params(struct bark_context * b, float temp, float fine_temp, float min_eos_p) {
    b->params.temp = temp; b->params.fine_temp = fine_temp; b->params.min_eos_p = min_eos_p;
}

void ref_reseed(struct bark_context * b, uint32_t seed) { b->rng = std::mt19937(seed); }

int ref_generate(struct bark_context * b, const char * text, int n_threads) {
    return bark_generate_audio(b, text, n_threads) ? 1 : 0;
}

void ref_free(struct bark_context * b) { bark_free(b); }

// ---- stage-by-stage drivers (same order as bark_forward_eval, bark.cpp:2106) -------------------
void ref_tokenize(struct bark_context * b, const char * text) { bark_tokenize_input(b, std::string(text)); }
int  ref_run_semantic(struct bark_context * b, int n_threads) { return bark_forward_text_encoder(b, n_threads); }
int  ref_run_coarse(struct bark_context * b, int n_threads)   { return bark_forward_coarse_encoder(b, n_threads); }
int  ref_run_fine(struct bark_context * b, int n_threads)     { return bark_forward_fine_encoder(b, n_threads); }

void ref_set_semantic(struct bark_context * b, const int32_t * t, int n) { b->semantic_tokens.assign(t, t + n); }
void ref_set_coarse(struct bark_context * b, const int32_t * t, int n_frames) {   // [T][2]
    b->coarse_tokens.clear();
    for (int i = 0; i < n_frames; i++) b->coarse_tokens.push_back({t[2*i], t[2*i+1]});
}

// ---- result accessors ---------------------------------------------------------------------------
int ref_n_prompt(struct bark_context * b)   { return (int) b->tokens.size(); }
int ref_n_semantic(struct bark_context * b) { return (int) b->semantic_tokens.size(); }
int ref_n_frames(struct bark_context * b)   { return (int) b->coarse_tokens.size(); }
int ref_n_fine_frames(struct bark_context * b) { return (int) b->fine_tokens.size(); }
void ref_get_prompt(struct bark_context * b, int32_t * o)   { memcpy(o, b->tokens.data(), 4 * b->tokens.size()); }
void ref_get_semantic(struct bark_context * b, int32_t * o) { memcpy(o, b->semantic_tokens.data(), 4 * b->semantic_tokens.size()); }
void ref_get_coarse(struct bark_context * b, int32_t * o) {      // [T][2]
    for (size_t i = 0; i < b->coarse_tokens.size(); i++) for (int j = 0; j < 2; j++) o[2*i+j] = b->coarse_tokens[i][j];
}
void ref_get_fine(struct bark_context * b, int32_t * o) {        // [T][8]
    for (size_t i = 0; i < b->fine_tokens.size(); i++) for (int j = 0; j < 8; j++) o[8*i+j] = b->fine_tokens[i][j];
}
int ref_n_audio(struct bark_context * b) { return bark_get_audio_data_size(b); }
void ref_get_audio(struct bark_context * b, float * o) { memcpy(o, bark_get_audio_data(b), 4 * (size_t) bark_get_audio_data_size(b)); }

void ref_get_stats(struct bark_context * b, int64_t * o) {
    // load, eval, semantic, coarse, fine (us); then per-model predict / sample us and n_sample
    o[0] = b->stats.t_load_us; o[1] = b->stats.t_eval_us;
    o[2] = b->stats.t_semantic_us; o[3] = b->stats.t_coarse_us; o[4] = b->stats.t_fine_us;
    gpt_model * m[3] = { &b->text_model.semantic_model, &b->text_model.coarse_model, &b->text_model.fine_model };
    for (int i = 0; i < 3; i++) { o[5+3*i] = m[i]->t_predict_us; o[6+3*i] = m[i]->t_sample_us; o[7+3*i] = m[i]->n_sample; }
}

void ref_get_hparams(struct bark_context * b, int which, int32_t * o) {
    gpt_model * m[3] = { &b->text_model.semantic_model, &b->text_model.coarse_model, &b->text_model.fine_model };
    const gpt_hparams & h = m[which]->hparams;
    o[0]=h.n_layer; o[1]=h.n_head; o[2]=h.n_embd; o[3]=h.block_size; o[4]=h.bias; o[5]=h.n_in_vocab;
    o[6]=h.n_out_vocab; o[7]=h.n_lm_heads; o[8]=h.n_wtes; o[9]=h.ftype;
}

// ---- teacher forcing: one causal-GPT evaluation (bark.cpp:1586) ----------------------------------
// which: 0 semantic, 1 coarse.  tokens/n: the ids fed this step.  *n_past is advanced like the
// reference does.  logits_out must hold n_out_vocab floats.
int ref_gpt_eval(struct bark_context * b, int which, const int32_t * tokens, int n, int * n_past,
                 int merge_ctx, int n_threads, float * logits_out) {
    gpt_model & model = which == 0 ? b->text_model.semantic_model : b->text_model.coarse_model;
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(model.backend));
    bark_sequence in(tokens, tokens + n);
    std::vector<float> logits;
    bool ok = bark_eval_encoder_internal(model, allocr, in, logits, n_past, merge_ctx != 0, n_threads);
    if (ok) memcpy(logits_out, logits.data(), sizeof(float) * logits.size());
    ggml_gallocr_free(allocr);
    return ok ? 1 : 0;
}

// One non-causal fine pass (bark.cpp:1907).  in_buffer: [8][1024] ids, nn: codebook to predict
// (2..7).  logits_out: [1024][n_out_vocab(1056)].
int ref_fine_eval(struct bark_context * b, const int32_t * in_buffer, int nn, int n_threads, float * logits_out) {
    gpt_model & model = b->text_model.fine_model;
    b->allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(model.backend));
    bark_sequence in(in_buffer, in_buffer + 8 * 1024);
    std::vector<float> logits(1024 * model.hparams.n_out_vocab);
    bool ok = bark_eval_fine_encoder_internal(b, in, logits, nn, n_threads);
    if (ok) memcpy(logits_out, logits.data(), sizeof(float) * logits.size());
    ggml_gallocr_free(b->allocr);
    return ok ? 1 : 0;
}

// host sampler exactly as the stage drivers call it (bark.cpp:249 gpt_sample)
int ref_sample(struct bark_context * b, const float * logits, int n, float temp, float * eos_p) {
    std::vector<float> l(logits, logits + n);
    int64_t t = 0, ns = 0;
    return gpt_sample(l, b->rng, temp, eos_p, &t, &ns);
}

// EnCodec decoder alone.  codes: [8][T] (codebook-major, bark.cpp:2151-2159). returns #samples.
int ref_encodec_decode(struct bark_context * b, const int32_t * codes, int n_codes, int n_threads) {
    encodec_set_target_bandwidth(b->encodec_ctx, b->params.target_bandwidth);
    encodec_set_sample_rate(b->encodec_ctx, b->params.sample_rate);
    if (!encodec_decompress_audio(b->encodec_ctx, codes, n_codes, n_threads)) return -1;
    b->generated_audio     = encodec_get_audio(b->encodec_ctx);
    b->n_generated_samples = encodec_get_audio_size(b->encodec_ctx);
    return b->n_generated_samples;
}

// 65536-entry GELU table as the reference builds it at init (ggml.c:3795-3810): indexed by the
// f16 bit pattern, stored as f16 bit patterns.  Run through a one-op graph so that whatever the
// compiler did to the scalar formula is captured (SURVEY App. C, contraction caveat).
void ref_gelu_table(uint16_t * out) {
    struct ggml_init_params ip = { 16u * 1024 * 1024, NULL, false };
    struct ggml_context * ctx = ggml_init(ip);
    struct ggml_tensor * x = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, 65536);
    for (int i = 0; i < 65536; i++) ((float *) x->data)[i] = ggml_fp16_to_fp32((ggml_fp16_t) i);
    struct ggml_tensor * y = ggml_gelu(ctx, x);
    struct ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, y);
    ggml_graph_compute_with_ctx(ctx, gf, 1);
    for (int i = 0; i < 65536; i++) out[i] = ggml_fp32_to_fp16(((float *) y->data)[i]);
    ggml_free(ctx);
}

// the reference's own quantize tool entry point (bark.cpp:2300) so fixtures can be made without
// building examples/quantize.
int ref_quantize(const char * in, const char * out, int ftype) { return bark_model_quantize(in, out, (ggml_ftype) ftype) ? 1 : 0; }

const char * ref_build_info(void) {
    return "bark.cpp 5d5be84 / encodec.cpp 1cc279d / ggml c18f9ba; " REF_BUILD_FLAGS;
}

}  // extern "C"
