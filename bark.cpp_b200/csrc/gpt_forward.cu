// Per-call orchestration of the GPT kernels: the device-side replacement of bark_eval_encoder_internal (bark.cpp:1586-1643) and
// bark_eval_fine_encoder_internal (bark.cpp:1907-1959).  No graph is built or allocated per step: the workspace is sized once at load
// for the worst case (block_size rows).
#include "context.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <vector>
#include <time.h>

namespace bark {

int64_t now_us() {
    timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
    return (int64_t) ts.tv_sec * 1000000 + ts.tv_nsec / 1000;
}


// Quantised weights take f32 rows (told W_Q4_0; row stride E, 4E after fc); f32 / f16 weights the group-major operand of the
// workspace's row capacity, whose group stride is the same for both widths
static ActLayout act_layout(const Workspace & ws, const GPTModel & m) {
    if (is_quant(m.wtype)) return {W_Q4_0, m.n_embd, 4 * m.n_embd};
    return {m.wtype, ws.max_rows * kGmGroup, ws.max_rows * kGmGroup};
}

template <class KV> void run_layers(bark_context * ctx, const GPTModel & m, int rows, const KV & kv) {
    Workspace & ws = ctx->ws;
    cudaStream_t s = ctx->stream;
    const int E = m.n_embd;
    const ActLayout a = act_layout(ws, m);
    for (int il = 0; il < m.n_layer; il++) {
        const GPTLayer & L = m.layers[(size_t) il];
        layernorm_act(ws.x, rows, E, L.ln_1_g, L.ln_1_b, ws.act, a.wt, a.kpE, ctx->d_ln_fallbacks, s);
        MatmulEpilogue qkv; qkv.mode = EPI_QKV; qkv.out = ws.q; qkv.ldo = E;
        kv.store(ctx, m, il, rows, qkv);
        lane_matmul(L.c_attn, ws.act, a.kpE, rows, qkv, &ctx->q8, s);
        kv.attend(ctx, m, il, rows, a);
        MatmulEpilogue res; res.mode = EPI_RESID; res.out = ws.x; res.ldo = E;
        lane_matmul(L.c_proj, ws.act, a.kpE, rows, res, &ctx->q8, s);                                                 // + inpL
        layernorm_act(ws.x, rows, E, L.ln_2_g, L.ln_2_b, ws.act, a.wt, a.kpE, ctx->d_ln_fallbacks, s);
        MatmulEpilogue ge; ge.mode = EPI_GELU_ACT; ge.act_out = ws.act2; ge.act_wt = (int) a.wt; ge.act_Kp = a.kp4E; ge.gelu_tab = ctx->d_gelu_tab;
        lane_matmul(L.fc, ws.act, a.kpE, rows, ge, &ctx->q8, s);
        lane_matmul(L.proj, ws.act2, a.kp4E, rows, res, &ctx->q8, s);                                                // + inpFF
    }
}
template void run_layers(bark_context *, const GPTModel &, int, const ShardKV &);

// K / V in this device's memory: layer il's rows at k / v + il * layer_floats, this call's rows from position n_past on.  The causal
// cache ([L][block_size][E], bark.cpp:1294-1300; each row attends to the keys up to its own position) or the fine model's scratch
// (one [1024][E] buffer that every layer reuses, no mask).
struct LocalKV {
    float * k, * v; size_t layer_floats; int n_past; bool causal;
    void store(bark_context *, const GPTModel & m, int il, int, MatmulEpilogue & qkv) const {
        const size_t at = il * layer_floats + (size_t) n_past * m.n_embd;
        qkv.k_out = k + at; qkv.v_out = v + at;
    }
    void attend(bark_context * ctx, const GPTModel & m, int il, int rows, const ActLayout & a) const {
        Workspace & ws = ctx->ws;
        attention(ws.q, k + il * layer_floats, v + il * layer_floats, rows, n_past + rows, n_past, m.n_embd, m.n_head, causal, ws.scores, ws.act, a.wt,
                  a.kpE, ctx->stream);
    }
};

// The rows of a batched decode step (gpt_step_batch): row b belongs to its own sequence, with its own KV cache slot and position.
// The K / V rows are staged in ws.kbuf / ws.vbuf, and the batched attention appends each to its own cache.
struct SlotKV {
    float * const * slot_k, * const * slot_v; const int32_t * d_pos; int max_kv;
    void store(bark_context * ctx, const GPTModel &, int, int, MatmulEpilogue & qkv) const { qkv.k_out = ctx->ws.kbuf; qkv.v_out = ctx->ws.vbuf; }
    void attend(bark_context * ctx, const GPTModel & m, int il, int rows, const ActLayout & a) const {
        Workspace & ws = ctx->ws;
        const size_t layer = (size_t) il * m.block_size * m.n_embd;
        BatchKV kv;
        for (int b = 0; b < rows; b++) { kv.k[b] = slot_k[b] + layer; kv.v[b] = slot_v[b] + layer; }
        attention_batch(ws.q, ws.kbuf, ws.vbuf, kv, d_pos, rows, max_kv, m.n_embd, m.n_head, ws.scores, ws.act, a.wt, a.kpE, ctx->stream);
    }
};

void output_head(bark_context * ctx, const GPTModel & m, const float * x, int rows, const DMat & head, float * logits, int lo) {
    const ActLayout a = act_layout(ctx->ws, m);
    layernorm_act(x, rows, m.n_embd, m.ln_f_g, m.ln_f_b, ctx->ws.act, a.wt, a.kpE, ctx->d_ln_fallbacks, ctx->stream);
    MatmulEpilogue st; st.mode = EPI_STORE; st.out = logits + lo; st.ldo = m.n_out_vocab;
    lane_matmul(head, ctx->ws.act, a.kpE, rows, st, &ctx->q8, ctx->stream);
    ctx->last_logits = logits;
}

// count device logits at d_src + offset -> host_dst + offset through the pinned buffer, waiting for the stream (nothing without host_dst)
static void read_logits(bark_context * ctx, const float * d_src, size_t offset, size_t count, float * host_dst) {
    if (!host_dst) return;
    const size_t nb = count * sizeof(float);
    BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_logits, d_src + offset, nb, cudaMemcpyDeviceToHost, ctx->stream)); g_d2h_bytes += nb;
    BARK_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    memcpy(host_dst + offset, ctx->h_logits, nb);
}

// the logits [lm_lo, lm_hi) a causal pass computes: all of them when lm_hi <= 0 or the range is not one of the model's
static void clamp_lm(const GPTModel & m, int & lm_lo, int & lm_hi) {
    if (lm_hi <= 0 || lm_hi > m.n_out_vocab || lm_lo < 0 || lm_lo >= lm_hi) { lm_lo = 0; lm_hi = m.n_out_vocab; }
}

// Phase table + exchange buffers of the persistent decode kernel (decode_kernels.cu), once per causal model.
void build_decode_tables(bark_context * ctx, GPTModel & m) {
    const int L = m.n_layer, E = m.n_embd;
    // Fixed capacities of gpt_decode_step_kernel: shared-memory vectors of 1024 (x, q / probabilities) and 4096 (activation operand)
    // floats, 128 phase slots, one soft_max tile per CTA (H * head/16 tiles).  A model outside them steps
    // through the per-op kernels instead (same results, slower) — never through a kernel it would overrun.
    const int D = E / m.n_head;
    m.decode_ok = E <= 1024 && 4 * E <= 4096 && 4 * L + 1 <= 128 && m.block_size <= 1024 && m.n_head * (D / 16) <= ctx->n_sm;
    if (!m.decode_ok) {
        fprintf(stderr, "bark_b200: model (n_embd %d, n_layer %d, n_head %d, block_size %d) exceeds the persistent decode kernel's capacities; decoding with the per-op kernels\n", E, L, m.n_head, m.block_size);
        return;
    }
    const size_t es = m.wtype == W_F16 ? 2 : 4;
    const bool q4 = m.wtype == W_Q4_0;
    std::vector<DecodePhase> ph((size_t) 4 * L + 1);
    std::vector<DecodeLayerVec> lv((size_t) L);
    auto set = [&](DecodePhase & p, const DMat & d) {        // q4_0: 16 nibble bytes per 32-element block, block scales in a second array
        p.w = d.p; p.n_out = d.n_out; p.K = d.K; p.row_bytes = q4 ? d.K / 2 : (int)(d.Kp * es); p.pad = 0; p.ws = q4 ? d.scales : nullptr;
    };
    for (int l = 0; l < L; l++) {
        const GPTLayer & G = m.layers[(size_t) l];
        set(ph[(size_t) 4 * l], G.c_attn); set(ph[(size_t) 4 * l + 1], G.c_proj); set(ph[(size_t) 4 * l + 2], G.fc); set(ph[(size_t) 4 * l + 3], G.proj);
        lv[(size_t) l] = DecodeLayerVec{G.ln_1_g, G.ln_1_b, G.ln_2_g, G.ln_2_b};
    }
    set(ph[(size_t) 4 * L], m.lm_head[0]);
    m.d_phases = ctx_alloc(ctx, ph.size() * sizeof(DecodePhase));
    m.d_layer_vecs = ctx_alloc(ctx, lv.size() * sizeof(DecodeLayerVec));
    BARK_CUDA_CHECK(cudaMemcpy(m.d_phases, ph.data(), ph.size() * sizeof(DecodePhase), cudaMemcpyHostToDevice));
    BARK_CUDA_CHECK(cudaMemcpy(m.d_layer_vecs, lv.data(), lv.size() * sizeof(DecodeLayerVec), cudaMemcpyHostToDevice));
    auto tagged = [&](size_t n) { void * p = ctx_alloc(ctx, n * 8); BARK_CUDA_CHECK(cudaMemset(p, 0, n * 8)); return (unsigned long long *) p; };   // epoch 0 = never published
    const size_t R = kDecodeReplicas;                         // vectors every CTA gathers exist in R copies (decode_kernels.cu)
    m.gx = tagged(R * E); m.gq = tagged(R * E); m.gk = tagged((size_t) E); m.gv = tagged((size_t) E); m.gatt = tagged(R * E);
    m.gff = tagged(R * 4 * E); m.gscores = tagged((size_t) m.n_head * m.block_size);
    m.glogits = (float *) ctx_alloc(ctx, (size_t) m.n_out_vocab * 4);
}

// one decode token through the persistent kernel at position *pos: its logits become last_logits and the position advances
static void decode_step(bark_context * ctx, GPTModel & m, int token, const int32_t * d_token, int * pos, int lm_lo, int lm_hi, float * mem_k, float * mem_v) {
    const int n_past = *pos;
    // Epochs are 32-bit and must never repeat while a stale word could still carry the old value (~30 M tokens for 24 layers):
    // before the counter wraps, drain the stream, clear every exchange word (epoch 0 = never published) and start over.
    const unsigned step_tags = (unsigned) decode_tags_per_step(m.n_layer);
    if (ctx->tag_base + step_tags + 1u < ctx->tag_base) {
        BARK_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        for (GPTModel * g : {&ctx->semantic, &ctx->coarse}) {
            if (!g->decode_ok) continue;
            const size_t E8 = (size_t) g->n_embd * 8, R = kDecodeReplicas;
            BARK_CUDA_CHECK(cudaMemsetAsync(g->gx, 0, R * E8, ctx->stream)); BARK_CUDA_CHECK(cudaMemsetAsync(g->gq, 0, R * E8, ctx->stream));
            BARK_CUDA_CHECK(cudaMemsetAsync(g->gatt, 0, R * E8, ctx->stream)); BARK_CUDA_CHECK(cudaMemsetAsync(g->gff, 0, R * 4 * E8, ctx->stream));
            BARK_CUDA_CHECK(cudaMemsetAsync(g->gk, 0, E8, ctx->stream)); BARK_CUDA_CHECK(cudaMemsetAsync(g->gv, 0, E8, ctx->stream));
            BARK_CUDA_CHECK(cudaMemsetAsync(g->gscores, 0, (size_t) g->n_head * g->block_size * 8, ctx->stream));
        }
        ctx->tag_base = 0;
    }
    DecodeArgs a{};
    a.phases = (const DecodePhase *) m.d_phases; a.layer_vecs = (const DecodeLayerVec *) m.d_layer_vecs;
    a.wte = m.wte[0]; a.wpe = m.wpe; a.ln_f_g = m.ln_f_g; a.ln_f_b = m.ln_f_b; a.gelu_tab = ctx->d_gelu_tab;
    a.mem_k = mem_k; a.mem_v = mem_v;
    a.gx = m.gx; a.gq = m.gq; a.gk = m.gk; a.gv = m.gv; a.gatt = m.gatt; a.gff = m.gff; a.gscores = m.gscores; a.logits = m.glogits;
    a.tag_base = ctx->tag_base; a.ln_fallbacks = ctx->d_ln_fallbacks; a.timing = ctx->d_timing;
    a.E = m.n_embd; a.H = m.n_head; a.L = m.n_layer; a.block_size = m.block_size; a.n_past = n_past; a.token = token; a.lm_lo = lm_lo; a.lm_hi = lm_hi;
    a.token_ptr = d_token; a.n_vocab_in = m.n_in_vocab;
    a.inv_E = 1.0 / (double) m.n_embd;
    for (int i = 0; i < 6; i++) a.headstart[i] = ctx->headstart[i];
    a.timing_tid = ctx->timing_tid; a.poll_ns = ctx->poll_ns;
    const double es = m.wtype == W_Q4_0 ? 18.0 / 32.0 : m.wtype == W_F16 ? 2.0 : 4.0;
    const double E = m.n_embd, L = m.n_layer;
    g_next_bytes = (12.0 * L * E * E + (double)(lm_hi - lm_lo) * E) * es + 2.0 * L * (double)(n_past + 1) * E * 4.0 + 2.0 * L * E * 4.0 + (double)(lm_hi - lm_lo) * 4.0;   // SURVEY §8d B_tok
    g_next_flops = 2.0 * (12.0 * L * E * E + (double)(lm_hi - lm_lo) * E) + 4.0 * L * (double)(n_past + 1) * E;
    launch_decode_step(a, m.wtype, ctx->n_sm, ctx->stream);
    ctx->tag_base += (unsigned) decode_tags_per_step(m.n_layer);
    ctx->last_logits = m.glogits;
    *pos += 1;
}

bool gpt_eval(bark_context * ctx, GPTModel & m, const int32_t * tokens, int n, int * n_past, bool merge_ctx, float * logits_host, int lm_lo, int lm_hi,
              float * mem_k, float * mem_v) {
    if (!n_past) { fprintf(stderr, "%s: n_past is null\n", __func__); return false; }
    if (!mem_k || !mem_v) { mem_k = m.mem_k; mem_v = m.mem_v; }
    const int64_t t0 = now_us();
    Workspace & ws = ctx->ws;
    cudaStream_t s = ctx->stream;
    const int E = m.n_embd;
    int N = n;
    bool merge = false;
    clamp_lm(m, lm_lo, lm_hi);
    if (!tokens || n < 1 || n > 8 * 1024) { fprintf(stderr, "%s: bad token buffer (n = %d)\n", __func__, n); return false; }
    for (int i = 0; i < n; i++) if (tokens[i] < 0 || tokens[i] >= m.n_in_vocab) {      // the embedding gather is unchecked on the device
        fprintf(stderr, "%s: token id %d at position %d is outside the model's input vocabulary (%d)\n", __func__, tokens[i], i, m.n_in_vocab); return false;
    }
    if (*n_past > 0 && N == 1) {
        if (ctx->use_decode_kernel && m.decode_ok && *n_past + 1 <= m.block_size) {
            decode_step(ctx, m, tokens[0], nullptr, n_past, lm_lo, lm_hi, mem_k, mem_v);
            read_logits(ctx, m.glogits, lm_lo, lm_hi - lm_lo, logits_host);
            m.t_predict_us += now_us() - t0;
            return true;
        }
    } else if (merge_ctx && *n_past == 0) {
        if (N != 513) { fprintf(stderr, "%s: merged prompt must hold 256+256+1 ids (got %d)\n", __func__, N); return false; }
        N = 257; merge = true;                                                                                  // bark.cpp:1230-1233
    }
    if (N < 1 || *n_past + N > m.block_size) { fprintf(stderr, "%s: context overflow (n_past %d + %d > %d)\n", __func__, *n_past, N, m.block_size); return false; }
    memcpy(ctx->h_tok, tokens, (size_t) n * sizeof(int32_t));
    BARK_CUDA_CHECK(cudaMemcpyAsync(ws.tok, ctx->h_tok, (size_t) n * sizeof(int32_t), cudaMemcpyHostToDevice, s)); g_h2d_bytes += (size_t) n * sizeof(int32_t);
    gpt_embed_causal(m, ws.tok, N, *n_past, merge, ws.x, s);
    run_layers(ctx, m, N, LocalKV{mem_k, mem_v, (size_t) m.block_size * E, *n_past, true});
    output_head(ctx, m, ws.x + (size_t)(N - 1) * E, 1, m.lm_head[0], ws.logits);                                  // the last position only
    read_logits(ctx, ws.logits, 0, m.n_out_vocab, logits_host);
    *n_past += N;
    m.t_predict_us += now_us() - t0;
    return true;
}

// Output rows [lo, hi) of W as a matrix of their own.  Every output of a mat-mul is its own dot product, so the slice computes
// the same values as the full matrix.  (Few-row kernels only: the group-major copy is not sliced.)
static DMat output_rows(const DMat & W, int lo, int hi) {
    DMat d = W;
    d.n_out = hi - lo; d.p_gm = nullptr; d.p_rm = nullptr;
    const size_t nb = (size_t) W.K / 32, r = (size_t) lo;
    auto at = [](void * p, size_t bytes) { return p ? (void *)((unsigned char *) p + bytes) : nullptr; };
    if (W.type == W_F16 || W.type == W_F32) { d.p = at(W.p, r * W.Kp * (W.type == W_F16 ? 2 : 4)); return d; }
    d.p = at(W.p, r * nb * (W.type == W_Q8_0 ? 32 : 16));             // q4_0 nibble words / qx codes
    d.scales = at(W.scales, r * nb * 2); d.mins = at(W.mins, r * nb * 2); d.qh = at(W.qh, r * nb * 4);
    return d;
}

bool gpt_step_batch(bark_context * ctx, GPTModel & m, int B, float * const * slot_k, float * const * slot_v, const int32_t * tokens, const int * n_past,
                    int lm_lo, int lm_hi, float * d_logits) {
    const int64_t t0 = now_us();
    Workspace & ws = ctx->ws;
    cudaStream_t s = ctx->stream;
    const int D = m.n_embd / m.n_head;
    if (B < 1 || B > 8) { fprintf(stderr, "%s: %d rows (1 to 8)\n", __func__, B); return false; }
    if (D % 32 || D > 128) { fprintf(stderr, "%s: unsupported head size %d (need a multiple of 32, <= 128)\n", __func__, D); return false; }
    clamp_lm(m, lm_lo, lm_hi);
    int max_kv = 0;
    for (int b = 0; b < B; b++) {
        if (tokens[b] < 0 || tokens[b] >= m.n_in_vocab) { fprintf(stderr, "%s: token id %d of row %d is outside the model's input vocabulary (%d)\n", __func__, tokens[b], b, m.n_in_vocab); return false; }
        if (n_past[b] < 0 || n_past[b] + 1 > m.block_size) { fprintf(stderr, "%s: context overflow in row %d (n_past %d + 1 > %d)\n", __func__, b, n_past[b], m.block_size); return false; }
        max_kv = std::max(max_kv, n_past[b] + 1);
    }
    int32_t * h = ctx->batch.h_step, * d = ctx->batch.d_step;
    for (int b = 0; b < B; b++) { h[b] = tokens[b]; h[8 + b] = n_past[b]; }
    BARK_CUDA_CHECK(cudaMemcpyAsync(d, h, 16 * sizeof(int32_t), cudaMemcpyHostToDevice, s)); g_h2d_bytes += 16 * sizeof(int32_t);
    gpt_embed_causal(m, d, B, 0, false, ws.x, s, d + 8);
    run_layers(ctx, m, B, SlotKV{slot_k, slot_v, d + 8, max_kv});
    output_head(ctx, m, ws.x, B, output_rows(m.lm_head[0], lm_lo, lm_hi), d_logits, lm_lo);     // only the sampled window, as the decode kernel does
    m.t_predict_us += now_us() - t0;
    return true;
}

// One decode step whose input token is read from device memory (the previous step's sample): nothing to wait for on the
// host, so a whole window of steps is enqueued back to back.
bool gpt_decode_chained(bark_context * ctx, GPTModel & m, const int32_t * d_token, int * n_past, int lm_lo, int lm_hi) {
    if (!ctx->use_decode_kernel || !m.decode_ok || *n_past < 1) { fprintf(stderr, "%s: needs the persistent decode kernel and a filled KV cache\n", __func__); return false; }
    if (*n_past + 1 > m.block_size) { fprintf(stderr, "%s: context overflow (n_past %d + 1 > %d)\n", __func__, *n_past, m.block_size); return false; }
    clamp_lm(m, lm_lo, lm_hi);
    decode_step(ctx, m, 0, d_token, n_past, lm_lo, lm_hi, m.mem_k, m.mem_v);
    return true;
}

bool fine_embed(bark_context * ctx, const int32_t * in_buffer, int nn, int row0, int rows, const char * fn) {
    const GPTModel & m = ctx->fine;
    Workspace & ws = ctx->ws;
    if (nn < 1 || nn > 7) { fprintf(stderr, "%s: codebook index %d out of range\n", fn, nn); return false; }
    for (int i = 0; i < (nn + 1) * 1024; i++) if (in_buffer[i] < 0 || in_buffer[i] >= m.n_in_vocab) {
        fprintf(stderr, "%s: code %d (codebook %d, frame %d) is outside the fine model's input vocabulary (%d)\n", fn, in_buffer[i], i / 1024, i % 1024, m.n_in_vocab); return false;
    }
    memcpy(ctx->h_tok, in_buffer, (size_t) 8 * 1024 * sizeof(int32_t));
    BARK_CUDA_CHECK(cudaMemcpyAsync(ws.tok, ctx->h_tok, (size_t) 8 * 1024 * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream)); g_h2d_bytes += (size_t) 8 * 1024 * sizeof(int32_t);
    gpt_embed_fine(m, ws.tok, nn, ws.x, ctx->stream, row0, rows);
    return true;
}

bool fine_eval(bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_host) {
    if (ctx->fast_mode) return fine_eval_fast(ctx, in_buffer, nn, logits_host);
    GPTModel & m = ctx->fine;
    Workspace & ws = ctx->ws;
    const int64_t t0 = now_us();
    if (!fine_embed(ctx, in_buffer, nn, 0, 1024, __func__)) return false;
    run_layers(ctx, m, 1024, LocalKV{ws.kbuf, ws.vbuf, 0, 0, false});
    output_head(ctx, m, ws.x, 1024, m.lm_head[nn - 1], ws.logits);                                               // n_codes_given = 1 (bark.cpp:61,1573)
    read_logits(ctx, ws.logits, 0, (size_t) 1024 * m.n_out_vocab, logits_host);
    m.t_predict_us += now_us() - t0;
    return true;
}

// FAST MODE: the same pass on the tensor cores (fast_kernels.cu): LayerNorm -> f16, wgmma GEMMs with fused epilogues, flash-style
// attention.  Same inputs / outputs as fine_eval; logits agree with the reference to f16-operand accuracy, not bit for bit.
bool fine_eval_fast(bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_host) {
    GPTModel & m = ctx->fine;
    const int64_t t0 = now_us();
    Workspace & ws = ctx->ws;
    cudaStream_t s = ctx->stream;
    const int E = m.n_embd, H = m.n_head, N = 1024, n_sm = ctx->n_sm_total;
    if (!fine_embed(ctx, in_buffer, nn, 0, N, __func__)) return false;
    for (int il = 0; il < m.n_layer; il++) {
        const GPTLayer & L = m.layers[(size_t) il];
        fast_layernorm(ws.x, N, E, L.ln_1_g, L.ln_1_b, ctx->f_a16, s);
        FastEpi qkv; qkv.mode = FEPI_QKV16; qkv.out16 = ctx->f_qk16; qkv.ldo = 2 * E; qkv.vt = ctx->f_vt16; qkv.vt_ld = N; qkv.v_col0 = 2 * E;
        if (!fast_gemm(ctx->f_a16, E, (const __half *) L.c_attn.p_rm, E, N, 3 * E, E, qkv, n_sm, 0, s)) return false;
        if (!fast_attention(ctx->f_qk16, 2 * E, E, ctx->f_vt16, N, E, H, ctx->f_att16, s)) return false;
        FastEpi res; res.mode = FEPI_RESID; res.out32 = ws.x; res.ldo = E;
        if (!fast_gemm(ctx->f_att16, E, (const __half *) L.c_proj.p_rm, E, N, E, E, res, n_sm, 0, s)) return false;
        fast_layernorm(ws.x, N, E, L.ln_2_g, L.ln_2_b, ctx->f_a16, s);
        FastEpi ge; ge.mode = FEPI_GELU16; ge.out16 = ctx->f_h16; ge.ldo = 4 * E;
        if (!fast_gemm(ctx->f_a16, E, (const __half *) L.fc.p_rm, E, N, 4 * E, E, ge, n_sm, 0, s)) return false;
        if (!fast_gemm(ctx->f_h16, 4 * E, (const __half *) L.proj.p_rm, 4 * E, N, E, 4 * E, res, n_sm, 0, s)) return false;
    }
    fast_layernorm(ws.x, N, E, m.ln_f_g, m.ln_f_b, ctx->f_a16, s);
    FastEpi st; st.mode = FEPI_F32; st.out32 = ws.logits; st.ldo = m.n_out_vocab;
    if (!fast_gemm(ctx->f_a16, E, (const __half *) m.lm_head[nn - 1].p_rm, E, N, m.n_out_vocab, E, st, n_sm, 0, s)) return false;
    ctx->last_logits = ws.logits;
    read_logits(ctx, ws.logits, 0, (size_t) N * m.n_out_vocab, logits_host);
    m.t_predict_us += now_us() - t0;
    return true;
}

}  // namespace bark
