// Host-callable launchers of the GPT kernels (gpt_kernels.cu, decode_kernels.cu).
#pragma once
#include "model.h"

namespace bark {

enum EpiMode : int { EPI_STORE = 0, EPI_RESID = 1, EPI_GELU_ACT = 2, EPI_QKV = 3 };

struct MatmulEpilogue {
    int mode = EPI_STORE;
    float * out = nullptr; int ldo = 0;              // STORE / RESID target ([m][ldo]); QKV: q rows with ldo = E
    float * k_out = nullptr, * v_out = nullptr;      // QKV: K/V rows (KV cache slot of the first new position, or the fine model's buffers)
    // row-sharded fine pass (shard.cu): the same K/V rows are also stored into the other GPUs' buffers over NVLink (peer pointers),
    // so the all-gather of K and V is the mat-mul's own epilogue
    int n_peer = 0; float * k_peer[7] = {nullptr}, * v_peer[7] = {nullptr};
    void * act_out = nullptr; int act_wt = 0, act_Kp = 0;   // GELU_ACT: operand for the following mul_mat (act_Kp = its group stride)
    const __half * gelu_tab = nullptr;
};

void permute_to_li(const void * src_rowmajor, void * dst_li, int n_out, int K, WType t, cudaStream_t s);
void permute_to_gm(const void * src_rowmajor, void * dst_gm, int n_out, int o_pad, int K, WType t, cudaStream_t s);

// d_pos (device, optional): row r sits at position d_pos[r] instead of n_past + r (the rows of a batched decode step)
void gpt_embed_causal(const GPTModel & m, const int32_t * d_tok, int N, int n_past, bool merge, float * x, cudaStream_t s, const int32_t * d_pos = nullptr);
void gpt_embed_fine(const GPTModel & m, const int32_t * d_ids, int nn, float * x, cudaStream_t s, int row0 = 0, int rows = 1024);   // rows [row0, row0 + rows) of the window

// `Kp` of the activation operands below is the GROUP STRIDE of the group-major layout (elements), not a row length
void layernorm_act(const float * x, int rows, int E, const float * g, const float * b, void * act, WType wt, int Kp,
                   unsigned * fallback_counter, cudaStream_t s);

// q8 activation operand of the quantised mat-muls, owned by the caller: int8 [rows][K], f32 block scales d and q8_1 block sums s
// [rows][K/32] (sums for q4_1 / q5_1 only)
struct Q8Scratch { int8_t * q = nullptr; float * d = nullptr, * s = nullptr; };

// q8: the scratch a quantised W needs (null for f32 / f16 weights).  f32 / f16 W: below 16 rows the few-row kernel (lane_matmul_rows,
// on W's row-major LI copy), else lane_gemm_tiled (on its group-major copy).  Returns the kernel launched: kLaneRowsVariant for the
// few-row kernel, else lane_gemm_tiled's block-tile variant; 0 for quantised W.
constexpr int kLaneRowsVariant = 3;
int  lane_matmul(const DMat & W, const void * act, int act_gs, int rows, const MatmulEpilogue & ep, const Q8Scratch * q8, cudaStream_t s);
// The few-row kernel at any row count: lane_matmul_kernel<T, 1> for one row, <T, 8> over 8-row blocks otherwise; f32 / f16 W in the
// row-major LI layout (W.p, W.Kp), activations group-major.
void lane_matmul_rows(const DMat & W, const void * act, int act_gs, int rows, const MatmulEpilogue & ep, cudaStream_t s);

// Multi-row attention (gemm_kernels.cu): N query rows Q[N][E] against n_kv <= 1024 key / value rows Kc, Vc [n_kv][E], H heads of 32, 64,
// 96 or 128; causal masks key k for query q when k > n_past + q.  Result -> activation operand for c_proj.
// Enough rows to give every SM a (head, 32-query) tile: attn_fused_kernel, scores in shared memory.  Up to attn_tiled_max_rows(H, SMs)
// rows: three kernels that pass the scores through `scores` (H * N * n_kv floats).  Both give the same bits; path forces one (tests).
enum AttnPath : int { ATTN_AUTO = 0, ATTN_FUSED = 1, ATTN_TILED = 2 };
int  attn_tiled_max_rows(int H, int n_sm);
void attention(const float * Q, const float * Kc, const float * Vc, int N, int n_kv, int n_past, int E, int H, bool causal,
               float * scores, void * act, WType wt, int Kp, cudaStream_t s, AttnPath path = ATTN_AUTO);
// softmax_row on each of `rows` rows of n <= 1024 floats, in place, one warp per row; replays counts the sequential replays
void softmax_rows(float * S, int rows, int n, unsigned * replays, cudaStream_t s);

// Decode attention for B <= 8 rows of different sequences (batched step): row b's query is Q[b], its new K / V rows are staged in
// Kst[b] / Vst[b] and are appended to its cache (kv.k[b], kv.v[b]: the layer's [block_size][E] slab) at position d_pos[b]; it attends
// over d_pos[b] + 1 keys.  max_kv = the largest of those.  scores: B * H * max_kv floats.  Result -> activation operand, as attention()
// leaves it.
struct BatchKV { float * k[8], * v[8]; };
void attention_batch(const float * Q, const float * Kst, const float * Vst, const BatchKV & kv, const int32_t * d_pos, int B, int max_kv, int E, int H,
                     float * scores, void * act, WType wt, int Kp, cudaStream_t s);

// ---- q4_0 weights (q4_kernels.cu) ---------------------------------------------------------------------------------
void q4_split(const void * raw_blocks, size_t n_blocks, void * qs, void * scales, cudaStream_t s);
void q4_matmul(const DMat & W, const void * act_f32, int ld_act, int rows, const MatmulEpilogue & ep, const Q8Scratch * q8, cudaStream_t s);

// ---- q4_1 / q5_0 / q5_1 / q8_0 weights (qx_kernels.cu) ---------------------------------------------------------------------------
bool   qx_supported(WType t);
size_t qx_block_bytes(WType t);
void   qx_split(const void * raw_blocks, size_t n_blocks, WType t, void * qs, void * qh, void * d, void * m, cudaStream_t s);
// quantize_q8x_kernel: f32 rows x [rows][ldx] -> q8 blocks, K per row, into q / d, and the block sums into s unless it is null
void   quantize_q8(const float * x, int ldx, int rows, int K, int8_t * q, float * d, float * s, cudaStream_t stream);
void   qx_embed_causal(const GPTModel & m, const int32_t * d_tok, int N, int n_past, bool merge, float * x, cudaStream_t s, const int32_t * d_pos);
void   qx_embed_fine(const GPTModel & m, const int32_t * d_ids, int nn, float * x, cudaStream_t s);
void   qx_matmul(const DMat & W, const void * act_f32, int ld_act, int rows, const MatmulEpilogue & ep, const Q8Scratch * q8, cudaStream_t s);

// ---- register-tiled multi-row kernels (gemm_kernels.cu) ------------------------------------------------------------
// W needs its group-major copy with o_pad a multiple of kGemmOPad (the widest block tile), the activation operand a row capacity
// (act_gs / 128) that is a multiple of 32 (the tallest).  variant: 0 = the block tile picked for the weight type, 1 = 32 x 16 (8 warps,
// two CTAs per SM), 2 = 32 x 32 (16 warps, one CTA per SM).  Returns the variant launched, 0 if it does not exist.
constexpr int kGemmOPad = 32;
int lane_gemm_tiled(const DMat & W, const void * act, int act_gs, int rows, const MatmulEpilogue & ep, cudaStream_t s, int variant = 0);

// ---- fast mode (fast_kernels.cu, BARK_B200_MODE=fast): wgmma GEMM + flash-style attention for the dense passes -------------------
enum { FEPI_F32 = 0, FEPI_RESID = 1, FEPI_GELU16 = 2, FEPI_QKV16 = 4 };
struct FastEpi {
    int mode = FEPI_F32;
    float * out32 = nullptr; __half * out16 = nullptr; int ldo = 0;      // row-major targets
    __half * vt = nullptr; int vt_ld = 0, v_col0 = 0;                    // QKV16: columns >= v_col0 are written transposed, vt[(n - v_col0) * vt_ld + m]
};
// bn: 0 = the cost model's tile width, else 64 / 128 / 256 forced.  Returns the tile width launched, 0 on failure.
int  fast_gemm(const __half * A, int lda, const __half * W, int ldw, int M, int N, int K, const FastEpi & ep, int n_sm, int bn, cudaStream_t s);
bool fast_attention(const __half * qk, int ldq, int k_col0, const __half * vt, int n, int E, int H, __half * out, cudaStream_t s);
void fast_layernorm(const float * x, int rows, int E, const float * g, const float * b, __half * out, cudaStream_t s);
// [n_out][K] weights of type t (f32, or q4_0 / q4_1 / q5_0 / q5_1 / q8_0 blocks as the file stores them), K % 32 == 0 -> dst [n_out][K]
// f16, the W operand of fast_gemm; *non_finite (device) grows by the number of inf / NaN results
void fast_convert(const void * src, WType t, int n_out, int K, __half * dst, int * non_finite, cudaStream_t s);

// ---- persistent decode step (decode_kernels.cu) -----------------------------------------------------------------
constexpr int kDecodeReplicas = 8;        // copies of each all-to-all exchange vector (gx, gq, gatt, gff): CTA c reads copy c % 8
struct DecodePhase { const void * w; int n_out, row_bytes, K, pad; const void * ws; };   // one streamed matrix: LI rows (f32 / f16), or q4_0 nibble words (16 B per block) with f16 block scales in ws
struct DecodeLayerVec { const float * ln_1_g, * ln_1_b, * ln_2_g, * ln_2_b; };
struct DecodeArgs {
    const DecodePhase * phases;          // [4L + 1]: per layer c_attn, c_proj, c_fc, mlp/c_proj; then lm_head
    const DecodeLayerVec * layer_vecs;   // [L]
    const void * wte; const float * wpe; const float * ln_f_g, * ln_f_b; const __half * gelu_tab;
    float * mem_k, * mem_v;              // f32 KV cache [L][block_size][E]
    // cross-CTA exchange vectors in L2: 8-byte {float value, u32 epoch} words
    unsigned long long * gx, * gq, * gk, * gv, * gatt, * gff, * gscores;
    float * logits;
    unsigned tag_base; unsigned * ln_fallbacks;
    unsigned long long * timing;         // optional [256][32] globaltimer stamps (debug, decode_kernels.cu tstamp)
    int E, H, L, block_size, n_past, token, lm_lo, lm_hi;
    const int32_t * token_ptr; int n_vocab_in;   // token_ptr != null: read the input token from device memory (written by sample_rows_kernel), clamped to the vocabulary
    double inv_E;                        // 1.0 / E (double), for the division-free LayerNorm decision
    unsigned headstart[6];               // head start (ns) before the first poll of each exchange: q, att (CTAs without a soft_max tile), x1, ff, x2, scores
    int timing_tid; unsigned poll_ns;    // debug: stamping thread; back-off between polls of the tagged words (ns)
};
int  decode_tags_per_step(int n_layer);
void launch_decode_step(const DecodeArgs & args, WType wt, int n_sm, cudaStream_t s);
// the decode kernels' LayerNorm (op 0) or soft_max (op 1) on `rows` rows of n <= 1024 floats, one CTA per row (tests):
// counters[0] / counters[1] count the LayerNorm / soft_max rows that took the sequential replay
void decode_rows(int op, const float * x, int rows, int n, const float * g, const float * b, float * out, unsigned * counters, cudaStream_t s);
// the decode kernels' q4_0 pieces on one f32 row x [K] (tests): quantize_act_q8, then row_dot_q4 over n_out rows (qs / scales as q4_split
// leaves them) through the per-op epilogue ep (row 0), in one CTA; staged: the rows are copied into shared memory first (row_dot_q4<true>),
// else read from global memory.  q_out [K] / d_out [K/32]: the q8 operand.  K <= 4096.
void decode_q4_rows(bool staged, const float * x, int K, const void * qs, const void * scales, int n_out, const MatmulEpilogue & ep, int8_t * q_out,
                    float * d_out, cudaStream_t s);

}  // namespace bark
