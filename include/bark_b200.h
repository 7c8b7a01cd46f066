/* bark_b200.h — additive C entry points of libbark_b200 (nothing here exists in the reference header).
 *
 * They expose, through the same C-ABI shared library, the per-call pieces the reference keeps file-static,
 * so that parity tests and the benchmark can drive and time one step of the hot path with HOST buffers:
 *
 *   bark_b200_gpt_eval ........ one causal GPT evaluation  == bark_eval_encoder_internal      (bark.cpp:1586-1643)
 *   bark_b200_fine_eval ....... one fine pass              == bark_eval_fine_encoder_internal (bark.cpp:1907-1959)
 *   bark_b200_encodec_decode .. codes -> waveform          == encodec_decompress_audio        (encodec.cpp/encodec.cpp:902-924)
 *   bark_b200_sample .......... gpt_sample on the context RNG                                 (bark.cpp:249-270)
 *   bark_b200_sample_rows ..... the same for `rows` logit rows, on the device sampler the stages use (host replay of rows it cannot decide)
 *   bark_b200_forward_* ....... extern "C" names for bark_forward_{text,coarse,fine}_encoder  (bark.cpp:1703,1865,2061)
 *   bark_b200_tokenize ........ bark_tokenize_input                                           (bark.cpp:622-662)
 *
 * plus device selection for one-context-per-GPU batching (SURVEY.md §8e): bark_context_params must keep the
 * reference layout, so the device is chosen by bark_b200_set_device() or the BARK_B200_DEVICE environment
 * variable before bark_load_model.
 */
#pragma once
#include "bark.h"

#ifdef __cplusplus
extern "C" {
#endif

BARK_API void bark_b200_set_device(int cuda_device);                       /* applies to subsequent bark_load_model calls */
BARK_API const char * bark_b200_version(void);

/* which: 0 semantic, 1 coarse.  Host pointers.  *n_past advances exactly like the reference (by 257 for the merged prompt). */
BARK_API int  bark_b200_gpt_eval(struct bark_context * ctx, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out);
/* in_buffer: [8][1024] ids; nn: codebook being predicted (2..7); logits_out: [1024][n_out_vocab] */
BARK_API int  bark_b200_fine_eval(struct bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_out);
/* codes: [8][n_frames]; returns number of samples (320 * n_frames), copies min(n, out_cap) floats to out (may be NULL) */
BARK_API int  bark_b200_encodec_decode(struct bark_context * ctx, const int32_t * codes, int n_frames, float * out, int out_cap);
BARK_API int  bark_b200_sample(struct bark_context * ctx, int which, const float * logits, int n, float temp, float * eos_p);
BARK_API int  bark_b200_sample_rows(struct bark_context * ctx, const float * logits /*[rows][n], host*/, int n, int rows, float temp, int32_t * tokens_out,
                                     float * eos_p_out /*[rows] or NULL*/);   /* returns the number of rows replayed on the host, <0 on error */
BARK_API void bark_b200_reseed(struct bark_context * ctx, uint32_t seed);
BARK_API void bark_b200_tokenize(struct bark_context * ctx, const char * text, int32_t * out513);

BARK_API bool bark_b200_forward_text_encoder(struct bark_context * ctx, int n_threads);
BARK_API bool bark_b200_forward_coarse_encoder(struct bark_context * ctx, int n_threads);
BARK_API bool bark_b200_forward_fine_encoder(struct bark_context * ctx, int n_threads);

/* stage: 0 semantic [n], 1 coarse [T][2], 2 fine [T][8], 3 prompt [513].  Returns the element count. */
BARK_API int  bark_b200_get_tokens(struct bark_context * ctx, int stage, int32_t * out, int cap);
BARK_API void bark_b200_set_tokens(struct bark_context * ctx, int stage, const int32_t * in, int n);
/* per_model9: {predict_us, sample_us, n_sample} x {semantic, coarse, fine} */
BARK_API void bark_b200_get_stats(struct bark_context * ctx, struct bark_statistics * out, int64_t * per_model9);
BARK_API void bark_b200_get_hparams(struct bark_context * ctx, int which, int32_t * out10);
BARK_API unsigned long long bark_b200_kernel_launches(void);               /* kernels launched by this library so far */
BARK_API unsigned bark_b200_layernorm_fallbacks(struct bark_context * ctx); /* LayerNorm rows replayed sequentially (DESIGN.md) */

/* measurement hooks used by bench.py */
BARK_API void bark_b200_profile_enable(int on);                            /* CUDA-event timing of every kernel launch; clears previous records */
BARK_API int  bark_b200_profile_report(char * buf, int cap);               /* JSON {kernel: {launches, ms, work}}; returns bytes needed */
BARK_API void bark_b200_io_counters(unsigned long long * h2d_bytes, unsigned long long * d2h_bytes, int reset);
/* with BARK_B200_DECODE_TIMING=1 in the environment at load: %globaltimer stamps [256][32] of the last decode step (rows 0..L: the
 * stamping thread of CTA 0 per layer; rows 64 + cta: every CTA at layer 5; slot meaning in tools/decode_timing.py) */
BARK_API int  bark_b200_decode_timing(struct bark_context * ctx, unsigned long long * out, int n);


/* ROW-SHARDED FINE STAGE (BASELINE configs[4]; csrc/shard.cu): one process per GPU; every rank loads the same file and the same coarse
 * tokens, evaluates rows [rank * 1024 / world, ...) of each fine pass, stores its K / V rows into the peers' buffers over NVLink from
 * the QKV mat-mul's epilogue, and ends with the full fine token array, bit-identical to the single-GPU run.
 *   1. bark_b200_shard_init(ctx, rank, world, handle64)   -> 64-byte CUDA IPC handle of this rank's exchange buffer
 *   2. (caller all-gathers the handles, e.g. torch.distributed)
 *   3. bark_b200_shard_connect(ctx, all_handles)           -> maps the peers' buffers; bark_b200_forward_fine_encoder is sharded from here on */
BARK_API int  bark_b200_shard_init(struct bark_context * ctx, int rank, int world, void * handle_out);
BARK_API int  bark_b200_shard_connect(struct bark_context * ctx, const void * all_handles);
BARK_API unsigned long long bark_b200_shard_nvlink_bytes(struct bark_context * ctx, int reset);

/* BATCHED GENERATION: up to 8 prompts per context, their semantic and coarse decode steps evaluated together (one pass over the
 * weights per step for all of them).  Item i's prompt, semantic, coarse and fine ids and waveform are bit-identical to a fresh
 * bark_load_model(path, params, seeds[i]) followed by bark_generate_audio(ctx, texts[i]): they do not depend on n, on i's place in the
 * batch or on the other items.  The context's own generation state is not touched: its RNG, the ids bark_b200_get_tokens returns
 * and what bark_get_audio_data returns.  ctx->params applies to every item; the progress callback is not called during a batch.
 * Statistics: t_eval_us and the stage times are the batch's wall time, the n_sample_* counts are summed over the items.
 * Per-item KV caches (f32, 151 MB per item for bark-small, 402 MB for bark-large) are allocated on the first batch of n items, grown
 * by a larger one and freed by bark_free.
 *   bark_b200_generate_batch ... 1 <= n <= 8 prompts with their seeds; false (message on stderr) for anything else, a null text, or a
 *                                context whose fine stage is sharded (bark_b200_shard_connect)
 *   bark_b200_batch_audio ...... samples of item i of the last successful batch; copies min(n, cap) to out (may be NULL); -1 if no such item.
 *                                A failed batch leaves those results and the context's statistics as they were.
 *   bark_b200_batch_tokens ..... ids of item i; stage as bark_b200_get_tokens (0 semantic, 1 coarse [T][2], 2 fine [T][8], 3 prompt)
 * Test hooks: the batched step on the slots' KV caches (slot 0..7, which: 0 semantic, 1 coarse, host buffers):
 *   bark_b200_gpt_eval_slot .... bark_b200_gpt_eval on slot's cache instead of the model's own
 *   bark_b200_gpt_step_batch ... one decode step of B distinct slots: row r feeds tokens[r] at position n_past[r] through slots[r]'s
 *                                cache; logits_out [B][n_out_vocab]; n_past[r] advances by one */
BARK_API bool bark_b200_generate_batch(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds, int n, int n_threads);
BARK_API int  bark_b200_batch_audio(struct bark_context * ctx, int i, float * out, int cap);
BARK_API int  bark_b200_batch_tokens(struct bark_context * ctx, int i, int stage, int32_t * out, int cap);
BARK_API int  bark_b200_gpt_eval_slot(struct bark_context * ctx, int which, int slot, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out);
BARK_API int  bark_b200_gpt_step_batch(struct bark_context * ctx, int which, int B, const int32_t * slots, const int32_t * tokens, int * n_past, float * logits_out);

/* FAST MODE (BARK_B200_MODE=fast in the environment at load; opt-in, NOT bit-identical to the reference): the fine model's
 * 1024-row passes (bark.cpp:1416-1584) run as wgmma tensor-core GEMMs + flash-style attention (csrc/fast_kernels.cu).
 * The two kernel hooks below run on host buffers without a context, for the numerics tests:
 *   bark_b200_fast_gemm ....... A[M][K] (f16 bits) * W[N][K]^T (f16 bits), K % 64 == 0, through the fine pass's epilogue `epilogue`:
 *                                 0 F32     C = f32 [M][N]
 *                                 1 RESID   C = f32 [M][N], holds the residual on entry and residual + A W^T on return
 *                                 2 GELU16  C = f16 [M][N] (bits), GELU of the product
 *                                 4 QKV16   N % 6 == 0; C = f16 [M][2N/3] (columns < 2N/3), then f16 [N/3][M] (columns >= 2N/3, transposed)
 *                               bn: 0 = the tile width the cost model picks, 64 / 128 / 256 = that width forced.
 *                               Returns the tile width that ran, 0 on failure, -1 if a store landed in the guard bands around the output.
 *   bark_b200_fast_attention .. out[n][E] (f16 bits) = soft_max(Q K^T / 8) V per 64-wide head, non-causal, n % 128 == 0 */
BARK_API int  bark_b200_fast_mode(struct bark_context * ctx);              /* 1 if this context runs the fast fine passes */
BARK_API int  bark_b200_fast_gemm(const uint16_t * A, const uint16_t * W, void * C, int M, int N, int K, int epilogue, int bn);
BARK_API int  bark_b200_fast_attention(const uint16_t * q, const uint16_t * k, const uint16_t * v, uint16_t * out, int n, int E, int H);

/* Parity-path attention on host buffers without a context (tests, tools/attn_bench.py): out[N][E] = soft_max(mask(Q K^T / sqrt(E/H))) V
 * per head, bit-identical to the reference's ggml graph, for q [N][E], k / v [n_kv][E] f32, n_kv <= 1024, head size E/H in
 * {32, 64, 96, 128}.  causal != 0 masks key j for query i when j > n_past + i.  path: 0 = the kernels the library picks for this
 * shape, 1 = the fused kernel (scores in shared memory), 2 = the three-kernel path for few rows (N <= 32 * (ceil(SMs / H) - 1)).
 * Returns 1 on success, 0 on failure. */
BARK_API int  bark_b200_parity_attention(const float * q, const float * k, const float * v, float * out, int N, int n_kv, int n_past, int E, int H, int causal,
                                         int path);

/* Parity-path row reductions on host buffers without a context (tests).  op 0: LayerNorm (eps 1e-5, g required, b may be NULL), the f32
 * value before any operand rounding; op 1: soft_max, the probability as its consumers form it.  impl 0: the multi-row kernels
 * (layernorm_act_kernel / softmax_row), impl 1: the decode kernels' device functions (block_layernorm / softmax_exp_rcp) in a
 * one-CTA-per-row wrapper of 512 threads.  x, out: [rows][n] f32 row-major; n <= 1024.  *replays: number of bracket failures that took
 * the sequential replay.  Returns 1 on success, 0 on invalid arguments or failure. */
BARK_API int  bark_b200_parity_rows(int op, int impl, const float * x, int rows, int n, const float * g, const float * b, float * out, unsigned * replays);

/* The device sampler on host rows without a context (tests): gpt_sample for each of `rows` logit rows of n (packed [rows][n] f32) with
 * the uniform draw u[r] given (u may be NULL when temp == 0, where it is not used).  Runs sample_rows_kernel with `threads` threads per
 * row (0: as the library picks, 1024 for a single row and 256 otherwise; or 256, or 1024), then replays every row the kernel flags on
 * the host with the reference's sequence, as the library does.  tokens: the final tokens; device_tokens: the kernel's tokens before the
 * replay; flags: 1 where the kernel could not prove its decision; eos_p: the probability of the last logit.  2 <= n, n * 4 <= 64 KB,
 * 1 <= rows <= 1024, temp finite and >= 0, every u in [0, 1).  Returns the number of replayed rows, or -1 on invalid arguments or failure. */
BARK_API int  bark_b200_sample_given_u(const float * logits, int n, int rows, float temp, const double * u, int threads, int32_t * tokens,
                                       int32_t * device_tokens, int32_t * flags, float * eos_p);

/* Parity-path tiled GEMM on host buffers without a context (tests, tools/gemm_bench.py): C = A W^T with every output the reference's
 * vec_dot of its two rows, for A [M][K] and W [N][K] of wtype 0 (f32) or 1 (f16 bits), K % 32 == 0, through the multi-row passes'
 * epilogue `epilogue`:
 *   0 STORE     C = f32 [M][N]
 *   1 RESID     C = f32 [M][N], holds the residual on entry and residual + A W^T on return
 *   2 GELU_ACT  C = [M][N] in wtype: GELU of the product through gelu_tab (65536 f16 entries), as the next mat-mul's operand holds it
 *   3 QKV       N % 3 == 0; C = f32 Q [M][N/3], then K [M][N/3], then V [M][N/3]
 * variant: 0 = the block tile the library picks, 1 = 32 x 16 outputs (8 warps, two CTAs per SM), 2 = 32 x 32 (16 warps, one CTA
 * per SM).  Returns the variant that ran, 0 on failure or invalid arguments, -1 if a store landed in the guard bands around the output. */
BARK_API int  bark_b200_parity_gemm(const void * A, const void * W, void * C, int M, int N, int K, int wtype, int epilogue, int variant,
                                    const uint16_t * gelu_tab);

#ifdef __cplusplus
}
#endif
