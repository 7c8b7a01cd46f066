// bark_context: everything one generation needs, owned by bark_load_model / bark_free.
// Host control plane in C++ (like the reference's bark.cpp:133-164), all tensors in HBM.
#pragma once
#include "../../include/bark.h"
#include "model.h"

#include <map>
#include <random>
#include <string>
#include <vector>

// row-sharded fine stage (shard.cu): this rank's IPC-exported buffer and the peers' mapped ones
struct ShardState {
    bool on = false; int rank = 0, world = 1;
    unsigned char * local = nullptr, * peer[8] = {nullptr};
    unsigned epoch = 0; unsigned * d_err = nullptr;
    unsigned long long nvlink_bytes = 0;             // bytes this rank stored into peer memory (K / V rows, sampled ids)
};

// What one generation reads and produces: its RNG, its token streams and its waveform.  The context holds one (bark.h's
// single-prompt calls); every item of a batch (bark_b200_generate_batch) holds its own, so a batch leaves the context's untouched.
struct Generation {
    std::mt19937 rng;                                // seeded once at load (bark.cpp:1179), or per batch item
    std::vector<int32_t> tokens;                     // 513 prompt ids
    std::vector<int32_t> semantic_tokens;
    std::vector<int32_t> coarse_tokens;              // [T][2] flattened
    std::vector<int32_t> fine_tokens;                // [T][8] flattened
    std::vector<float> audio;
};

// Batched generation (bark_api.cu): one f32 KV cache [L][block_size][E] per item and causal model, allocated on the first batch and
// grown when a later one has more items; the [8][n_out] logits of the batched step; the step's ids and positions (device + pinned).
struct BatchSlots {
    int cap = 0;
    float * k[2][8] = {}, * v[2][8] = {};            // [semantic / coarse][slot]
    float * d_logits = nullptr;                      // [8][max n_out of the causal models]
    int32_t * d_step = nullptr, * h_step = nullptr;  // [0, 8): input ids, [8, 16): positions (n_past) of the step's rows
    std::vector<Generation> results;                 // the last batch's items (bark_b200_batch_audio / bark_b200_batch_tokens)
};

struct bark_context {
    int device = 0;
    cudaStream_t stream = nullptr;

    bark::GPTModel semantic, coarse, fine;
    bark::CodecModel codec;
    std::map<std::string, int32_t> token_to_id;      // WordPiece vocabulary (bark.cpp:664-690)

    __half * d_gelu_tab = nullptr;                   // 65536-entry table, ggml.c:3795-3810
    unsigned * d_ln_fallbacks = nullptr;             // [0] LayerNorm rows, [1] soft_max rows replayed sequentially
    unsigned tag_base = 0;                           // epoch counter of the decode kernel's tagged exchanges (advances 6*L per token)
    int n_sm = 0, n_sm_total = 0; bool use_decode_kernel = true;   // n_sm: CTAs of the persistent decode kernel (knob); n_sm_total: SMs of the device
    bool kv_reuse = true; unsigned long long n_kv_reused = 0;   // coarse windows start from the cached prefix (bark_api.cu run_coarse)
    // decode-kernel knobs (BARK_B200_DECODE_TIMING_TID / BARK_B200_POLL_NS / BARK_B200_HEADSTART); defaults:
    // 40 ns back-off between polls, 500 ns head start for the two residual exchanges
    bool decode_cluster = false;                     // BARK_B200_DECODE=cluster: the decode step inside one 16-CTA cluster (decode_kernels.cu) where the model fits
    unsigned headstart[6] = {0, 2000, 500, 400, 500, 0};   // BARK_B200_HEADSTART=q:att:x1:ff:x2:scores (ns): sleep before the first poll of each exchange
    int timing_tid = 0; unsigned poll_ns = 40;
    unsigned long long * d_timing = nullptr;         // optional phase timestamps of the decode kernel (BARK_B200_DECODE_TIMING=1)

    // BARK_B200_MODE=fast: the fine model's passes run on the tensor cores (fast_kernels.cu); not bit-identical to the reference
    bool fast_mode = false;
    __half * f_a16 = nullptr, * f_h16 = nullptr, * f_qk16 = nullptr, * f_vt16 = nullptr, * f_att16 = nullptr;   // [1024][E], [1024][4E], [1024][2E], [E][1024], [1024][E]

    ShardState shard;

    bark::Workspace ws;
    void * d_q8_sums = nullptr;                       // experimental q4_1 / q5_1: q8_1 block sums s = f16(d * sum(q))
    void * d_q8 = nullptr, * d_q8_scales = nullptr;  // q4_0 models: q8_0 activation operand (int8 [rows][4E], f32 scales [rows][4E/32])
    const float * last_logits = nullptr;             // device logits of the latest gpt_eval / fine_eval
    double * d_u = nullptr, * h_u = nullptr;         // device sampling: uniforms, tokens, flags, eos probabilities (1024 rows)
    int32_t * d_stok = nullptr, * h_stok = nullptr, * d_sflags = nullptr, * h_sflags = nullptr;
    float * d_seos = nullptr, * h_seos = nullptr;
    int32_t * d_feed = nullptr;                      // token handed from sample_rows_kernel to the next decode step
    bool sample_on_device = true; long long n_sample_host_replays = 0;
    int debug_flag_every = 0; long long n_sample_calls = 0;   // BARK_B200_SAMPLE_FLAG_EVERY=k: force every k-th sample through the host replay (tests)
    float * h_logits = nullptr;                      // pinned, max(n_out) or 1024*fine_vocab
    int32_t * h_tok = nullptr;                       // pinned, 8*1024 ids

    // codec scratch
    float * c_buf[3] = {nullptr, nullptr, nullptr}; size_t c_cap = 0;   // ping-pong activations (floats)
    float * c_gi = nullptr;                                            // LSTM input projections
    float * c_hbuf = nullptr; unsigned * c_counter = nullptr;          // LSTM hidden-state exchange + grid barrier counter
    int32_t * d_codes = nullptr;

    Generation gen;                                  // the bark.h calls' generation state
    BatchSlots batch;

    bark_context_params params;
    bark_statistics stats{};

    std::vector<void *> device_allocs;               // everything cudaMalloc'ed for this context
};

namespace bark {

// loader.cu
bool load_model_file(const std::string & path, bark_context * ctx);
void * ctx_alloc(bark_context * ctx, size_t bytes);

// gpt_forward.cu — one evaluation of a causal model; mirrors bark_eval_encoder_internal (bark.cpp:1586-1643)
// logits [lm_lo, lm_hi) are computed and copied to logits_host + lm_lo (lm_hi <= 0: all of them).  mem_k / mem_v: the KV cache
// to use (null: the model's own)
bool gpt_eval(bark_context * ctx, GPTModel & m, const int32_t * tokens, int n, int * n_past, bool merge_ctx, float * logits_host, int lm_lo = 0, int lm_hi = 0,
              float * mem_k = nullptr, float * mem_v = nullptr);
// one decode step of B <= 8 independent sequences: row b feeds tokens[b] at position n_past[b] through the KV cache
// (slot_k[b], slot_v[b]); logits [lm_lo, lm_hi) of row b land in d_logits + b * n_out_vocab (device)
bool gpt_step_batch(bark_context * ctx, GPTModel & m, int B, float * const * slot_k, float * const * slot_v, const int32_t * tokens, const int * n_past,
                    int lm_lo, int lm_hi, float * d_logits);
void build_decode_tables(bark_context * ctx, GPTModel & m);
// one non-causal pass of the fine model; mirrors bark_eval_fine_encoder_internal (bark.cpp:1907-1959)
bool fine_eval(bark_context * ctx, const int32_t * in_buffer /*[8][1024]*/, int nn, float * logits_host /*[1024][n_out]*/);
bool fine_eval_shard(bark_context * ctx, const int32_t * in_buffer, int nn);                          // this rank's rows of one pass (shard.cu)
bool sample_shard(bark_context * ctx, std::mt19937 & rng, int n, float temp, int32_t * out_all /*[1024]*/);
bool fine_eval_fast(bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_host);      // tensor-core variant (fast mode)
// EnCodec decode; codes [8][T] on the host; result in `audio`
bool codec_decode(bark_context * ctx, const int32_t * codes, int T, std::vector<float> & audio);

// sampling.cu / gpt_forward.cu / bark_api.cu
void sample_rows(const float * logits, int ld, int n, int rows, float temp, const double * d_u, int32_t * d_out_tok, int tok_add, int32_t * d_feed,
                 float * d_eos_p, int32_t * d_flags, int force_flag, cudaStream_t s);
void sample_rows_threads(int threads, const float * logits, int n, int rows, float temp, const double * d_u, int32_t * d_out_tok, float * d_eos_p,
                         int32_t * d_flags, cudaStream_t s);
bool gpt_decode_chained(bark_context * ctx, GPTModel & m, const int32_t * d_token, int * n_past, int lm_lo, int lm_hi);
bool sample_device(bark_context * ctx, GPTModel & m, std::mt19937 & rng, const float * d_logits, int ld, int n, int rows, float temp, int32_t * out_tok, float * out_eos);
int32_t sample_token_given_u(const float * logits, int n, float temp, double u, float * eos_p);

int64_t now_us();

}  // namespace bark
