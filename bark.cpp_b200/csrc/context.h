// bark_context: everything one generation needs, owned by bark_load_model / bark_free.
// Host control plane in C++ (like the reference's bark.cpp:133-164), all tensors in HBM.
#pragma once
#include "../../include/bark_b200.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <fstream>
#include <functional>
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

// A speaker history prompt (bark_b200_set_history_prompt): upstream Bark's voice-file arrays, codebook-major, validated.
// No semantic ids: no prompt.
struct HistoryPrompt {
    std::vector<int32_t> semantic;                   // [n_s]
    std::vector<int32_t> coarse;                     // [2][n_c]
    std::vector<int32_t> fine;                       // [8][n_f], n_f may be 0
    bool empty() const { return semantic.empty(); }
};

// What one generation reads and produces: its RNG, its history prompt, its token streams and its waveform.  The context holds one
// (bark.h's single-prompt calls); every item of a batch (bark_b200_generate_batch) holds its own, so a batch leaves the context's untouched.
struct Generation {
    std::mt19937 rng;                                // seeded once at load (bark.cpp:1179), or per batch item
    HistoryPrompt prompt;                            // conditions the three stages (generation.cu); empty: every generation starts from nothing
    std::vector<int32_t> tokens;                     // 513 prompt ids
    std::vector<int32_t> semantic_tokens;
    std::vector<int32_t> coarse_tokens;              // [T][2] flattened
    std::vector<int32_t> fine_tokens;                // [T][8] flattened
    std::vector<float> audio;
};

// Batched generation (generation.cu): one f32 KV cache [L][block_size][E] per item and causal model, allocated on the first batch and
// grown when a later one has more items; the [8][n_out] logits of the batched step; the step's ids and positions (device + pinned).
struct BatchSlots {
    int cap = 0;
    float * k[2][8] = {}, * v[2][8] = {};            // [semantic / coarse][slot]
    float * d_logits = nullptr;                      // [8][max n_out of the causal models]
    int32_t * d_step = nullptr, * h_step = nullptr;  // [0, 8): input ids, [8, 16): positions (n_past) of the step's rows
    std::vector<Generation> results;                 // the last batch's items (bark_b200_batch_audio / bark_b200_batch_tokens)
};

// One chunk of the last long-form generation (long_form.cu): its text and its ids, as the Generation fields of the same names hold them
struct LongFormChunk {
    std::string text;
    std::vector<int32_t> tokens, semantic_tokens, coarse_tokens, fine_tokens;
};

// Long-form generation (bark_b200_set_long_form, DESIGN.md §18): the settings of the context's later bark_generate_audio calls, and the
// chunks of the last successful long-form call (bark_b200_long_chunk_*)
struct LongForm {
    bool on = false;
    bark_b200_long_form settings{BARK_B200_VOICE_CHAIN, 48, 6000};
    std::vector<LongFormChunk> chunks;
};

struct bark_context {
    int device = 0;
    cudaStream_t stream = nullptr;

    bark::GPTModel semantic, coarse, fine;
    bark::CodecModel codec;
    std::map<std::string, int32_t> token_to_id;      // WordPiece vocabulary (bark.cpp:664-690)
    int tokenizer = BARK_B200_TOKENIZER_REFERENCE;   // bark_b200_set_tokenizer / BARK_B200_TOKENIZER; every batch item follows it

    __half * d_gelu_tab = nullptr;                   // 65536-entry table, ggml.c:3795-3810
    unsigned * d_ln_fallbacks = nullptr;             // [0] LayerNorm rows, [1] soft_max rows replayed sequentially
    unsigned tag_base = 0;                           // epoch counter of the decode kernel's tagged exchanges (advances 6*L per token)
    int n_sm = 0, n_sm_total = 0; bool use_decode_kernel = true;   // n_sm: CTAs of the persistent decode kernel (knob); n_sm_total: SMs of the device
    bool kv_reuse = true; unsigned long long n_kv_reused = 0;   // coarse windows start from the cached prefix (generation.cu run_coarse)
    // decode-kernel knobs (BARK_B200_DECODE_TIMING_TID / BARK_B200_POLL_NS / BARK_B200_HEADSTART); defaults:
    // 40 ns back-off between polls, 500 ns head start for the two residual exchanges
    unsigned headstart[6] = {0, 2000, 500, 400, 500, 0};   // BARK_B200_HEADSTART=q:att:x1:ff:x2:scores (ns): sleep before the first poll of each exchange
    int timing_tid = 0; unsigned poll_ns = 40;
    unsigned long long * d_timing = nullptr;         // optional phase timestamps of the decode kernel (BARK_B200_DECODE_TIMING=1)

    // BARK_B200_MODE=fast: the fine model's passes run on the tensor cores (fast_kernels.cu); not bit-identical to the reference
    bool fast_mode = false;
    __half * f_a16 = nullptr, * f_h16 = nullptr, * f_qk16 = nullptr, * f_vt16 = nullptr, * f_att16 = nullptr;   // [1024][E], [1024][4E], [1024][2E], [E][1024], [1024][E]

    ShardState shard;

    bark::Workspace ws;
    bark::Q8Scratch q8;                              // quantised models: the q8 activation operand ([rows][4E] codes, [rows][4E/32] d and s)
    const float * last_logits = nullptr;             // device logits of the latest gpt_eval / fine_eval
    double * d_u = nullptr, * h_u = nullptr;         // device sampling: uniforms, tokens, flags, eos probabilities (1024 rows)
    int32_t * d_stok = nullptr, * h_stok = nullptr, * d_sflags = nullptr, * h_sflags = nullptr;
    float * d_seos = nullptr, * h_seos = nullptr;
    int32_t * d_feed = nullptr;                      // token handed from sample_rows_kernel to the next decode step
    // top-k / top-p of the semantic [0] and coarse [1] stages (bark_b200_set_sampling), shared by every batch item; both off by default
    bark_b200_sampling sampling[2] = {{0, 0, 1.0f}, {0, 0, 1.0f}};
    float * d_frow = nullptr;                        // filter_rows_kernel's output: kMaxFilterRows filtered rows of kSampleMaxLogits
    int32_t * d_fflags = nullptr, * h_fflags = nullptr;   // its flags, per sample (1024)
    long long n_sample_host_replays = 0;
    int debug_flag_every = 0; long long n_sample_calls = 0;   // BARK_B200_SAMPLE_FLAG_EVERY=k: force every k-th sample through the host replay (tests)
    float * h_logits = nullptr;                      // pinned, max(n_out) or 1024*fine_vocab
    int32_t * h_tok = nullptr;                       // pinned, 8*1024 ids

    bark::CodecScratch codec_scratch;

    Generation gen;                                  // the bark.h calls' generation state
    BatchSlots batch;
    LongForm long_form;

    bark_context_params params;
    bark_statistics stats{};

    bark::DeviceArena arena;                         // everything else cudaMalloc'ed for this context
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
bool gpt_decode_chained(bark_context * ctx, GPTModel & m, const int32_t * d_token, int * n_past, int lm_lo, int lm_hi);
// The first step of every fine pass: nn and each code of the window checked (messages name fn), the [8][1024] ids uploaded and
// rows [row0, row0 + rows) of the window embedded into ws.x
bool fine_embed(bark_context * ctx, const int32_t * in_buffer, int nn, int row0, int rows, const char * fn);
// final LayerNorm + lm_head (bark.cpp:1391-1405) on `rows` rows from x: the logits of head's outputs land at logits + lo, rows
// n_out_vocab apart, and logits becomes the context's last_logits
void output_head(bark_context * ctx, const GPTModel & m, const float * x, int rows, const DMat & head, float * logits, int lo = 0);

// The activation operand of a model's per-op mat-muls (gpt_forward.cu act_layout): what the producers are told, and its group stride
// in front of the E-wide and the 4E-wide mat-muls
struct ActLayout { WType wt; int kpE, kp4E; };
// The per-op transformer body on `rows` rows of ws.x, updated in place (gpt_forward.cu).  kv keeps the pass's K and V:
// kv.store(ctx, m, il, rows, qkv) points the QKV epilogue's K / V stores at layer il's rows, and kv.attend(ctx, m, il, rows, a)
// runs that layer's attention from ws.q into ws.act.
template <class KV> void run_layers(bark_context * ctx, const GPTModel & m, int rows, const KV & kv);
// K / V of the row-sharded fine pass (shard.cu)
struct ShardKV {
    int row0;
    void store(bark_context * ctx, const GPTModel & m, int il, int rows, MatmulEpilogue & qkv) const;
    void attend(bark_context * ctx, const GPTModel & m, int il, int rows, const ActLayout & a) const;
};
// loader.cu: reads the codec section at f's position into c: every tensor, codebooks 0..max_q-1 (at least 8 must exist); buffers from
// arena.  Shared by bark_context (8 codebooks) and encodec_context (encodec_api.cu).
bool load_codec(std::ifstream & f, CodecModel & c, int max_q, DeviceArena & arena, cudaStream_t s, bool verbose);
// codec_pipeline.cu — the EnCodec pipelines, shared by bark_context and encodec_context.
// Both take n clips of independent lengths.  Every item is validated before anything is enqueued; batch_fn: the public batch call, whose
// name the messages carry and which name the item (null: a single call's messages, under the pipeline's own name);
// the items then run in consecutive launches, each one pass of the codec kernels over all its items with one
// synchronisation at its end.  Item i's results are bit-identical to the same clip run alone.
// Frames of one launch (about 320 s of audio): its scratch is 131 KB per frame, 3.1 GB at the budget.  A longer clip runs alone.
constexpr int kCodecLaunchFrames = 24000;
// Decode codes[i] ([n_q][T[i]] on the host, checked against the codebooks, T[i] >= kCodecMinFrames) to kCodecHop T[i] samples in audio[i].
bool codec_decode(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, int n, const int32_t * const * codes, const int * T, int n_q,
                  std::vector<float> * audio, const char * batch_fn = nullptr);
// What an encode copies back for item i where the array is set: its codes [n_q][T_i] to codes[i], its latent [128][T_i] to latent[i]
// and the decoder's waveform of those codes (encodec_reconstruct_audio) to audio[i].
struct CodecOutputs { std::vector<int32_t> * codes = nullptr; std::vector<float> * latent = nullptr, * audio = nullptr; };
// Encode (encodec_compress_audio): audio[i], n_samples[i] mono 24 kHz samples -> T_i = ceil(n_samples[i] / kCodecHop) frames, the
// outputs of out.  false (message on stderr) without encoder tensors, for n_samples < kCodecMinSamples, a non-finite sample or n_q
// outside the loaded codebooks.
// With fmt, item i is n_samples[i] interleaved frames [n][fmt[i].channels] at fmt[i].sample_rate, down-mixed and resampled to 24 kHz on
// the device first (DESIGN.md §16); its resampled length L_i then stands for n_samples[i].  Mono 24 kHz items go in unchanged.
constexpr int kCodecSampleRate = 24000;
struct AudioFormat { int channels, sample_rate; };
bool codec_encode(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, int n, const float * const * audio, const int * n_samples, int n_q,
                  const CodecOutputs & out, const char * batch_fn = nullptr, const AudioFormat * fmt = nullptr);
// false (message naming fn, and the item for a batch) for a format or clip outside the resampler's limits: 1 to 8 channels, 4000 to
// 384000 Hz, fewer than 2^31 samples, every sample finite with |x| <= 2^64
bool resample_input_ok(const char * fn, const std::string & item, const float * x, int n_frames, int channels, int sample_rate);
// "item i: " in the messages of a batch call (batch_fn set), whatever its size; nothing for a single call, whose messages stay as they were
std::string item_tag(const char * batch_fn, int i);
// sizes sc for one launch of `frames` frames of n_q codebooks: false (message naming caller) when the device is out of memory
bool codec_scratch(CodecScratch & sc, size_t frames, int n_q, const char * caller);
// sizes sc.stage (source frames before the resampler) to `floats`, the same way
bool stage_scratch(CodecScratch & sc, size_t floats, const char * caller);

// codec_stream.cu — streaming EnCodec (DESIGN.md §19).  A stream goes one way: mono 24 kHz samples to codes, or codes to samples, at the
// n_q it opened with.  Its state lives on the device: per windowed layer the input columns later outputs still read, per LSTM layer
// (h, c).  Pending outputs wait on the host until read: codes frame-major [k][n_q], or samples.
constexpr int kStreamEncode = 0, kStreamDecode = 1;
// the outputs final after n inputs, before finish: frames after n samples (encode), samples after n frames (decode)
long long codec_stream_ready(int direction, long long n);
// The same for a stream at another format (DESIGN.md §20): frames after n interleaved frames at sample_rate (encode), samples at
// sample_rate after n frames (decode)
long long codec_stream_ready_resampled(int direction, int sample_rate, long long n);
// A stream's resampler (DESIGN.md §20): an encode's interleaved source frames at `rate` to the encoder's 24 kHz samples, or a decode's
// 24 kHz samples to `rate`.  It keeps its input from the next block's first read on, raw, and its own device copy of the taps.
struct StreamResampler {
    int channels = 1, rate = 0;
    ResampleTable t;                                     // bound to taps (null for equal rates)
    void * taps = nullptr;
    float * hist = nullptr; int cap = 0, h = 0;          // hist [cap][channels], h frames held: the global frames in - h .. in - 1
    long long in = 0, out = 0;                           // frames in, outputs final
};
struct CodecStream {
    int direction = kStreamEncode, n_q = 0;
    bool finished = false, failed = false;               // failed: a pass did not complete (a CUDA failure); the state is lost
    long long n_in = 0, n_out = 0;                       // the codec's inputs pushed, outputs final (24 kHz samples on a resampled stream)
    bool resampled = false; StreamResampler rs;          // any format other than mono 24 kHz
    struct Window { int C = 0, cap = 0, h = 0; long long in = 0, out = 0; float * hist = nullptr; };   // hist [C][cap], h columns held
    std::vector<Window> win;                             // in layer-list order
    float * lstm[4] = {nullptr, nullptr, nullptr, nullptr};   // (h, c) [2][512] of the four LSTM layers (two for the direction's model)
    float * mem = nullptr;                               // the device allocation behind win and lstm
    std::vector<int32_t> codes;
    std::vector<float> audio;
    void release();
};
// allocates st's device state for direction at n_q codebooks, and for any format but mono 24 kHz (channels 1 for a decode) its
// resampler (a CUDA failure throws)
bool codec_stream_init(const CodecModel & cm, CodecStream & st, int direction, int n_q, int channels = 1, int sample_rate = kCodecSampleRate);
// pushes n[i] inputs at in[i] (samples, interleaved frames [n[i]][channels] on a resampled encode, or codes [n_q][n[i]]) to the count <= kCodecMaxItems checked streams st[i] of one model and
// direction in one pass of the kernels (or several for a long push), or with finish none, closing them.  Returns the outputs that
// became final, -1 (message naming fn) on a failure.
int codec_stream_run(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, CodecStream * const * st, const void * const * in, const int * n, int count,
                     bool finish, const char * fn);

// sampling.cu
constexpr int kSampleMaxLogits = 16384;          // logits of one row: sample_rows_kernel holds the row in 64 KB of shared memory
// sample_rows_kernel over `rows` rows of n logits (stride ld); threads 256 or 1024 per row, 0 picks 1024 for one row and 256 otherwise
void sample_rows(const float * logits, int ld, int n, int rows, float temp, const double * d_u, int32_t * d_out_tok, int tok_add, int32_t * d_feed,
                 float * d_eos_p, int32_t * d_flags, int force_flag, int threads, cudaStream_t s);
// gpt_sample of one row on the host with the uniform u already drawn (unused when temp == 0)
int32_t sample_token_given_u(const float * logits, int n, float temp, double u, float * eos_p);
// top-k / top-p (DESIGN.md §14): on when top_k >= 1 or use_top_p
inline bool filter_on(const bark_b200_sampling & f) { return f.top_k > 0 || f.use_top_p != 0; }
// top-k / top-p settings: false with a message naming `fn` for anything the rule does not define
bool sampling_valid(const char * fn, const bark_b200_sampling & s);
constexpr int kMaxFilterRows = 8;                // rows filtered at once: one decode step of a batch
// filter_rows_kernel over `rows` rows of n <= kSampleMaxLogits raw logits (stride ld): d_out [rows][n] gets each row with the removed
// logits set to -inf, d_kept (may be null) the number kept, d_flags 1 where the device cannot decide the row exactly (a NaN, a
// non-finite maximum, an exp within rounding of a float boundary).  threads as sample_rows.
void filter_rows(const float * logits, int ld, int n, int rows, const bark_b200_sampling & f, float * d_out, int32_t * d_kept, int32_t * d_flags, int threads,
                 cudaStream_t s);
// the same filter on the host with libm's exp, in place; returns the number of logits kept
int filter_row_host(float * row, int n, const bark_b200_sampling & f);
// Copies the sampler's outputs of rows [start, stop) back to the host — tokens to ctx->h_stok, flags to h_sflags, with want_eos the
// probabilities of the last logit to h_seos, with filtered the filter's flags to h_fflags — and synchronises the stream.
void read_back_samples(bark_context * ctx, int start, int stop, bool want_eos, bool filtered);
// after read_back_samples: row r must be decided on the host (flagged by the sampler, or by the filter when one ran)
inline bool sample_flagged(const bark_context * ctx, int r, bool filtered) { return ctx->h_sflags[r] || (filtered && ctx->h_fflags[r]); }
// Samples `rows` (<= 1024; <= kMaxFilterRows with a filter) rows of device logits, row r at d_logits + r * ld + lo, n <= kSampleMaxLogits
// wide, with the uniforms the caller put in ctx->h_u[0, rows) (temp != 0).  With f set and on, filter_rows runs first and the sampler
// reads its output.  One read_back_samples brings the tokens (lo added), the flags and, with want_eos, the probabilities of the last
// logit back; every row flagged by either kernel is then replayed on the host (filter_row_host from the raw logits, then
// sample_token_given_u with the same uniform).  Returns the number of rows replayed.
int sample_and_replay(bark_context * ctx, const float * d_logits, int ld, int lo, int n, int rows, float temp, bool want_eos, const bark_b200_sampling * f = nullptr);
// sample_and_replay with `rows` uniforms drawn from rng; tokens to out_tok, eos probabilities to out_eos when it is set
bool sample_device(bark_context * ctx, GPTModel & m, std::mt19937 & rng, const float * d_logits, int ld, int n, int rows, float temp, int32_t * out_tok, float * out_eos);

// tokenizer.cu — the reference's tokenizer and upstream Bark's (DESIGN.md §17), by kind (BARK_B200_TOKENIZER_*).  tokenizer_known: false
// (message naming fn) for an unknown kind; tokenizer_from_env: BARK_B200_TOKENIZER's kind, -1 (message) for a value it does not name.
bool tokenizer_known(int kind, const char * fn);
int tokenizer_from_env(const char * fn);
// The ids of text under kind, cut to a prompt of cap ids as each tokenizer cuts it (the reference's stops at cap - 1 pieces, upstream's
// keeps the first cap); false with a message naming fn for an unknown kind or a refused text or vocabulary.  warn: the reference's
// message for a character it skips.  count_text_ids: their uncapped number, without that message; -1 where text_ids fails.
bool text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, int cap, std::vector<int32_t> & ids, const char * fn, bool warn);
int count_text_ids(const std::map<std::string, int32_t> & vocab, int kind, const std::string & text, const char * fn);
// upstream Bark's ids, untruncated; false with a message naming fn for invalid UTF-8 or a vocabulary without [UNK]
bool bert_tokenize(const std::map<std::string, int32_t> & vocab, const std::string & text, std::vector<int32_t> & out, const char * fn);
// Python's \s (str.isspace)
bool py_space(uint32_t cp);
// Strict UTF-8 (RFC 3629) to code points; false with the offending byte's offset in *bad
bool decode_utf8(const std::string & s, std::vector<uint32_t> & out, size_t * bad);
void append_utf8(std::string & s, uint32_t cp);

// generation.cu — the prompt, the three stages and the codec of one generation, and batches of up to kMaxBatch of them
constexpr int kMaxBatch = 8;
bool tokenize_input(bark_context * ctx, Generation & g, const std::string & text, const char * fn);
bool run_semantic(bark_context * ctx, Generation & g);
bool run_coarse(bark_context * ctx, Generation & g);
bool run_fine(bark_context * ctx, Generation & g, bool progress = true);
bool generate_one(bark_context * ctx, const std::string & text);
bool make_history_prompt(const bark_context_params & P, const bark_b200_history_prompt & p, HistoryPrompt & h);
bool generate_batch(bark_context * ctx, const char * const * texts, const uint32_t * seeds, const bark_b200_history_prompt * const * prompts, int n);
bool ensure_batch_slots(bark_context * ctx, int n);

// long_form.cu (DESIGN.md §18).  The chunks of text under long-form rules 1-4: text validated and its whitespace normalised into norm,
// split into sentences and over-long sentences into pieces of at most max_ids ids by count (count_text_ids on the chunk text); chunks
// without ids dropped.  [begin, end) byte offsets into norm go to bounds.  Returns their number, or -1 with a message naming fn (invalid
// UTF-8, max_ids outside [1, 255], a count that fails, no chunk left or more than kLongFormMaxChunks).
constexpr int kLongFormMaxChunks = 1024;
int split_text(const std::string & text, int max_ids, const std::function<int(const std::string &)> & count, std::string & norm,
               std::vector<std::pair<size_t, size_t>> & bounds, const char * fn);
// bark_generate_audio with long form on: every chunk one generate_one on the context's generation, prompted as the voice setting says,
// the waveforms joined with gap_samples zeros; the context's prompt restored at the end.  A refused text changes nothing.
bool generate_long(bark_context * ctx, const std::string & text);

int64_t now_us();
// bark_api.cu: the device of the calling thread's next context (bark_b200_set_device, else BARK_B200_DEVICE, else 0), made current;
// -1 with a message from `caller` when it is missing or not an sm_90 device
int select_device(const char * caller, cudaDeviceProp * prop);

// The call path of every bark_context entry point: a null context is "fn: invalid bark context" and fail; otherwise f() runs with the
// context's device current (a host thread may drive contexts on several devices), and a CUDA failure or exception is fail.
template <typename R, typename F> R with_context(bark_context * ctx, const char * fn, R fail, F && f) {
    if (!ctx) { fprintf(stderr, "%s: invalid bark context\n", fn); return fail; }
    return guarded(fail, [&]() -> R { BARK_CUDA_CHECK(cudaSetDevice(ctx->device)); return f(); });
}

// The copy-out of the entry points that fill a caller's array: the first min(size, cap) elements of v to out when it is set (none for
// cap < 0); returns v's size
template <class V> int copy_out(const V & v, typename V::value_type * out, int cap) {
    if (out) std::copy_n(v.data(), std::min(v.size(), (size_t) std::max(cap, 0)), out);
    return (int) v.size();
}

}  // namespace bark
