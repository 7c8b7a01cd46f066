/* bark_b200.h — additive C entry points of libbark_b200 (nothing here exists in the reference header).
 *
 * They expose, through the same C-ABI shared library, the per-call pieces the reference keeps file-static,
 * so that parity tests and the benchmark can drive and time one step of the hot path with HOST buffers:
 *
 *   bark_b200_gpt_eval ........ one causal GPT evaluation  == bark_eval_encoder_internal      (bark.cpp:1586-1643)
 *   bark_b200_fine_eval ....... one fine pass              == bark_eval_fine_encoder_internal (bark.cpp:1907-1959)
 *   bark_b200_encodec_decode .. codes -> waveform          == encodec_decompress_audio        (encodec.cpp/encodec.cpp:902-924)
 *   bark_b200_encodec_encode .. waveform -> codes          == encodec_compress_audio          (encodec.cpp/encodec.cpp:878-900)
 *   bark_b200_sample .......... gpt_sample on the context RNG                                 (bark.cpp:249-270)
 *   bark_b200_sample_rows ..... the same for `rows` logit rows, on the device sampler the stages use (host replay of rows it cannot decide)
 *   bark_b200_forward_* ....... extern "C" names for bark_forward_{text,coarse,fine}_encoder  (bark.cpp:1703,1865,2061)
 *   bark_b200_tokenize ........ bark_tokenize_input                                           (bark.cpp:622-662; or upstream Bark's, see TEXT TOKENIZERS)
 *
 * plus device selection for one-context-per-GPU batching (SURVEY.md §8e): bark_context_params must keep the
 * reference layout, so the device is chosen by bark_b200_set_device() or the BARK_B200_DEVICE environment
 * variable before bark_load_model (and before encodec_load_model, include/encodec.h).
 */
#pragma once
#include "bark.h"

#ifdef __cplusplus
extern "C" {
#endif

BARK_API void bark_b200_set_device(int cuda_device);                       /* applies to subsequent bark_load_model / encodec_load_model calls */
BARK_API const char * bark_b200_version(void);

/* which: 0 semantic, 1 coarse.  Host pointers.  *n_past advances exactly like the reference (by 257 for the merged prompt). */
BARK_API int  bark_b200_gpt_eval(struct bark_context * ctx, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out);
/* in_buffer: [8][1024] ids; nn: codebook being predicted (2..7); logits_out: [1024][n_out_vocab] */
BARK_API int  bark_b200_fine_eval(struct bark_context * ctx, const int32_t * in_buffer, int nn, float * logits_out);
/* codes: [8][n_frames]; returns number of samples (320 * n_frames), copies min(n, out_cap) floats to out (may be NULL) */
BARK_API int  bark_b200_encodec_decode(struct bark_context * ctx, const int32_t * codes, int n_frames, float * out, int out_cap);
/* EnCodec encode == encodec_compress_audio (encodec.cpp/encodec.cpp:878-900) at 6 kbps, bit-identical to it; the context's generation
 * state (RNG, ids, bark_get_audio_data) is not touched.
 * audio: n_samples mono 24 kHz f32, finite, n_samples >= 1921.  codes: [8][T] codebook-major (the layout bark_b200_encodec_decode
 * takes), T = ceil(n_samples / 320); copies min(8 T, codes_cap) values (codes may be NULL).  latent (may be NULL): the encoder output
 * before quantisation, [128][T] f32, min(128 T, latent_cap) values.  Returns T, or -1 (message on stderr), also for a model file
 * written without the encoder tensors. */
BARK_API int  bark_b200_encodec_encode(struct bark_context * ctx, const float * audio, int n_samples, int32_t * codes, int codes_cap,
                                       float * latent, int latent_cap);
/* Test hook, no context: the RVQ encode kernel on host buffers.  latent [hidden][T], codebooks [n_q][n_bins][hidden] f32, codes [n_q][T];
 * hidden % 32 == 0 and <= 128, n_bins <= 1024, n_q <= 32.  Returns 1 on success, 0 on invalid arguments or failure. */
BARK_API int  bark_b200_rvq_encode(const float * latent, int T, const float * codebooks, int hidden, int n_bins, int n_q, int32_t * codes);
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

/* SPEAKER HISTORY PROMPTS: condition the semantic, coarse and fine stages on a voice prompt's ids, as upstream Bark's history_prompt
 * (its semantic_prompt / coarse_prompt / fine_prompt voice-file arrays) does, so that consecutive generations keep one voice.  A
 * finished generation's own ids are a valid prompt for the next one; bark_b200_encodec_encode's codes are a fine prompt.  C and F are
 * codebook-major, the layout of the voice files and of bark_b200_encodec_encode.  A prompt is valid when n_semantic >= 1 and every
 * semantic id is in [0, semantic_vocab_size); n_coarse_frames >= 1, n_fine_frames >= 0 and every code is in [0, codebook_size); and
 * the two lengths align as upstream checks it, round(n_c / n_s, 1) == round(stc / n_coarse_codebooks, 1) with stc = coarse_rate_hz /
 * semantic_rate_hz * n_coarse_codebooks: 29 n_s < 20 n_c < 31 n_s for the default rates.  What a prompt changes (DESIGN.md §12):
 *   semantic  prompt positions [256, 512) hold the last 256 semantic ids, right-padded
 *   coarse    each window starts from up to 209 prompt semantic ids and up to 628 prompt coarse ids before the generated ones
 *   fine      the last min(n_fine_frames, 512) prompt frames precede the coarse frames in the fine windows
 * The generated ids, bark_get_audio_data, the statistics and bark_b200_get_tokens stages 0-2 describe the generated part only; stage
 * 3 returns the prompted 513 ids. */
struct bark_b200_history_prompt {
    const int32_t * semantic; int n_semantic;        /* [n_semantic] */
    const int32_t * coarse;   int n_coarse_frames;   /* [2][n_coarse_frames] */
    const int32_t * fine;     int n_fine_frames;     /* [8][n_fine_frames], may be 0 frames */
};
/* Validates and copies; NULL clears.  Applies to later bark_generate_audio, bark_b200_tokenize and bark_b200_forward_* calls
 * on this context.  Returns 1, or 0 with a message; a rejected prompt leaves the previous one in place. */
BARK_API int  bark_b200_set_history_prompt(struct bark_context * ctx, const struct bark_b200_history_prompt * prompt);
/* bark_b200_generate_batch with one prompt per item: prompts may be NULL, and so may any entry (no prompt).  Item i equals a fresh
 * context with seeds[i] and prompts[i] set, generating texts[i].  A rejected prompt fails the batch before anything runs.
 * bark_b200_generate_batch itself ignores the context's prompt. */
BARK_API bool bark_b200_generate_batch_prompted(struct bark_context * ctx, const char * const * texts, const uint32_t * seeds,
                                                const struct bark_b200_history_prompt * const * prompts, int n, int n_threads);

/* TOP-K / TOP-P SAMPLING of the semantic and coarse stages, upstream Bark's generate_text_semantic / generate_coarse filter on the
 * reference's arithmetic (DESIGN.md §14).  The row the stage samples (semantic: all n_out_vocab logits; coarse: the 1024-wide codebook
 * window) is ordered by logit descending, equal logits (+0 and -0 included) by descending index.  top-p removes sorted position j >= 1
 * when the float cumulative sum of the reference's softmax of the sorted row up to position j - 1 exceeds top_p; top-k then removes
 * every logit below the k-th largest that remains (ties of the k-th value stay).  Removed logits become -inf before gpt_sample, which
 * is otherwise unchanged: the same single uniform draw, the same RNG stream; eos_p is 0 when the last logit was removed.  The fine
 * stage has no filter.  Both off: every stage is exactly what it is without this call. */
struct bark_b200_sampling {
    int32_t top_k;       /* 0: off; k >= 1 */
    int32_t use_top_p;   /* 0: off */
    float   top_p;       /* with use_top_p: finite, in [0, 1] (0 keeps only sorted position 0: of tied maxima, the highest index) */
};
/* stage 0 semantic, 1 coarse; s NULL turns both filters of the stage off.  Validates and copies; returns 1, or 0 with a message (the
 * previous settings stay).  Applies to later bark_generate_audio and bark_b200_forward_text_encoder / _coarse_encoder calls, and to
 * every item of bark_b200_generate_batch[_prompted]. */
BARK_API int  bark_b200_set_sampling(struct bark_context * ctx, int stage, const struct bark_b200_sampling * s);
/* Test hook, no context: bark_b200_sample_given_u with the filter s (NULL: off) applied first, on the device by filter_rows_kernel and,
 * for a flagged row, on the host from the raw logits.  flags: bit 0 the sampler flagged the row, bit 1 the filter did; kept (may be
 * NULL): the number of logits the device filter kept.  Returns the number of replayed rows, or -1 on invalid arguments or failure. */
BARK_API int  bark_b200_sample_filtered_given_u(const float * logits, int n, int rows, float temp, const struct bark_b200_sampling * s,
                                                const double * u, int threads, int32_t * tokens, int32_t * device_tokens, int32_t * flags,
                                                float * eos_p, int32_t * kept);

/* TEXT TOKENIZERS (DESIGN.md §17).  The reference's tokenizer (bark.cpp:480-662) folds 52 Latin-1 letters to ASCII and skips every
 * other non-ASCII byte, so most of Bark's 13 languages reach the model as nothing but digits and punctuation.  The BERT tokenizer is
 * upstream Bark's: BertTokenizer("bert-base-multilingual-cased").encode(re.sub(r"\s+", " ", text).strip(), add_special_tokens=False)
 * with the tokenizers pipeline of transformers 5 (BertNormalizer with clean_text and handle_chinese_chars, no accent stripping, no
 * lowercasing; BertPreTokenizer; WordPiece with ## continuations, a word over 100 code points one [UNK]), on the file's vocabulary;
 * [PAD] [UNK] [CLS] [SEP] [MASK] found literally in the text are single tokens.  Its prompt keeps the first min(block_size, 256) ids
 * (the reference keeps 255), adds text_encoding_offset and pads with text_pad_token; the semantic history and infer token follow as
 * before.  Text must be valid UTF-8; no Unicode normalisation is applied (transformers 4's Python tokenizer applies NFC first), so pass
 * NFC text.  Everything after the 513 prompt ids is unchanged. */
#define BARK_B200_TOKENIZER_REFERENCE 0   /* bark.cpp's (default; every existing result) */
#define BARK_B200_TOKENIZER_BERT      1   /* upstream Bark's: bert-base-multilingual-cased rules, above */
/* Applies to later bark_generate_audio and bark_b200_tokenize calls and to every item of bark_b200_generate_batch[_prompted].
 * BARK_B200_TOKENIZER=bert (or reference) in the environment at bark_load_model sets a context's initial kind; another value fails
 * the load.  A text the BERT tokenizer refuses (invalid UTF-8) fails bark_generate_audio or the batch before anything changes, and
 * leaves bark_b200_tokenize's output untouched.  Returns 1, or 0 with a message (unknown kind); the previous choice stays. */
BARK_API int bark_b200_set_tokenizer(struct bark_context * ctx, int kind);
/* The raw WordPiece ids of text under kind (before truncation, offset and padding); copies min(count, cap) to out (may be
 * NULL).  Returns the count, or -1 with a message (invalid UTF-8 for BERT, NULL arguments, unknown kind). */
BARK_API int bark_b200_text_ids(struct bark_context * ctx, int kind, const char * text, int32_t * out, int cap);
/* Test hook, no context, no device: BERT ids of text over vocab[0..n_vocab) (id = index, later duplicates win), as
 * bark_b200_text_ids; -1 with a message for invalid UTF-8, NULL arguments or a vocabulary without [UNK]. */
BARK_API int bark_b200_bert_tokenize(const char * const * vocab, int n_vocab, const char * text, int32_t * out, int cap);

/* LONG-FORM GENERATION (DESIGN.md §18): upstream Bark's long-form recipe inside bark_generate_audio.  One call generates at most
 * about 14 s (255 text ids, n_steps_text_encoder semantic ids); with long form on, the text is split into sentences, each generated as
 * its own bark_generate_audio on a speaker prompt that keeps one voice, and the waveforms are joined with silence between them.
 *   1. normalise  the text must be valid UTF-8 (under either tokenizer); every run of Python's \s becomes one space, both ends stripped
 *   2. sentences  a sentence ends after a run of . ! ? … 。 ！ ？ ｡ । ॥ and the closing marks " ' ) ] } » ” ’ 」 』 ） directly after
 *                 it, when the run holds one of 。！？｡।॥ or a space or the end of the text follows; the space after it is dropped.  So
 *                 "3.5" and "e.g.x" do not split and "Mr. Smith" does: no abbreviation list is kept.  Empty sentences are dropped
 *   3. pieces     a sentence with more than max_chunk_ids ids under the context's tokenizer (as bark_b200_text_ids counts them) is
 *                 split greedily: words (split at spaces) while the piece stays within max_chunk_ids, a first word that is over
 *                 alone split the same way code point by code point (at least one); repeated on the rest.  Short sentences are not
 *                 merged.  A chunk is a sentence or a piece of one
 *   4. drop, cap  a chunk without ids is dropped; a text that leaves no chunk or more than 1024 is refused
 *   5. voice      BARK_B200_VOICE_CHAIN: chunk 0 uses the context's history prompt (or none), chunk k > 0 chunk k-1's own ids
 *                 (semantic, coarse, fine) when they are a valid prompt, else chunk k-1's prompt.  BARK_B200_VOICE_FIXED: every chunk
 *                 uses the context's prompt (or none)
 *   6. calls      the whole call equals, bit for bit, setting chunk k's prompt and calling bark_generate_audio on chunk k's text, in
 *                 order on this context: same RNG stream, progress callbacks and stage functions.  Afterwards the history prompt is what
 *                 it was before the call
 *   7. results    bark_get_audio_data: the chunks' waveforms in order with gap_samples zeros between consecutive ones; chunk k starts at
 *                 the sum over j < k of (320 fine frames of j + gap_samples).  bark_b200_get_tokens: the last chunk's ids.  The
 *                 statistics count the whole call: each stage's samples and time summed over the chunks, t_eval_us its wall time
 * A refused text (invalid UTF-8, no chunk, more than 1024 chunks) fails bark_generate_audio before anything runs: ids, waveform,
 * statistics, prompt, RNG and the chunk results stay as they were.  A context whose fine stage is sharded refuses long-form generation. */
#define BARK_B200_VOICE_CHAIN 0   /* each chunk prompted by the previous chunk's ids (default) */
#define BARK_B200_VOICE_FIXED 1   /* every chunk prompted by the context's history prompt, or none */
struct bark_b200_long_form {
    int32_t voice;           /* BARK_B200_VOICE_CHAIN or BARK_B200_VOICE_FIXED */
    int32_t max_chunk_ids;   /* 1 to 255 text ids per chunk (default 48) */
    int32_t gap_samples;     /* 0 to 240000 zeros between chunks (default 6000: 0.25 s at 24 kHz) */
};
/* Validates and copies; NULL turns long form off.  Returns 1, or 0 with a message (the previous settings stay).  Applies to later
 * bark_generate_audio calls only: bark_b200_tokenize, bark_b200_forward_* and bark_b200_generate_batch[_prompted] ignore it.
 * BARK_B200_LONG_FORM=chain or fixed in the environment at bark_load_model turns it on with that voice and the defaults; empty or off
 * leaves it off; another value fails the load. */
BARK_API int bark_b200_set_long_form(struct bark_context * ctx, const struct bark_b200_long_form * lf);
/* Chunks of the last successful long-form bark_generate_audio; 0 after a later generation without long form (-1 for a NULL context). */
BARK_API int bark_b200_long_chunks(struct bark_context * ctx);
/* Chunk k's text (UTF-8, a piece of the normalised text, no NUL appended): copies min(bytes, cap) to out (may be NULL) and returns its
 * bytes, or -1 for no such chunk. */
BARK_API int bark_b200_long_chunk_text(struct bark_context * ctx, int k, char * out, int cap);
/* Chunk k's ids of stage 0-3, as bark_b200_get_tokens returns them for a single call; -1 for no such chunk or stage. */
BARK_API int bark_b200_long_chunk_tokens(struct bark_context * ctx, int k, int stage, int32_t * out, int cap);
/* Test hook, no context, no device: rules 1-4 on text over vocab[0..n_vocab) (id = index, later duplicates win) under tokenizer kind.
 * Writes chunk i's [begin, end) byte offsets into the normalised text to bounds[2 i], bounds[2 i + 1] for i < cap (bounds may be NULL)
 * and returns the chunk count, or -1 with a message (invalid UTF-8, NULL arguments, unknown kind, max_chunk_ids outside [1, 255], no
 * chunk left, more than 1024 chunks). */
BARK_API int bark_b200_split_text(const char * const * vocab, int n_vocab, int kind, const char * text, int max_chunk_ids, int32_t * bounds,
                                  int cap);

/* BATCHED ENCODEC on an encodec_context (include/encodec.h): n clips of independent lengths in one call, for tokenising a dataset.
 * Item i's codes and waveform are bit-identical to encodec_compress_audio / _decompress_audio / _reconstruct_audio of that clip alone on
 * the same context: they do not depend on n, on i's place in the batch or on the other items.  The context's current bandwidth and
 * sample rate apply to every item.  1 <= n <= BARK_B200_ENCODEC_MAX_BATCH.  Every item is checked before anything runs, by the single
 * calls' rules (audio: n_samples[i] >= 1921 and finite; codes: n_codes[i] a multiple of n_q, n_codes[i] / n_q >= 7 frames, each code in
 * [0, n_bins)); a null array or entry, n out of range or a bad item returns false with a message naming the item, and changes nothing.
 * Inside the library the items run in consecutive launches of at most 32 items and 24000 frames (320 s of audio) each, a longer clip
 * alone; the codec scratch grows to the largest launch (131 KB per frame) and stays with the context.
 * A batch leaves encodec_get_codes / encodec_get_audio as they were; encodec_get_statistics' t_compute_us is the batch's wall time.
 *   bark_b200_encodec_compress_batch ..... audio[i]: n_samples[i] mono samples -> codes [n_q][T_i], T_i = ceil(n_samples[i] / 320)
 *   bark_b200_encodec_decompress_batch ... codes[i]: n_codes[i] codes [n_q][T_i] -> 320 T_i samples
 *   bark_b200_encodec_reconstruct_batch .. compress then decompress, the codes staying on the device -> 320 T_i samples
 *   bark_b200_encodec_batch_codes ........ codes of item i of the last successful compress batch; copies min(count, cap) to out (may
 *                                          be NULL); returns the count, or -1 if there is no such item
 *   bark_b200_encodec_batch_audio ........ samples of item i of the last successful decompress or reconstruct batch, the same way */
#define BARK_B200_ENCODEC_MAX_BATCH 1024
BARK_API bool bark_b200_encodec_compress_batch(struct encodec_context * e, const float * const * audio, const int * n_samples, int n);
BARK_API bool bark_b200_encodec_decompress_batch(struct encodec_context * e, const int32_t * const * codes, const int * n_codes, int n);
BARK_API bool bark_b200_encodec_reconstruct_batch(struct encodec_context * e, const float * const * audio, const int * n_samples, int n);
BARK_API int  bark_b200_encodec_batch_codes(struct encodec_context * e, int i, int32_t * out, int cap);
BARK_API int  bark_b200_encodec_batch_audio(struct encodec_context * e, int i, float * out, int cap);

/* RESAMPLED ENCODEC: audio at any sample rate and channel count, down-mixed and resampled to the encoder's 24 kHz on the GPU first
 * (DESIGN.md §16).  Audio is interleaved frames [n_frames][channels] (WAV order) at sample_rate Hz.  The rule is upstream EnCodec's
 * convert_audio order with torchaudio's resampler: the frame's channels summed in order in f32 and divided by channels, then
 * torchaudio.functional.resample(mono, sample_rate, 24000) with its defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99),
 * taps in double rounded to f32 and each output a double sum in tap order, rounded once (upstream EnCodec resamples with julius, whose
 * filter differs).  The resampled length is L = ceil(24000 n_frames / sample_rate) (exactly, in integers); mono 24 kHz goes in
 * unchanged, so these calls then equal their mono 24 kHz counterparts bit for bit.  Limits: 1 <= channels <= 8, 4000 <= sample_rate <=
 * 384000, n_frames * channels < 2^31, every sample finite with |x| <= 2^64, L >= 1921 (7 frames).  None of these calls changes the
 * context's sample rate (encodec_set_sample_rate, which only sets n_q) or its bandwidth.
 *   bark_b200_encodec_compress_resampled ......... encodec_compress_audio of the resampled clip: codes from encodec_get_codes
 *   bark_b200_encodec_reconstruct_resampled ...... encodec_reconstruct_audio of it: samples (24 kHz) from encodec_get_audio
 *   bark_b200_encodec_compress_batch_resampled ... bark_b200_encodec_compress_batch with a format per item: channels[i], sample_rates[i];
 *                                                  results from bark_b200_encodec_batch_codes, refusals as for that call
 *   bark_b200_encodec_reconstruct_batch_resampled  the same for bark_b200_encodec_reconstruct_batch: bark_b200_encodec_batch_audio
 *   bark_b200_encodec_encode_resampled ........... bark_b200_encodec_encode on a bark context (a fine prompt from a speaker clip); it
 *                                                  leaves the generation state alone
 *   bark_b200_resample ........................... no context, host buffers: writes the L resampled samples at out_rate to out (cap >=
 *                                                  L; out NULL only asks for L) and returns L, or -1 on invalid arguments or failure.
 *                                                  Both rates in [4000, 384000]; for the tests, and for Bark's 24 kHz output at 44.1 or
 *                                                  48 kHz. */
BARK_API bool bark_b200_encodec_compress_resampled(struct encodec_context * e, const float * audio, int n_frames, int channels, int sample_rate);
BARK_API bool bark_b200_encodec_reconstruct_resampled(struct encodec_context * e, const float * audio, int n_frames, int channels, int sample_rate);
BARK_API bool bark_b200_encodec_compress_batch_resampled(struct encodec_context * e, const float * const * audio, const int * n_frames, const int * channels,
                                                         const int * sample_rates, int n);
BARK_API bool bark_b200_encodec_reconstruct_batch_resampled(struct encodec_context * e, const float * const * audio, const int * n_frames, const int * channels,
                                                            const int * sample_rates, int n);
BARK_API int  bark_b200_encodec_encode_resampled(struct bark_context * ctx, const float * audio, int n_frames, int channels, int sample_rate, int32_t * codes,
                                                 int codes_cap, float * latent, int latent_cap);
BARK_API int  bark_b200_resample(const float * in, int n_frames, int channels, int in_rate, int out_rate, float * out, int cap);

/* STREAMING ENCODEC on an encodec_context (DESIGN.md §19): code live audio chunk by chunk, or play codes as they arrive.  A stream goes one
 * way, BARK_B200_STREAM_ENCODE (mono 24 kHz samples in, codes out) or BARK_B200_STREAM_DECODE (codes in, samples out), at the n_q of the
 * context's bandwidth when it opens; a later encodec_set_target_bandwidth does not touch it.  Pushes take chunks of any size, 0 included,
 * and a stream hands back each output as soon as no later input can change it.  Everything a stream returns, up to and including
 * finish, is bit-identical to the single call on all its input: encodec_compress_audio's codes [n_q][ceil(n / 320)] for an encode,
 * encodec_decompress_audio's 320 T samples for a decode, whatever the chunk sizes and whatever else runs on the context in between.
 *   encode: after n samples, frames 0 .. n / 320 - 1 are final once n >= 2240 (7 frames), none before; finish adds the last
 *           ceil(n / 320) - floor(n / 320) frames, padded on the right as the whole clip is, and refuses n < 1921.
 *   decode: after T >= 7 frames all 320 T samples are final, none before; finish adds nothing and refuses T < 7.
 * bark_b200_encodec_stream_ready(direction, n) is that rule: the outputs final after n inputs before finish (-1 for an unknown direction
 * or n < 0).  A stream's state is a few columns per layer on the device and its counters are 64-bit: it may run for hours.  Streams
 * leave the context's codes, audio and statistics alone, and the context's other calls leave streams alone.
 *   bark_b200_encodec_stream_open ........ NULL with a message for a null context, an unknown direction, an encode without encoder tensors
 *                                          or a bandwidth the file cannot give
 *   bark_b200_encodec_stream_push ........ encode: in = n float samples; decode: in = n frames of codes [n_q][n], codebook-major.  Returns
 *                                          the outputs that became final (frames, or samples), waiting for read; -1 refused
 *   bark_b200_encodec_stream_push_batch .. count <= 32 streams of one context and one direction in one pass of the kernels, stream i
 *                                          pushed in[i], n[i]; each gets exactly what its own push would have.  Returns the sum
 *   bark_b200_encodec_stream_read ........ takes k = min(ready, cap) final outputs to out: codes [n_q][k] for k frames, or k samples;
 *                                          returns k (out NULL: only returns the count ready, taking nothing), -1 for a null stream
 *   bark_b200_encodec_stream_finish ...... ends the stream: returns the outputs it added, -1 refused (the stream is unchanged)
 *   bark_b200_encodec_stream_codebooks ... the stream's n_q
 *   bark_b200_encodec_stream_close ....... frees the stream; close every stream before encodec_free of its context
 * A push or finish is refused with a message, leaving every stream of the call exactly as it was, for a null argument, a negative count,
 * a non-finite sample, a code outside [0, n_bins), a finished stream, or a batch that mixes contexts or directions, repeats a stream or
 * holds more than 32.  The refused call followed by the corrected one gives the same bits as the corrected one alone. */
#define BARK_B200_STREAM_ENCODE 0
#define BARK_B200_STREAM_DECODE 1
#define BARK_B200_STREAM_MAX_BATCH 32
struct bark_b200_encodec_stream;
BARK_API struct bark_b200_encodec_stream * bark_b200_encodec_stream_open(struct encodec_context * e, int direction);
BARK_API int  bark_b200_encodec_stream_push(struct bark_b200_encodec_stream * s, const void * in, int n);
BARK_API int  bark_b200_encodec_stream_push_batch(struct bark_b200_encodec_stream * const * s, const void * const * in, const int * n, int count);
BARK_API int  bark_b200_encodec_stream_read(struct bark_b200_encodec_stream * s, void * out, int cap);
BARK_API int  bark_b200_encodec_stream_finish(struct bark_b200_encodec_stream * s);
BARK_API long long bark_b200_encodec_stream_ready(int direction, long long n);
BARK_API int  bark_b200_encodec_stream_codebooks(struct bark_b200_encodec_stream * s);
BARK_API void bark_b200_encodec_stream_close(struct bark_b200_encodec_stream * s);

/* RESAMPLED STREAMS (DESIGN.md §20): a stream at any sample rate and channel count, as the RESAMPLED ENCODEC calls take whole clips.
 * encode: in = n interleaved frames [n][channels] at sample_rate (1 <= channels <= 8, 4000 <= sample_rate <= 384000), down-mixed and
 *         resampled to 24 kHz on the GPU, then encoded; the n of a push counts frames.  Everything returned, joined, equals
 *         bark_b200_encodec_compress_resampled(e, all frames, n, channels, sample_rate) bit for bit.
 * decode: channels must be 1; the samples read back are at sample_rate, and everything returned, joined, equals
 *         bark_b200_resample(encodec_decompress_audio's 320 T samples, 320 T, 1, 24000, sample_rate) bit for bit.
 * Mono 24 kHz is the plain stream, bit for bit and in readiness.  push, push_batch, read, finish, codebooks and close take these streams
 * unchanged; a push_batch may mix formats and plain streams (one context, one direction), each stream getting what its own push would.
 * Readiness, an integer closed form of the rates: with o = sr / g, q = new_sr / g (g = gcd) and w = ceil(6 o / (0.99 min(o, q))) the
 * filter's half width (§16), output k q + j reads the frames k o - w .. k o + o + w - 1, so after n input frames
 *   R(n) = q * max(0, floor((n - w) / o)) resampled samples are final (R(n) = n for equal rates).
 *   encode: after n frames, bark_b200_encodec_stream_ready(ENCODE, R(n)) code frames are final (48 kHz: w = 13, o = 2, so the first
 *           frame needs 4493 frames; 44.1 kHz: w = 12, o = 147);
 *   decode: after n code frames, R'(bark_b200_encodec_stream_ready(DECODE, n)) samples are final, R' for 24000 -> sample_rate.
 * finish: an encode resamples its tail up to L = ceil(q n / o) with zeros past the last frame, as the whole clip does, and finishes the
 * encoder on L samples; it refuses L < 1921 (at 48 kHz 3840 frames are refused, 3841 accepted).  A decode refuses T < 7 as before and
 * adds the resampler's tail up to ceil(q' 320 T / o').  On top of the plain streams' refusals: open refuses channels outside 1..8, a
 * rate outside 4000..384000 and a decode with channels != 1 (NULL with a message); a push refuses n * channels >= 2^31 and a sample
 * with |x| > 2^64, leaving every stream of the call unchanged.  The state stays O(1) in the stream's length: the resampler keeps at most
 * 2w + o - 1 frames and its own copy of the rate pair's taps (18 MB at 383999 Hz).
 *   bark_b200_encodec_stream_open_resampled ... a stream at that format
 *   bark_b200_encodec_stream_ready_resampled .. the rule above: the outputs final after n inputs (frames, or code frames) before
 *                                               finish; -1 for an unknown direction, a rate outside the limits or n < 0
 *   bark_b200_resample_window .................. no context, host buffers, for the tests: n <= 32 items of their own channels[b] and
 *                                               rates in_rates[b] -> out_rates[b] in one launch.  Item b's n_frames[b] interleaved
 *                                               frames (in, item after item) are the global frames org[b] ..; out (item after item)
 *                                               gets its n_out[b] global outputs from first[b] on.  Frames below 0, and at or past
 *                                               end[b] where end is not NULL and end[b] >= 0, read as zeros.  Returns 1, 0 on invalid
 *                                               arguments or a window whose outputs read a frame it does not hold, -1 if a store
 *                                               landed in the guard bands around the output. */
BARK_API struct bark_b200_encodec_stream * bark_b200_encodec_stream_open_resampled(struct encodec_context * e, int direction, int channels, int sample_rate);
BARK_API long long bark_b200_encodec_stream_ready_resampled(int direction, int sample_rate, long long n);
BARK_API int  bark_b200_resample_window(const float * in, const int * n_frames, const int * channels, const int * in_rates, const int * out_rates,
                                        const long long * org, const long long * first, const int * n_out, const long long * end, int n, float * out);

/* FAST MODE (BARK_B200_MODE=fast in the environment at load; opt-in, NOT bit-identical to the reference): the fine model's
 * 1024-row passes (bark.cpp:1416-1584) run as wgmma tensor-core GEMMs + flash-style attention (csrc/fast_kernels.cu).
 * Every weight type the loader reads runs it: an f16 file's fine matrices are used as stored; those of an f32, q4_0, q4_1, q5_0, q5_1
 * or q8_0 file are converted once at load to one f16 copy (bark_b200_fast_convert), each element the round to nearest even of the f32
 * the reference's dequantize_row_<type> gives.  A fine weight that is not finite in f16 refuses fast mode for the context, with a
 * message naming it: bark_b200_fast_mode then returns 0 and the parity path runs.
 * The kernel hooks below run on host buffers without a context, for the numerics tests:
 *   bark_b200_fast_gemm ....... A[M][K] (f16 bits) * W[N][K]^T (f16 bits), K % 64 == 0, through the fine pass's epilogue `epilogue`:
 *                                 0 F32     C = f32 [M][N]
 *                                 1 RESID   C = f32 [M][N], holds the residual on entry and residual + A W^T on return
 *                                 2 GELU16  C = f16 [M][N] (bits), GELU of the product
 *                                 4 QKV16   N % 6 == 0; C = f16 [M][2N/3] (columns < 2N/3), then f16 [N/3][M] (columns >= 2N/3, transposed)
 *                               bn: 0 = the tile width the cost model picks, 64 / 128 / 256 = that width forced.
 *                               Returns the tile width that ran, 0 on failure, -1 if a store landed in the guard bands around the output.
 *   bark_b200_fast_attention .. out[n][E] (f16 bits) = soft_max(Q K^T / 8) V per 64-wide head, non-causal, n % 128 == 0
 *   bark_b200_fast_convert .... the load-time conversion: src [n_out][K] of wtype (enum ggml_type) 0 f32, 2 q4_0 (18-byte blocks),
 *                               3 q4_1 (20), 6 q5_0 (22), 7 q5_1 (24) or 8 q8_0 (34) as the model file stores it, K % 32 == 0 -> dst
 *                               [n_out][K] f16 bits; *non_finite = the number of results that are inf or NaN.  Returns 1, 0 on invalid
 *                               arguments or failure, -1 if a store landed in the guard bands around the output. */
BARK_API int  bark_b200_fast_mode(struct bark_context * ctx);              /* 1 if this context runs the fast fine passes */
BARK_API int  bark_b200_fast_gemm(const uint16_t * A, const uint16_t * W, void * C, int M, int N, int K, int epilogue, int bn);
BARK_API int  bark_b200_fast_convert(int wtype, const void * src, int n_out, int K, uint16_t * dst, int * non_finite);
BARK_API int  bark_b200_fast_attention(const uint16_t * q, const uint16_t * k, const uint16_t * v, uint16_t * out, int n, int E, int H);

/* Parity-path attention on host buffers without a context (tests, tools/attn_bench.py): out[N][E] = soft_max(mask(Q K^T / sqrt(E/H))) V
 * per head, bit-identical to the reference's ggml graph, for q [N][E], k / v [n_kv][E] f32, n_kv <= 1024, head size E/H in
 * {32, 64, 96, 128}.  causal != 0 masks key j for query i when j > n_past + i.  path: 0 = the kernels the library picks for this
 * shape, 1 = the fused kernel (scores in shared memory), 2 = the three-kernel path for few rows (N <= 32 * (ceil(SMs / H) - 1)).
 * Returns 1 on success, 0 on failure. */
BARK_API int  bark_b200_parity_attention(const float * q, const float * k, const float * v, float * out, int N, int n_kv, int n_past, int E, int H, int causal,
                                         int path);

/* The batched decode step's attention on host buffers without a context (tests): B <= 8 rows of different sequences, row b the one new
 * query q[b] at position pos[b] of its own sequence, attending over its pos[b] + 1 keys.  q, k_new, v_new: [B][E] f32, the step's query
 * and new K / V rows; k_cache, v_cache: [B][cap][E] f32, row b's caches, cap <= 1024, 0 <= pos[b] < cap, head size E/H in
 * {32, 64, 96, 128}.  The kernels append k_new[b] / v_new[b] at row pos[b] of row b's caches and attend; on return the caches hold
 * rows < pos[b] as given, the appended row, and NaN from pos[b] + 1 on (those rows are NaN while the kernels run).  act: the operand
 * format the result is stored in, 0 f32 rows (quantised models), 1 f16 group-major (f16 models), 2 f32 group-major (f32 models);
 * out: [B][E] row-major, f32, or f16 bits for act 1.  Returns 1, 0 on invalid arguments or failure, -1 if a store landed in the
 * guard bands around the output or a cache. */
BARK_API int  bark_b200_batch_attention(const float * q, const float * k_new, const float * v_new, float * k_cache, float * v_cache, const int32_t * pos,
                                        int B, int cap, int E, int H, int act, void * out);

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

/* Parity-path dense mat-muls on host buffers without a context (tests, tools/gemm_bench.py): C = A W^T with every output the reference's
 * vec_dot of its two rows, for A [M][K] and W [N][K] of wtype 0 (f32) or 1 (f16 bits), K % 32 == 0, through the parity passes'
 * epilogue `epilogue`:
 *   0 STORE     C = f32 [M][N]
 *   1 RESID     C = f32 [M][N], holds the residual on entry and residual + A W^T on return
 *   2 GELU_ACT  C = [M][N] in wtype: GELU of the product through gelu_tab (65536 f16 entries), as the next mat-mul's operand holds it
 *   3 QKV       N % 3 == 0; C = f32 Q [M][N/3], then K [M][N/3], then V [M][N/3]
 * variant: 0 = the kernel the library picks for M rows (the few-row kernel below 16 rows, else the tiled GEMM's block tile for wtype),
 * 1 = the tiled GEMM's 32 x 16 outputs (8 warps, two CTAs per SM), 2 = its 32 x 32 (16 warps, one CTA per SM), 3 = the few-row kernel
 * (one warp per output, 1 or 8 rows per CTA) at any M.  Every padding element of the permuted operands is NaN.  Returns the variant
 * that ran, 0 on failure or invalid arguments, -1 if a store landed in the guard bands around the output. */
BARK_API int  bark_b200_parity_gemm(const void * A, const void * W, void * C, int M, int N, int K, int wtype, int epilogue, int variant,
                                    const uint16_t * gelu_tab);

/* Quantised mat-muls on host buffers without a context (tests): C = A W^T with every output the reference's ggml_vec_dot_<type>_q8_0 /
 * _q8_1 of weight row o against activation row m after quantize_row_q8_0 / q8_1, for A [M][K] f32 and W [N][K/32] blocks as the model
 * file stores them, wtype (enum ggml_type) 2 q4_0 (18-byte blocks), 3 q4_1 (20), 6 q5_0 (22), 7 q5_1 (24) or 8 q8_0 (34), K % 32 == 0.
 * epilogue as bark_b200_parity_gemm (GELU_ACT: f32 [M][N], the operand a quantised model's next mat-mul quantises; QKV: N % 3 == 0).
 *   path 0: the per-op kernels the library runs for M rows (quantize_q8x_kernel + q4_matmul_kernel or qx_matmul_kernel)
 *   path 1 / 2: q4_0, M == 1, K <= 4096 only: the persistent decode step's quantize_act_q8 + row_dot_q4 in one CTA, the weight rows
 *               staged in shared memory (1) or read from global memory (2)
 * q [M][K] int8, d [M][K/32] f32 (the f16 scale, widened), s [M][K/32] f32 (q4_1 / q5_1 only, the f16 q8_1 sum): the quantised
 * activation blocks; each may be NULL.  The calling thread's context is unaffected.  Returns 1, 0 on failure or invalid arguments, -1 if
 * a store landed in the guard bands around the output. */
BARK_API int  bark_b200_quant_matmul(int wtype, const void * W, const float * A, float * C, int M, int N, int K, int epilogue, int path,
                                     const uint16_t * gelu_tab, int8_t * q, float * d, float * s);

/* EnCodec kernels on host buffers without a context (tests), each on n items (1 to 32 clips) of their own lengths, concatenated item by
 * item: item b of an activation [C][L_b] follows items 0..b-1.  f16 weights arrive as the model file stores them and are laid out by
 * the loader's own routines, with every padding element NaN.  Each returns a positive value on success, 0 on invalid arguments, on a
 * shape the launcher refuses (with a message) or on failure, -1 if a store landed in the guard bands around the output.
 *   bark_b200_codec_conv1d ....... strided_conv_1d: x [Cin][L_b] (ELU'd first when elu_in) -> y [Cout][T_b], T_b the reference's output
 *                                  length (L_b at stride 1), w [Cout][Cin][k] f16, bias [Cout], resid (stride 1 only, may be NULL)
 *                                  [Cout][T_b] added to the result; L_b > k - stride (refused by the launcher above stride 1).  Returns the kernel that ran: 1 conv1d_short_kernel,
 *                                  1000 + 10 KW + NG conv1d_lane_kernel<KW, NG>, 10000 + 100 KW + STRIDE conv1d_stream_kernel<KW, STRIDE>.
 *   bark_b200_codec_convtr1d ..... ELU, then strided_conv_transpose_1d with k = 2 stride, right-trimmed: x [Cin][T_b] -> y [Cout][T_b stride],
 *                                  w [Cin][Cout][k] f16, bias [Cout].  Returns the NG of convtr1d_lane_kernel<NG>.
 *   bark_b200_codec_lstm ......... one LSTM layer: x [C][T_b] -> out [C][T_b] (plus skip [C][T_b] when not NULL), wih / whh [4C][C] f16,
 *                                  bih / bhh [4C].  Returns 1 for the one-item recurrence, 2 for the batched one.
 *   bark_b200_codec_rvq_decode ... codes [n_q][T_b] (each in [0, n_bins)) through codebooks [n_q][n_bins][hidden] f32 -> x [hidden][T_b].
 * bark_b200_device_math evaluates one device function of the codec and soft_max, fn 0 glibc expm1f, 1 tanhf, 2 expf (restated), 3 ggml's
 * AVX2 ggml_v_expf, 4 ELU, 5 the sigmoid, 6 the round trip through f16, on the floats of bit patterns lo_bits + i * stride (mod 2^32),
 * i < count <= 2^24, into out [count].  Returns 1, 0 on invalid arguments or failure, -1 on a guard band store. */
BARK_API int  bark_b200_codec_conv1d(const float * x, int Cin, const int * L, int n, const uint16_t * w, const float * bias, int Cout, int k, int stride,
                                     int elu_in, const float * resid, float * y);
BARK_API int  bark_b200_codec_convtr1d(const float * x, int Cin, const int * T, int n, const uint16_t * w, const float * bias, int Cout, int stride,
                                       float * y);
BARK_API int  bark_b200_codec_lstm(const float * x, int C, const int * T, int n, const uint16_t * wih, const uint16_t * whh, const float * bih,
                                   const float * bhh, const float * skip, float * out);
BARK_API int  bark_b200_codec_rvq_decode(const int32_t * codes, int n_q, const int * T, int n, const float * codebooks, int hidden, int n_bins, float * x);
BARK_API int  bark_b200_device_math(int fn, uint32_t lo_bits, uint32_t stride, uint32_t count, float * out);
/* The same launchers over a window of each item's signal, as the streams run them (DESIGN.md §19): item b's columns [C][L_b] are the
 * global positions org[b] .. org[b] + L_b - 1 of its signal, and outputs first[b] .. first[b] + n_out[b] - 1 are computed, concatenated as
 * [Cout][n_out[b]] (the transposed conv: [Cout][n_out[b] stride], output frames of input frames).  Reflections apply where the global
 * position is outside the signal: below 0, and (strided convs) past the window's last column.  A window whose outputs read a column it
 * does not hold is refused.  Each equals the matching slice of the whole-signal hook's result.
 *   bark_b200_codec_conv1d_window .... bark_b200_codec_conv1d over windows; resid [Cout][n_out[b]] (stride 1, may be NULL)
 *   bark_b200_codec_convtr1d_window .. bark_b200_codec_convtr1d over windows; output frame t reads frames t - 1 (none for t = 0) and t
 *   bark_b200_codec_lstm_state ....... bark_b200_codec_lstm from the state (h, c) [n][2][C] (NULL: zeros), which on return holds each
 *                                      item's state after its last step */
BARK_API int  bark_b200_codec_conv1d_window(const float * x, int Cin, const int * L, int n, const long long * org, const long long * first, const int * n_out,
                                            const uint16_t * w, const float * bias, int Cout, int k, int stride, int elu_in, const float * resid, float * y);
BARK_API int  bark_b200_codec_convtr1d_window(const float * x, int Cin, const int * L, int n, const long long * org, const long long * first, const int * n_out,
                                              const uint16_t * w, const float * bias, int Cout, int stride, float * y);
BARK_API int  bark_b200_codec_lstm_state(const float * x, int C, const int * T, int n, const uint16_t * wih, const uint16_t * whh, const float * bih,
                                         const float * bhh, const float * skip, float * state, float * out);

#ifdef __cplusplus
}
#endif
