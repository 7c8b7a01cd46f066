/* bark.h — C API of the H100-native bark hot path.
 *
 * Declaration-for-declaration compatible with the reference header (bark.h:34-244 of PABannier/bark.cpp):
 * same enum values, same field order and types in bark_statistics / bark_context_params (the
 * params struct is passed BY VALUE, so its layout is ABI), same eleven entry points.  Callers such
 * as examples/main/main.cpp and examples/server/server.cpp compile against this header unchanged
 * (they also include "ggml.h" for ggml_time_* / enum ggml_ftype: include/ggml.h is a shim that
 * provides exactly those).
 *
 * Everything behind these functions runs as hand-written sm_90a CUDA; there is no CPU fallback:
 * bark_load_model fails (nullptr + message on stderr) when no CUDA device is usable.
 */
#pragma once

#include "encodec.h"
#include "ggml-backend.h"
#include "ggml.h"

#include <stdbool.h>
#include <stdint.h>

#if defined(_WIN32)
#  if defined(EXPORTING_BARK)
#    define BARK_API __declspec(dllexport)
#  else
#    define BARK_API __declspec(dllimport)
#  endif
#else
#  define BARK_API __attribute__((visibility("default")))
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* reference bark.h:37-41 */
enum bark_verbosity_level { LOW = 0, MEDIUM = 1, HIGH = 2 };
/* reference bark.h:43-47 */
enum bark_encoding_step { SEMANTIC = 0, COARSE = 1, FINE = 2 };

struct bark_context;
struct bark_model;
struct bark_vocab;
struct gpt_model;

/* reference bark.h:58 — invoked synchronously on the caller's thread once per generation step */
typedef void (*bark_progress_callback)(struct bark_context * bctx, enum bark_encoding_step step, int progress, void * user_data);

/* reference bark.h:60-79 (microseconds / sample counts) */
struct bark_statistics {
    int64_t t_load_us;
    int64_t t_eval_us;
    int64_t t_semantic_us;
    int64_t t_coarse_us;
    int64_t t_fine_us;
    int32_t n_sample_semantic;
    int32_t n_sample_coarse;
    int32_t n_sample_fine;
};

/* reference bark.h:81-141 — 25 fields, order is ABI */
struct bark_context_params {
    enum bark_verbosity_level verbosity;
    float   temp;                       /* semantic + coarse sampling temperature */
    float   fine_temp;                  /* fine sampling temperature */
    float   min_eos_p;                  /* semantic early stop threshold */
    int32_t sliding_window_size;        /* coarse window length (60) */
    int32_t max_coarse_history;         /* coarse history fed per window (630) */
    int32_t sample_rate;                /* 24000 */
    int32_t target_bandwidth;           /* 6 kbps -> 8 codebooks */
    int32_t cls_token_id;
    int32_t sep_token_id;
    int32_t n_steps_text_encoder;       /* max semantic tokens (768) */
    int32_t text_pad_token;
    int32_t text_encoding_offset;
    float   semantic_rate_hz;
    int32_t semantic_pad_token;
    int32_t semantic_vocab_size;
    int32_t semantic_infer_token;
    float   coarse_rate_hz;
    int32_t coarse_infer_token;
    int32_t coarse_semantic_pad_token;
    int32_t n_coarse_codebooks;
    int32_t n_fine_codebooks;
    int32_t codebook_size;
    bark_progress_callback progress_callback;
    void *  progress_callback_user_data;
};

BARK_API struct bark_context_params bark_context_default_params(void);                       /* ref bark.cpp:2202 */
BARK_API struct bark_context * bark_load_model(const char * model_path,
                                               struct bark_context_params params,
                                               uint32_t seed);                               /* ref bark.cpp:1165 */
BARK_API bool    bark_generate_audio(struct bark_context * bctx, const char * text, int n_threads); /* ref bark.cpp:2125; n_threads accepted and ignored */
BARK_API float * bark_get_audio_data(struct bark_context * bctx);                            /* ref bark.cpp:2379; borrowed until next generate/free */
BARK_API int     bark_get_audio_data_size(struct bark_context * bctx);                       /* ref bark.cpp:2385 */
BARK_API int64_t bark_get_load_time(struct bark_context * bctx);                             /* ref bark.cpp:2391 */
BARK_API int64_t bark_get_eval_time(struct bark_context * bctx);                             /* ref bark.cpp:2397 */
BARK_API void    bark_reset_statistics(struct bark_context * bctx);                          /* ref bark.cpp:2403 */
BARK_API bool    bark_model_quantize(const char * fname_inp, const char * fname_out, enum ggml_ftype ftype); /* ref bark.cpp:2300 */
BARK_API void    bark_free(struct bark_context * bctx);                                      /* ref bark.cpp:2189 */

#ifdef __cplusplus
}
#endif
