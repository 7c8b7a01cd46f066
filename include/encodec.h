/* encodec.h — encodec.cpp's C API (encodec.cpp/encodec.h of PABannier/encodec.cpp), served by libbark_b200.
 *
 * Same thirteen functions with the same signatures and the same encodec_statistics layout, so encodec.cpp's callers
 * (examples/{compress,decompress,main}) compile against include/ unchanged and link -lbark_b200 instead of encodec + ggml.
 * The 24 kHz mono model runs on the GPU as hand-written sm_90a CUDA; there is no CPU path: encodec_load_model returns NULL
 * (message on stderr) without a usable H100.  bark.h includes this header, as the reference's does.
 *
 * Semantics follow the reference, except that every input it would assert on, read out of bounds with or divide by zero
 * (see DESIGN.md §13) makes the call return false / NULL with a message and leaves the context usable.
 *   - The number of codebooks n_q follows the reference's rule: frame_rate = ceil(sample_rate / 320) with integer division,
 *     bw_per_q = (int)(log2(n_bins) * frame_rate), n_q = max(1, floor(bandwidth * 1000 / bw_per_q)).  At 24 kHz, bandwidth
 *     1, 2, 3, 6, 12, 24 gives 1, 2, 4, 8, 16, 32 codebooks.  A fresh context runs at the file's bandwidth (24).
 *   - Codes are [n_q][T] codebook-major, T = ceil(n_samples / 320); audio is 320 T samples.  The getters' pointers stay valid
 *     until the next call on the context or encodec_free.
 *   - n_threads and n_gpu_layers are accepted and ignored; the device is chosen like bark_load_model's (bark_b200_set_device,
 *     else the BARK_B200_DEVICE environment variable, else 0).
 * One context is used by one thread at a time. */
#pragma once

#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml.h"

#include <stdbool.h>
#include <stdint.h>

#if defined(_WIN32)
#  if defined(EXPORTING_BARK)
#    define ENCODEC_API __declspec(dllexport)
#  else
#    define ENCODEC_API __declspec(dllimport)
#  endif
#else
#  define ENCODEC_API __attribute__((visibility("default")))
#endif

#ifdef __cplusplus
extern "C" {
#endif

struct encodec_context;

struct encodec_statistics {
    int64_t t_load_us;        /* wall time of encodec_load_model */
    int64_t t_compute_us;     /* wall time of the last compress, decompress or reconstruct call */
};

/* offset: byte position of the codec section (0 for a standalone encodec.cpp file; a bark weight file's codec section otherwise) */
ENCODEC_API struct encodec_context * encodec_load_model(const char * model_path, const int offset, int n_gpu_layers);
ENCODEC_API void encodec_set_target_bandwidth(struct encodec_context * ectx, int bandwidth);     /* kbps; changes n_q only */
ENCODEC_API void encodec_set_sample_rate(struct encodec_context * ectx, int sample_rate);       /* Hz; changes n_q only */
/* audio -> codes -> audio, the codes staying on the device */
ENCODEC_API bool encodec_reconstruct_audio(struct encodec_context * ectx, const float * raw_audio, const int n_samples, int n_threads);
/* audio (n_samples >= 1921, finite) -> codes [n_q][T] */
ENCODEC_API bool encodec_compress_audio(struct encodec_context * ectx, const float * raw_audio, const int n_samples, int n_threads);
/* codes [n_q][T] (n_codes = n_q T, T >= 7, each in [0, n_bins)) -> audio */
ENCODEC_API bool encodec_decompress_audio(struct encodec_context * ectx, const int32_t * codes, const int n_codes, int n_threads);
ENCODEC_API float * encodec_get_audio(struct encodec_context * ectx);
ENCODEC_API int encodec_get_audio_size(struct encodec_context * ectx);
ENCODEC_API int32_t * encodec_get_codes(struct encodec_context * ectx);
ENCODEC_API int encodec_get_codes_size(struct encodec_context * ectx);
ENCODEC_API const struct encodec_statistics * encodec_get_statistics(struct encodec_context * ectx);
ENCODEC_API void encodec_reset_statistics(struct encodec_context * ectx);
ENCODEC_API void encodec_free(struct encodec_context * ectx);

#ifdef __cplusplus
}
#endif
