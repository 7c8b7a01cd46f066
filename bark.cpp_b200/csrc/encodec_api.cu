// encodec.cpp's C API (include/encodec.h) on the EnCodec pipelines that bark_context uses (gpt_forward.cu): an encodec_context owns a
// stream, the codec weights with all the file's codebooks and their norms, the codec scratch and the output vectors, and no GPT.
// Semantics follow encodec.cpp/encodec.cpp:933-1050; the inputs the reference asserts on or cannot run are refused with a message.
#include "../../include/encodec.h"
#include "context.h"
#include "codec_kernels.h"

#include <cmath>
#include <cstring>

using namespace bark;

struct encodec_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    CodecModel model;
    CodecScratch scratch;
    DeviceArena arena;
    int bandwidth = 0, sample_rate = 0;              // encodec_set_target_bandwidth / encodec_set_sample_rate; the file's at load
    std::vector<int32_t> codes;                      // [n_q][T] of the last compress
    std::vector<float> audio;                        // the last decompress / reconstruct
    encodec_statistics stats{};
};

namespace {

constexpr int kHop = 320;                            // product of the 24 kHz model's ratios 8, 5, 4, 2

// get_num_quantizers_for_bandwidth (encodec.cpp/utils.h:22-30) as encodec.cpp:650-651 calls it; false (message) where the reference
// divides by zero or would need more codebooks than the file has
bool codebooks_for(const encodec_context * e, const char * caller, int * n_q) {
    if (e->sample_rate < kHop) { fprintf(stderr, "%s: sample rate %d is below the hop length %d (frame rate 0)\n", caller, e->sample_rate, kHop); return false; }
    const int frame_rate = (int) ceilf((float)(e->sample_rate / kHop));
    const float bw_per_q = (float)(int32_t)(log2f((float) e->model.n_bins) * (float) frame_rate);
    if (!(bw_per_q > 0.0f)) { fprintf(stderr, "%s: %d codebook bins carry no bandwidth\n", caller, e->model.n_bins); return false; }
    const float q = fmaxf(1.0f, floorf((float) e->bandwidth * 1000.0f / bw_per_q));
    if (q > (float) e->model.n_q) {
        fprintf(stderr, "%s: bandwidth %d kbps at %d Hz needs %.0f codebooks; the file has %d\n", caller, e->bandwidth, e->sample_rate, q, e->model.n_q);
        return false;
    }
    *n_q = (int) q;
    return true;
}

// runs f with the context's device current; a CUDA failure or exception is a failed call (message on stderr)
template <typename F> bool run(encodec_context * e, const char * caller, F && f) {
    if (!e) { fprintf(stderr, "%s: null context\n", caller); return false; }
    const int64_t t0 = now_us();
    const bool ok = guarded(false, [&] { BARK_CUDA_CHECK(cudaSetDevice(e->device)); return f(); });
    if (ok) e->stats.t_compute_us = now_us() - t0;
    return ok;
}

}  // namespace

extern "C" struct encodec_context * encodec_load_model(const char * model_path, const int offset, int n_gpu_layers) {
    (void) n_gpu_layers;                             // the whole model runs on the GPU
    const int64_t t0 = now_us();
    if (!model_path) { fprintf(stderr, "%s: null model path\n", __func__); return nullptr; }
    std::ifstream f(model_path, std::ios::binary);
    if (!f) { fprintf(stderr, "%s: failed to open '%s'\n", __func__, model_path); return nullptr; }
    if (offset > 0) f.seekg(offset);                 // encodec.cpp:944-946
    cudaDeviceProp prop;
    const int dev = select_device(__func__, &prop);
    if (dev < 0) return nullptr;
    encodec_context * e = new encodec_context();
    e->device = dev;
    const bool ok = guarded(false, [&] {
        BARK_CUDA_CHECK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
        return load_codec(f, e->model, kMaxCodebooks, e->arena, e->stream, false);
    });
    if (!ok) {
        fprintf(stderr, "%s: failed to load model weights from '%s'\n", __func__, model_path);
        encodec_free(e);
        return nullptr;
    }
    e->bandwidth = e->model.bandwidth; e->sample_rate = e->model.sample_rate;
    e->stats.t_load_us = now_us() - t0;
    return e;
}

extern "C" void encodec_set_target_bandwidth(struct encodec_context * e, int bandwidth) { if (e) e->bandwidth = bandwidth; }
extern "C" void encodec_set_sample_rate(struct encodec_context * e, int sample_rate) { if (e) e->sample_rate = sample_rate; }

extern "C" bool encodec_compress_audio(struct encodec_context * e, const float * raw_audio, const int n_samples, int) {
    return run(e, __func__, [&] {
        int n_q;
        if (!raw_audio) { fprintf(stderr, "encodec_compress_audio: null input audio\n"); return false; }
        if (!codebooks_for(e, "encodec_compress_audio", &n_q)) return false;
        std::vector<int32_t> codes;
        if (!codec_encode(e->model, e->scratch, e->stream, raw_audio, n_samples, n_q, &codes, nullptr)) return false;
        e->codes.swap(codes);
        return true;
    });
}

extern "C" bool encodec_decompress_audio(struct encodec_context * e, const int32_t * codes, const int n_codes, int) {
    return run(e, __func__, [&] {
        int n_q;
        if (!codes) { fprintf(stderr, "encodec_decompress_audio: null codes\n"); return false; }
        if (!codebooks_for(e, "encodec_decompress_audio", &n_q)) return false;
        if (n_codes < 0 || n_codes % n_q != 0) { fprintf(stderr, "encodec_decompress_audio: %d codes are not a whole number of frames of %d codebooks\n", n_codes, n_q); return false; }
        std::vector<float> audio;
        if (!codec_decode(e->model, e->scratch, e->stream, codes, n_q, n_codes / n_q, audio)) return false;
        e->audio.swap(audio);
        return true;
    });
}

extern "C" bool encodec_reconstruct_audio(struct encodec_context * e, const float * raw_audio, const int n_samples, int) {
    return run(e, __func__, [&] {
        int n_q;
        if (!raw_audio) { fprintf(stderr, "encodec_reconstruct_audio: null input audio\n"); return false; }
        if (!codebooks_for(e, "encodec_reconstruct_audio", &n_q)) return false;
        if (!codec_encode(e->model, e->scratch, e->stream, raw_audio, n_samples, n_q, nullptr, nullptr)) return false;
        std::vector<float> audio;                    // decodes the codes codec_encode left in the scratch (encodec.cpp:592-602)
        if (!codec_decode(e->model, e->scratch, e->stream, nullptr, n_q, (n_samples - 1) / kHop + 1, audio)) return false;
        e->audio.swap(audio);
        return true;
    });
}

extern "C" float * encodec_get_audio(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return nullptr; }
    return e->audio.data();
}
extern "C" int encodec_get_audio_size(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return 0; }
    return (int) e->audio.size();
}
extern "C" int32_t * encodec_get_codes(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return nullptr; }
    return e->codes.data();
}
extern "C" int encodec_get_codes_size(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return 0; }
    return (int) e->codes.size();
}
extern "C" const struct encodec_statistics * encodec_get_statistics(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return nullptr; }
    return &e->stats;
}
extern "C" void encodec_reset_statistics(struct encodec_context * e) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return; }
    memset(&e->stats, 0, sizeof(e->stats));          // encodec.cpp:1012, load time included
}

extern "C" void encodec_free(struct encodec_context * e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    e->arena.release();
    e->scratch.release();
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}
