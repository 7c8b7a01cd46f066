// encodec.cpp's C API (include/encodec.h) on the EnCodec pipelines that bark_context uses (codec_pipeline.cu): an encodec_context owns a
// stream, the codec weights with all the file's codebooks and their norms, the codec scratch and the output vectors, and no GPT.
// Semantics follow encodec.cpp/encodec.cpp:933-1050; the inputs the reference asserts on or cannot run are refused with a message.
#include "../../include/encodec.h"
#include "../../include/bark_b200.h"
#include "context.h"
#include "codec_kernels.h"

#include <algorithm>
#include <climits>
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
    std::vector<std::vector<int32_t>> batch_codes;   // per item: the last successful bark_b200_encodec_compress_batch
    std::vector<std::vector<float>> batch_audio;     // per item: the last successful decompress / reconstruct batch
    encodec_statistics stats{};
};

namespace {

// get_num_quantizers_for_bandwidth (encodec.cpp/utils.h:22-30) as encodec.cpp:650-651 calls it; false (message) where the reference
// divides by zero or would need more codebooks than the file has
bool codebooks_for(const encodec_context * e, const char * caller, int * n_q) {
    if (e->sample_rate < kCodecHop) { fprintf(stderr, "%s: sample rate %d is below the hop length %d (frame rate 0)\n", caller, e->sample_rate, kCodecHop); return false; }
    const int frame_rate = (int) ceilf((float)(e->sample_rate / kCodecHop));
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

// n and the arrays of a batch call: false (message) for n outside [1, BARK_B200_ENCODEC_MAX_BATCH] or a null array or entry
template <typename P> bool batch_args(const char * caller, const P * const * items, const int * lens, int n) {
    if (n < 1 || n > BARK_B200_ENCODEC_MAX_BATCH) { fprintf(stderr, "%s: %d items (1 to %d per batch)\n", caller, n, BARK_B200_ENCODEC_MAX_BATCH); return false; }
    if (!items || !lens) { fprintf(stderr, "%s: null %s\n", caller, items ? "length array" : "item array"); return false; }
    for (int i = 0; i < n; i++) if (!items[i]) { fprintf(stderr, "%s: item %d is null\n", caller, i); return false; }
    return true;
}

// a batch call with per-item formats: batch_args' checks, then the two format arrays
bool resampled_batch_formats(const char * fn, const float * const * audio, const int * n_frames, const int * channels, const int * sample_rates, int n,
                             std::vector<AudioFormat> * fmt) {
    if (!batch_args(fn, audio, n_frames, n)) return false;
    if (!channels || !sample_rates) { fprintf(stderr, "%s: null %s\n", fn, channels ? "sample rate array" : "channel array"); return false; }
    fmt->resize((size_t) n);
    for (int i = 0; i < n; i++) (*fmt)[(size_t) i] = AudioFormat{channels[i], sample_rates[i]};
    return true;
}

// The clips of an encoder call: n arrays of lens[i] mono 24 kHz samples, or for a resampled call lens[i] frames of channels[i] channels
// at rates[i] Hz (one of each for a single call)
struct Clips {
    int n; const float * const * audio; const int * lens;
    bool resampled = false; const int * channels = nullptr, * rates = nullptr;
};
enum Keep { kKeepCodes, kKeepAudio };

// The eight encoder calls, named fn: the single call's null check, or batch_args (and the format arrays of a resampled batch), then the
// bandwidth's codebooks; then the pipeline, whose codes or waveforms replace the context's results of the same kind, single or batch
bool encode(encodec_context * e, const char * fn, bool batch, const Clips & c, Keep keep) {
    return run(e, fn, [&] {
        std::vector<AudioFormat> fmt;
        if (!batch && !c.audio[0]) { fprintf(stderr, "%s: null input audio\n", fn); return false; }
        if (batch && !(c.resampled ? resampled_batch_formats(fn, c.audio, c.lens, c.channels, c.rates, c.n, &fmt) : batch_args(fn, c.audio, c.lens, c.n))) return false;
        if (!batch && c.resampled) fmt.push_back(AudioFormat{*c.channels, *c.rates});
        int n_q;
        if (!codebooks_for(e, fn, &n_q)) return false;
        std::vector<std::vector<int32_t>> codes((size_t) c.n);
        std::vector<std::vector<float>> audio((size_t) c.n);
        CodecOutputs out;
        if (keep == kKeepCodes) out.codes = codes.data(); else out.audio = audio.data();
        if (!codec_encode(e->model, e->scratch, e->stream, c.n, c.audio, c.lens, n_q, out, batch ? fn : nullptr, c.resampled ? fmt.data() : nullptr)) return false;
        if (batch && keep == kKeepCodes) e->batch_codes.swap(codes);
        else if (batch) e->batch_audio.swap(audio);
        else if (keep == kKeepCodes) e->codes.swap(codes[0]);
        else e->audio.swap(audio[0]);
        return true;
    });
}

// The two decoder calls: n_codes[i] codes [n_q][T_i] per item, n_q of the bandwidth
bool decode(encodec_context * e, const char * fn, bool batch, int n, const int32_t * const * codes, const int * n_codes) {
    return run(e, fn, [&] {
        if (!batch && !codes[0]) { fprintf(stderr, "%s: null codes\n", fn); return false; }
        int n_q;
        if ((batch && !batch_args(fn, codes, n_codes, n)) || !codebooks_for(e, fn, &n_q)) return false;
        std::vector<int> T((size_t) n);
        for (int i = 0; i < n; i++) {
            if (n_codes[i] < 0 || n_codes[i] % n_q != 0) {
                fprintf(stderr, "%s: %s%d codes are not a whole number of frames of %d codebooks\n", fn, item_tag(batch ? fn : nullptr, i).c_str(), n_codes[i], n_q);
                return false;
            }
            T[(size_t) i] = n_codes[i] / n_q;
        }
        std::vector<std::vector<float>> audio((size_t) n);
        if (!codec_decode(e->model, e->scratch, e->stream, n, codes, T.data(), n_q, audio.data(), batch ? fn : nullptr)) return false;
        if (batch) e->batch_audio.swap(audio);
        else e->audio.swap(audio[0]);
        return true;
    });
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
    return encode(e, __func__, false, {1, &raw_audio, &n_samples}, kKeepCodes);
}
extern "C" bool encodec_decompress_audio(struct encodec_context * e, const int32_t * codes, const int n_codes, int) {
    return decode(e, __func__, false, 1, &codes, &n_codes);
}
extern "C" bool encodec_reconstruct_audio(struct encodec_context * e, const float * raw_audio, const int n_samples, int) {
    return encode(e, __func__, false, {1, &raw_audio, &n_samples}, kKeepAudio);   // decodes the codes the encode left on the device
}

// ---- batched calls (include/bark_b200.h, BATCHED ENCODEC) ----------------------------------------------------------------------
extern "C" bool bark_b200_encodec_compress_batch(struct encodec_context * e, const float * const * audio, const int * n_samples, int n) {
    return encode(e, __func__, true, {n, audio, n_samples}, kKeepCodes);
}
extern "C" bool bark_b200_encodec_decompress_batch(struct encodec_context * e, const int32_t * const * codes, const int * n_codes, int n) {
    return decode(e, __func__, true, n, codes, n_codes);
}
extern "C" bool bark_b200_encodec_reconstruct_batch(struct encodec_context * e, const float * const * audio, const int * n_samples, int n) {
    return encode(e, __func__, true, {n, audio, n_samples}, kKeepAudio);
}

// ---- resampled calls (include/bark_b200.h, RESAMPLED ENCODEC) -------------------------------------------------------------------
extern "C" bool bark_b200_encodec_compress_resampled(struct encodec_context * e, const float * audio, int n_frames, int channels, int sample_rate) {
    return encode(e, __func__, false, {1, &audio, &n_frames, true, &channels, &sample_rate}, kKeepCodes);
}
extern "C" bool bark_b200_encodec_reconstruct_resampled(struct encodec_context * e, const float * audio, int n_frames, int channels, int sample_rate) {
    return encode(e, __func__, false, {1, &audio, &n_frames, true, &channels, &sample_rate}, kKeepAudio);
}
extern "C" bool bark_b200_encodec_compress_batch_resampled(struct encodec_context * e, const float * const * audio, const int * n_frames, const int * channels,
                                                           const int * sample_rates, int n) {
    return encode(e, __func__, true, {n, audio, n_frames, true, channels, sample_rates}, kKeepCodes);
}
extern "C" bool bark_b200_encodec_reconstruct_batch_resampled(struct encodec_context * e, const float * const * audio, const int * n_frames, const int * channels,
                                                              const int * sample_rates, int n) {
    return encode(e, __func__, true, {n, audio, n_frames, true, channels, sample_rates}, kKeepAudio);
}

extern "C" int bark_b200_encodec_batch_codes(struct encodec_context * e, int i, int32_t * out, int cap) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return -1; }
    return i < 0 || i >= (int) e->batch_codes.size() ? -1 : copy_out(e->batch_codes[(size_t) i], out, cap);
}

extern "C" int bark_b200_encodec_batch_audio(struct encodec_context * e, int i, float * out, int cap) {
    if (!e) { fprintf(stderr, "%s: null context\n", __func__); return -1; }
    return i < 0 || i >= (int) e->batch_audio.size() ? -1 : copy_out(e->batch_audio[(size_t) i], out, cap);
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

// ---- streaming (include/bark_b200.h, STREAMING ENCODEC; DESIGN.md §19) ----------------------------------------------------------
static_assert(BARK_B200_STREAM_MAX_BATCH == kCodecMaxItems, "a batch of streams is one pass of the codec kernels");
struct bark_b200_encodec_stream {
    encodec_context * e;
    CodecStream st;
};

namespace {

// The checks of a push or finish on `count` streams (after which nothing can refuse it): false (message naming fn) for a null or
// repeated stream, streams of several contexts or directions, a finished stream, or a count outside [1, kCodecMaxItems]; with in and n,
// a null chunk, a negative count, a non-finite sample (on a resampled encode: n * channels >= 2^31, or |x| > 2^64, the limits of
// resample_input_ok) or a code outside the codebooks
bool stream_args(const char * fn, bark_b200_encodec_stream * const * s, const void * const * in, const int * n, int count) {
    if (!s || count < 1 || count > kCodecMaxItems) { fprintf(stderr, "%s: %d streams (1 to %d per call)\n", fn, s ? count : 0, kCodecMaxItems); return false; }
    for (int i = 0; i < count; i++) {
        const std::string tag = count > 1 ? "stream " + std::to_string(i) + ": " : std::string();
        if (!s[i]) { fprintf(stderr, "%s: %snull stream\n", fn, tag.c_str()); return false; }
        for (int j = 0; j < i; j++) if (s[j] == s[i]) { fprintf(stderr, "%s: stream %d is stream %d again\n", fn, i, j); return false; }
        if (s[i]->e != s[0]->e || s[i]->st.direction != s[0]->st.direction) { fprintf(stderr, "%s: %sanother context or direction than stream 0\n", fn, tag.c_str()); return false; }
        if (s[i]->st.finished) { fprintf(stderr, "%s: %sthe stream is finished\n", fn, tag.c_str()); return false; }
        if (s[i]->st.failed) { fprintf(stderr, "%s: %sthe stream failed earlier and has lost its state\n", fn, tag.c_str()); return false; }
        if (!in) continue;
        if (!in[i] || n[i] < 0) { fprintf(stderr, "%s: %s%s\n", fn, tag.c_str(), in[i] ? "negative count" : "null input"); return false; }
        const CodecStream & t = s[i]->st;
        if (t.direction == kStreamEncode && t.resampled) {
            const float * x = (const float *) in[i];
            const long long C = t.rs.channels, floats = n[i] * C;
            if (floats > INT_MAX) { fprintf(stderr, "%s: %s%d frames of %lld channels (at most 2^31 - 1 samples per push)\n", fn, tag.c_str(), n[i], C); return false; }
            for (long long k = 0; k < floats; k++) if (!(std::fabs(x[k]) <= 0x1p64f)) {
                fprintf(stderr, "%s: %ssample %lld (frame %lld, channel %lld) is not finite or exceeds 2^64 in magnitude (%g)\n", fn, tag.c_str(), k, k / C, k % C, (double) x[k]);
                return false;
            }
        } else if (t.direction == kStreamEncode) {
            const float * x = (const float *) in[i];
            for (int k = 0; k < n[i]; k++) if (!std::isfinite(x[k])) { fprintf(stderr, "%s: %ssample %d is not finite (%g)\n", fn, tag.c_str(), k, (double) x[k]); return false; }
        } else {
            const int32_t * c = (const int32_t *) in[i];
            const int bins = s[i]->e->model.n_bins;
            for (size_t k = 0; k < (size_t) t.n_q * n[i]; k++) if (c[k] < 0 || c[k] >= bins) {
                fprintf(stderr, "%s: %scode %d (codebook %zu, frame %zu) is outside the codebooks (%d bins)\n", fn, tag.c_str(), c[k], k / n[i], k % n[i], bins);
                return false;
            }
        }
    }
    return true;
}

// the stream calls: the context's device current, a CUDA failure or exception is `fail`; the context's statistics are left alone
template <typename R, typename F> R stream_call(bark_b200_encodec_stream * s, R fail, F && f) {
    return guarded(fail, [&]() -> R { BARK_CUDA_CHECK(cudaSetDevice(s->e->device)); return f(); });
}

int push(const char * fn, bark_b200_encodec_stream * const * s, const void * const * in, const int * n, int count) {
    if (!in || !n) { fprintf(stderr, "%s: null %s\n", fn, in ? "count array" : "input array"); return -1; }
    if (!stream_args(fn, s, in, n, count)) return -1;
    std::vector<CodecStream *> st((size_t) count);
    for (int i = 0; i < count; i++) st[(size_t) i] = &s[i]->st;
    return stream_call(s[0], -1, [&] { return codec_stream_run(s[0]->e->model, s[0]->e->scratch, s[0]->e->stream, st.data(), in, n, count, false, fn); });
}

// a stream of e in direction at a format (mono 24 kHz: the plain stream), named fn
bark_b200_encodec_stream * open_stream(const char * fn, encodec_context * e, int direction, int channels, int sample_rate) {
    if (!e) { fprintf(stderr, "%s: null context\n", fn); return nullptr; }
    if (direction != BARK_B200_STREAM_ENCODE && direction != BARK_B200_STREAM_DECODE) { fprintf(stderr, "%s: unknown direction %d\n", fn, direction); return nullptr; }
    if (channels < 1 || channels > kResampleMaxChannels) { fprintf(stderr, "%s: %d channels (1 to %d)\n", fn, channels, kResampleMaxChannels); return nullptr; }
    if (sample_rate < kResampleMinRate || sample_rate > kResampleMaxRate) {
        fprintf(stderr, "%s: sample rate %d Hz (%d to %d)\n", fn, sample_rate, kResampleMinRate, kResampleMaxRate); return nullptr;
    }
    if (direction == BARK_B200_STREAM_DECODE && channels != 1) { fprintf(stderr, "%s: a decode stream gives mono samples (channels 1, got %d)\n", fn, channels); return nullptr; }
    if (direction == BARK_B200_STREAM_ENCODE && !e->model.enc.present) { fprintf(stderr, "%s: the model file has no EnCodec encoder tensors (encoder.*)\n", fn); return nullptr; }
    int n_q;
    if (!codebooks_for(e, fn, &n_q)) return nullptr;
    auto * s = new bark_b200_encodec_stream{e, CodecStream()};
    if (!guarded(false, [&] { BARK_CUDA_CHECK(cudaSetDevice(e->device)); return codec_stream_init(e->model, s->st, direction, n_q, channels, sample_rate); })) {
        fprintf(stderr, "%s: could not allocate the stream's state\n", fn);
        bark_b200_encodec_stream_close(s);
        return nullptr;
    }
    return s;
}

}  // namespace

extern "C" struct bark_b200_encodec_stream * bark_b200_encodec_stream_open(struct encodec_context * e, int direction) {
    return open_stream(__func__, e, direction, 1, kCodecSampleRate);
}

extern "C" struct bark_b200_encodec_stream * bark_b200_encodec_stream_open_resampled(struct encodec_context * e, int direction, int channels, int sample_rate) {
    return open_stream(__func__, e, direction, channels, sample_rate);
}

extern "C" int bark_b200_encodec_stream_push(struct bark_b200_encodec_stream * s, const void * in, int n) {
    return push(__func__, &s, &in, &n, 1);
}

extern "C" int bark_b200_encodec_stream_push_batch(struct bark_b200_encodec_stream * const * s, const void * const * in, const int * n, int count) {
    return push(__func__, s, in, n, count);
}

extern "C" int bark_b200_encodec_stream_read(struct bark_b200_encodec_stream * s, void * out, int cap) {
    if (!s) { fprintf(stderr, "%s: null stream\n", __func__); return -1; }
    CodecStream & t = s->st;
    const size_t per = t.direction == kStreamEncode ? (size_t) t.n_q : 1, ready = (t.direction == kStreamEncode ? t.codes.size() : t.audio.size()) / per;
    const size_t k = std::min(ready, (size_t) std::max(cap, 0));
    if (!out) return (int) std::min(ready, (size_t) INT_MAX);
    if (t.direction == kStreamDecode) {
        std::copy_n(t.audio.begin(), k, (float *) out);
        t.audio.erase(t.audio.begin(), t.audio.begin() + (ptrdiff_t) k);
    } else {                                             // frame-major pending -> [n_q][k]
        int32_t * o = (int32_t *) out;
        for (size_t f = 0; f < k; f++)
            for (size_t q = 0; q < per; q++) o[q * k + f] = t.codes[f * per + q];
        t.codes.erase(t.codes.begin(), t.codes.begin() + (ptrdiff_t)(k * per));
    }
    return (int) k;
}

extern "C" int bark_b200_encodec_stream_finish(struct bark_b200_encodec_stream * s) {
    const char * fn = __func__;
    if (!stream_args(fn, &s, nullptr, nullptr, 1)) return -1;
    const CodecStream & t = s->st;
    if (t.resampled && t.direction == kStreamEncode) {              // the encoder finishes on the resampled clip's L samples
        const long long L = resample_len(t.rs.in, t.rs.rate, kCodecSampleRate);
        if (L < kCodecMinSamples) {
            fprintf(stderr, "%s: %lld frames at %d Hz resample to %lld samples at %d Hz (at least %d: %d frames)\n", fn, t.rs.in, t.rs.rate, L, kCodecSampleRate,
                    kCodecMinSamples, kCodecMinFrames);
            return -1;
        }
    } else if (t.direction == kStreamEncode ? t.n_in < kCodecMinSamples : t.n_in < kCodecMinFrames) {
        fprintf(stderr, "%s: need at least %d %s (reflect padding of the k=7 convolutions), got %lld\n", fn, t.direction == kStreamEncode ? kCodecMinSamples : kCodecMinFrames,
                t.direction == kStreamEncode ? "samples" : "frames", t.n_in);
        return -1;
    }
    CodecStream * st = &s->st;
    const int zero = 0;
    const void * none = nullptr;
    return stream_call(s, -1, [&] { return codec_stream_run(s->e->model, s->e->scratch, s->e->stream, &st, &none, &zero, 1, true, fn); });
}

extern "C" long long bark_b200_encodec_stream_ready(int direction, long long n) {
    if ((direction != BARK_B200_STREAM_ENCODE && direction != BARK_B200_STREAM_DECODE) || n < 0) return -1;
    return codec_stream_ready(direction, n);
}

extern "C" long long bark_b200_encodec_stream_ready_resampled(int direction, int sample_rate, long long n) {
    if ((direction != BARK_B200_STREAM_ENCODE && direction != BARK_B200_STREAM_DECODE) || n < 0) return -1;
    if (sample_rate < kResampleMinRate || sample_rate > kResampleMaxRate) return -1;
    return codec_stream_ready_resampled(direction, sample_rate, n);
}

extern "C" int bark_b200_encodec_stream_codebooks(struct bark_b200_encodec_stream * s) {
    if (!s) { fprintf(stderr, "%s: null stream\n", __func__); return -1; }
    return s->st.n_q;
}

extern "C" void bark_b200_encodec_stream_close(struct bark_b200_encodec_stream * s) {
    if (!s) return;
    cudaSetDevice(s->e->device);
    if (s->e->stream) cudaStreamSynchronize(s->e->stream);
    s->st.release();
    delete s;
}
