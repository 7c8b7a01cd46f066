// The EnCodec pipelines on the host: the device-side replacement of encodec_eval (encodec.cpp/encodec.cpp:819-847) for the decoder and
// of encodec_compress_audio's encoder (encodec.cpp:878-900), for n clips at once.  Every item is checked first; the items then run in
// launches of consecutive items, each one pass of the codec kernels over its items into a scratch grown on demand.
#include "codec_kernels.h"
#include "codec_layers.h"
#include "context.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <string>
#include <vector>

namespace bark {

// codec scratch for one launch of `frames` frames over its items: three activation buffers of 10240 floats per frame (the decoder's largest
// activation is [64][160T] = [32][320T]; the encoder's, [32][n_samples], is no larger), the LSTM input projections and the [n_q][T] codes
bool codec_scratch(CodecScratch & sc, size_t frames, int n_q, const char * caller) {
    const size_t need = (size_t) 10240 * frames + 1024, codes_need = (size_t) n_q * frames;
    if (need > sc.cap || codes_need > sc.codes_cap) {
        // out of memory here is recoverable (a very long clip): report it and return false like the reference's failed encodec_eval
        auto grow = [&](void ** p, size_t bytes) { if (*p) { cudaFree(*p); *p = nullptr; } return cudaMalloc(p, bytes) == cudaSuccess; };
        const size_t cap = std::max(need, sc.cap), ccap = std::max(codes_need, sc.codes_cap);
        sc.cap = sc.codes_cap = 0;
        bool ok = true;
        for (int i = 0; i < 3; i++) ok = ok && grow((void **) &sc.buf[i], cap * sizeof(float));
        ok = ok && grow((void **) &sc.gi, (cap - 1024) / 10240 * 2048 * sizeof(float)) && grow((void **) &sc.codes, ccap * sizeof(int32_t));
        if (ok && !sc.hbuf) ok = cudaMalloc((void **) &sc.hbuf, (size_t) 2 * kCodecMaxItems * 512 * sizeof(float)) == cudaSuccess &&
                                 cudaMalloc((void **) &sc.counter, sizeof(unsigned)) == cudaSuccess;
        if (!ok) { (void) cudaGetLastError(); fprintf(stderr, "%s: out of device memory for %zu frames\n", caller, frames); return false; }
        sc.cap = cap; sc.codes_cap = ccap;
    }
    return true;
}

bool stage_scratch(CodecScratch & sc, size_t floats, const char * caller) {
    if (floats <= sc.stage_cap) return true;
    if (sc.stage) { cudaFree(sc.stage); sc.stage = nullptr; }
    sc.stage_cap = 0;
    if (cudaMalloc((void **) &sc.stage, floats * sizeof(float)) != cudaSuccess) {
        (void) cudaGetLastError(); fprintf(stderr, "%s: out of device memory for %zu source samples\n", caller, floats); return false;
    }
    sc.stage_cap = floats;
    return true;
}

void CodecScratch::release() {
    for (int i = 0; i < 3; i++) if (buf[i]) cudaFree(buf[i]);
    for (void * p : {(void *) gi, (void *) hbuf, (void *) counter, (void *) codes, (void *) stage}) if (p) cudaFree(p);
    for (auto & t : tables) if (t.second) cudaFree(t.second);
    *this = CodecScratch();
}

// Rate pairs whose taps a scratch keeps; a launch needs at most kCodecMaxItems of them, and the cache is emptied between launches
// when a new one would pass this
constexpr size_t kResampleTablesKept = 64;

// the taps of sr -> kCodecSampleRate, built and uploaded on first use
static ResampleTable scratch_table(CodecScratch & sc, int sr) {
    for (const auto & t : sc.tables) if (t.first.sr == sr) return t.first;
    ResampleTable t;
    const std::vector<unsigned char> bytes = resample_table(sr, kCodecSampleRate, &t);
    void * d = nullptr;
    if (!bytes.empty()) {
        BARK_CUDA_CHECK(cudaMalloc(&d, bytes.size()));
        sc.tables.emplace_back(t, d);                    // owned from here, so a failed copy does not leak it
        BARK_CUDA_CHECK(cudaMemcpy(d, bytes.data(), bytes.size(), cudaMemcpyHostToDevice)); g_h2d_bytes += bytes.size();
        resample_bind(sc.tables.back().first, d);
        return sc.tables.back().first;
    }
    sc.tables.emplace_back(t, nullptr);
    return t;
}

bool resample_input_ok(const char * fn, const std::string & item, const float * x, int n_frames, int channels, int sample_rate) {
    if (channels < 1 || channels > kResampleMaxChannels) { fprintf(stderr, "%s: %s%d channels (1 to %d)\n", fn, item.c_str(), channels, kResampleMaxChannels); return false; }
    if (sample_rate < kResampleMinRate || sample_rate > kResampleMaxRate) {
        fprintf(stderr, "%s: %ssample rate %d Hz (%d to %d)\n", fn, item.c_str(), sample_rate, kResampleMinRate, kResampleMaxRate); return false;
    }
    if (n_frames < 1 || (long long) n_frames * channels > INT_MAX) {
        fprintf(stderr, "%s: %s%d frames of %d channels (1 frame to 2^31 - 1 samples)\n", fn, item.c_str(), n_frames, channels); return false;
    }
    // |x| <= 2^64: neither the channel sum nor the filter's double sum can overflow
    for (long long k = 0; k < (long long) n_frames * channels; k++) if (!(std::fabs(x[k]) <= 0x1p64f)) {
        fprintf(stderr, "%s: %ssample %lld (frame %lld, channel %lld) is not finite or exceeds 2^64 in magnitude (%g)\n", fn, item.c_str(), k, k / channels,
                k % channels, (double) x[k]);
        return false;
    }
    return true;
}

// [first, last) item ranges of the launches: consecutive items, at most kCodecMaxItems and kCodecLaunchFrames frames, at least one item
static std::vector<std::pair<int, int>> codec_launches(const int * T, int n) {
    std::vector<std::pair<int, int>> groups;
    for (int i = 0; i < n;) {
        int j = i + 1;
        long long frames = T[i];
        while (j < n && j - i < kCodecMaxItems && frames + T[j] <= kCodecLaunchFrames) frames += T[j++];
        groups.emplace_back(i, j);
        i = j;
    }
    return groups;
}

std::string item_tag(const char * batch_fn, int i) { return batch_fn ? "item " + std::to_string(i) + ": " : std::string(); }

// The whole-clip runner of the layer lists (codec_layers.h): n items of L[b] columns of C channels in cur, the other two activation
// buffers free; every layer runs once over all the items' columns and leaves its output in cur.
struct ClipRunner {
    CodecScratch & sc; cudaStream_t s; int n, C; std::vector<int> L; float * cur, * a, * b;
    void conv(const ConvW & cv, bool elu_in, int stride) {
        conv1d(cur, C, L.data(), n, cv, elu_in, nullptr, a, s, stride);
        if (stride > 1) for (int & x : L) x = conv1d_out_len(x, cv.k, stride);
        C = cv.cout; std::swap(cur, a);
    }
    template <class B> void resblock(const B & blk) {
        conv1d(cur, C, L.data(), n, blk.sc, false, nullptr, a, s);      // shortcut on the block input
        conv1d(cur, C, L.data(), n, blk.c1, true, nullptr, b, s);       // ELU -> k3 -> [C/2][L]
        conv1d(b, C / 2, L.data(), n, blk.c2, true, a, cur, s);         // ELU -> k1, + shortcut
    }
    void convtr(const ConvW & cv, int stride) {
        convtr1d(cur, C, L.data(), n, cv, stride, a, s);
        for (int & x : L) x *= stride;
        C = cv.cout; std::swap(cur, a);
    }
    void lstm2(const CodecLSTM & w) {
        lstm_layer(cur, C, L.data(), n, w.ih_w[0], w.hh_w[0], w.Kp, w.ih_b[0], w.hh_b[0], nullptr, sc.gi, sc.hbuf, sc.counter, a, s);
        lstm_layer(a, C, L.data(), n, w.ih_w[1], w.hh_w[1], w.Kp, w.ih_b[1], w.hh_b[1], cur, sc.gi, sc.hbuf, sc.counter, b, s);
        std::swap(cur, b);
    }
};

// The decoder on the codes in sc.codes ([n_q][T_b] per item, item-major) of n items of T[b] frames; returns the waveforms, [kCodecHop T_b] per item.
static const float * decode_launch(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, const int * T, int n, int n_q) {
    ClipRunner r{sc, s, n, cm.hidden_dim, std::vector<int>(T, T + n), sc.buf[0], sc.buf[1], sc.buf[2]};
    rvq_decode(cm, sc.codes, n_q, T, n, r.cur, s);                                           // [128][T]
    decoder_layers(cm, r);
    return r.cur;
}

// The encoder and the RVQ on the samples in sc.buf[2] ([n_b] per item, concatenated) of n items; codes to sc.codes ([n_q][T_b] per
// item); returns the latents ([128][T_b] per item), null (message) on an unsupported shape.
static const float * encode_launch(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, const int * n_samples, int n, int n_q, const char * caller) {
    ClipRunner r{sc, s, n, 1, std::vector<int>(n_samples, n_samples + n), sc.buf[2], sc.buf[0], sc.buf[1]};
    encoder_layers(cm.enc, r);
    for (int b = 0; b < n; b++)
        if (r.L[(size_t) b] != (n_samples[b] - 1) / kCodecHop + 1) { fprintf(stderr, "%s: internal error: %d latent frames for %d samples\n", caller, r.L[(size_t) b], n_samples[b]); return nullptr; }
    if (!rvq_encode(cm.embed, cm.embed_norm, n_q, cm.n_bins, cm.hidden_dim, r.cur, r.L.data(), n, sc.codes, s)) { fprintf(stderr, "%s: unsupported codebook shape (%d bins of %d)\n", caller, cm.n_bins, cm.hidden_dim); return nullptr; }
    return r.cur;
}

// v = the count values at src, copied back on s
template <class V> static void fetch(std::vector<V> & v, const V * src, size_t count, cudaStream_t s) {
    v.resize(count);
    BARK_CUDA_CHECK(cudaMemcpyAsync(v.data(), src, count * sizeof(V), cudaMemcpyDeviceToHost, s)); g_d2h_bytes += count * sizeof(V);
}

// The launches of n checked items of T[i] frames.  Per launch: the scratch sized, upload(first, last, &latent) enqueues the items'
// inputs (for an encode, and the encoder, whose latents it points latent at; false with a message on failure), then the outputs of
// `out` come back item by item (codes and latent, then the decoder's waveform of the codes in the scratch), and one synchronisation.
template <class Upload>
static bool run_launches(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, int n, const int * T, int n_q, const CodecOutputs & out,
                         const char * fn, const Upload & upload) {
    const size_t Hd = (size_t) cm.hidden_dim;
    for (const auto & g : codec_launches(T, n)) {
        size_t frames = 0;
        for (int i = g.first; i < g.second; i++) frames += (size_t) T[i];
        if (!codec_scratch(sc, frames, n_q, fn)) return false;
        const float * lat = nullptr;
        if (!upload(g.first, g.second, &lat)) return false;
        size_t f = 0;
        for (int i = g.first; i < g.second; f += (size_t) T[i], i++) {
            if (out.codes) fetch(out.codes[i], sc.codes + (size_t) n_q * f, (size_t) n_q * T[i], s);
            if (out.latent) fetch(out.latent[i], lat + Hd * f, Hd * T[i], s);
        }
        if (out.audio) {                                                 // decodes the codes in the scratch (encodec.cpp:592-602)
            const float * wav = decode_launch(cm, sc, s, T + g.first, g.second - g.first, n_q);
            f = 0;
            for (int i = g.first; i < g.second; f += (size_t) T[i], i++) fetch(out.audio[i], wav + (size_t) kCodecHop * f, (size_t) kCodecHop * T[i], s);
        }
        BARK_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return true;
}

bool codec_decode(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, int n, const int32_t * const * codes, const int * T, int n_q, std::vector<float> * audio,
                  const char * batch_fn) {
    const char * fn = batch_fn ? batch_fn : "codec_decode";
    for (int i = 0; i < n; i++)
        if (T[i] < kCodecMinFrames) {
            fprintf(stderr, "%s: %sneed at least %d frames (reflect padding of the k=7 convolutions), got %d\n", fn, item_tag(batch_fn, i).c_str(), kCodecMinFrames, T[i]);
            return false;
        }
    if (n_q < 1 || n_q > cm.n_q) { fprintf(stderr, "%s: %d codebooks requested, %d loaded\n", fn, n_q, cm.n_q); return false; }
    for (int i = 0; i < n; i++)
        for (size_t k = 0; k < (size_t) n_q * T[i]; k++) if (codes[i][k] < 0 || codes[i][k] >= cm.n_bins) {
            fprintf(stderr, "%s: %scode %d (codebook %zu, frame %zu) is outside the codebooks (%d bins)\n", fn, item_tag(batch_fn, i).c_str(), codes[i][k], k / T[i], k % T[i], cm.n_bins);
            return false;
        }
    CodecOutputs out;
    out.audio = audio;
    return run_launches(cm, sc, s, n, T, n_q, out, fn, [&](int first, int last, const float **) {
        size_t f = 0;
        for (int i = first; i < last; f += (size_t) T[i], i++) {
            const size_t nb = (size_t) n_q * T[i] * sizeof(int32_t);
            BARK_CUDA_CHECK(cudaMemcpyAsync(sc.codes + (size_t) n_q * f, codes[i], nb, cudaMemcpyHostToDevice, s)); g_h2d_bytes += nb;
        }
        return true;
    });
}

bool codec_encode(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, int n, const float * const * audio, const int * n_samples, int n_q,
                  const CodecOutputs & out, const char * batch_fn, const AudioFormat * fmt) {
    const char * fn = batch_fn ? batch_fn : "codec_encode";
    if (!cm.enc.present) { fprintf(stderr, "%s: the model file has no EnCodec encoder tensors (encoder.*)\n", fn); return false; }
    if (n_q < 1 || n_q > cm.n_q) { fprintf(stderr, "%s: %d codebooks requested, %d loaded\n", fn, n_q, cm.n_q); return false; }
    // the encoder's input samples per item, and whether the item goes through the resampler (mono 24 kHz does not)
    std::vector<int> len(n_samples, n_samples + n);
    std::vector<char> resampled((size_t) n, 0);
    size_t stage = 0;                                    // floats of the largest resampled item's source
    for (int i = 0; i < n; i++) {
        if (fmt) {
            const std::string item = item_tag(batch_fn, i);
            if (!resample_input_ok(fn, item, audio[i], n_samples[i], fmt[i].channels, fmt[i].sample_rate)) return false;
            const long long L = resample_len(n_samples[i], fmt[i].sample_rate, kCodecSampleRate);
            if (L < kCodecMinSamples || L > INT_MAX) {
                fprintf(stderr, "%s: %s%d frames at %d Hz resample to %lld samples at %d Hz (%d to 2^31 - 1: at least %d frames)\n", fn, item.c_str(),
                        n_samples[i], fmt[i].sample_rate, L, kCodecSampleRate, kCodecMinSamples, kCodecMinFrames);
                return false;
            }
            len[(size_t) i] = (int) L;
            resampled[(size_t) i] = fmt[i].channels != 1 || fmt[i].sample_rate != kCodecSampleRate;
            if (resampled[(size_t) i]) stage = std::max(stage, (size_t) n_samples[i] * fmt[i].channels);
            continue;
        }
        if (n_samples[i] < kCodecMinSamples) {
            fprintf(stderr, "%s: %sneed at least %d samples (%d frames), got %d\n", fn, item_tag(batch_fn, i).c_str(), kCodecMinSamples, kCodecMinFrames, n_samples[i]);
            return false;
        }
        for (int k = 0; k < n_samples[i]; k++) if (!std::isfinite(audio[i][k])) {
            fprintf(stderr, "%s: %ssample %d is not finite (%g)\n", fn, item_tag(batch_fn, i).c_str(), k, (double) audio[i][k]); return false;
        }
    }
    if (!stage_scratch(sc, stage, fn)) return false;
    std::vector<int> T((size_t) n);
    for (int i = 0; i < n; i++) T[(size_t) i] = (len[(size_t) i] - 1) / kCodecHop + 1;
    return run_launches(cm, sc, s, n, T.data(), n_q, out, fn, [&](int first, int last, const float ** lat) {
        if (fmt && sc.tables.size() + (size_t)(last - first) > kResampleTablesKept) {
            for (auto & t : sc.tables) if (t.second) cudaFree(t.second);          // no launch in flight: the last one synchronised
            sc.tables.clear();
        }
        size_t off = 0;
        for (int i = first; i < last; off += (size_t) len[(size_t) i], i++) {
            if (resampled[(size_t) i]) {                 // the source through the staging buffer, reused item by item on the stream
                const size_t nb = (size_t) n_samples[i] * fmt[i].channels * sizeof(float);
                BARK_CUDA_CHECK(cudaMemcpyAsync(sc.stage, audio[i], nb, cudaMemcpyHostToDevice, s)); g_h2d_bytes += nb;
                resample(sc.stage, n_samples[i], fmt[i].channels, scratch_table(sc, fmt[i].sample_rate), sc.buf[2] + off, len[(size_t) i], s);
                continue;
            }
            const size_t nb = (size_t) n_samples[i] * sizeof(float);
            BARK_CUDA_CHECK(cudaMemcpyAsync(sc.buf[2] + off, audio[i], nb, cudaMemcpyHostToDevice, s)); g_h2d_bytes += nb;
        }
        *lat = encode_launch(cm, sc, s, len.data() + first, last - first, n_q, fn);
        return *lat != nullptr;
    });
}

}  // namespace bark
