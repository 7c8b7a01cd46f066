// Streaming EnCodec (DESIGN.md §19): the layer lists of codec_layers.h run over each layer's window of [history | new columns], so a
// stream pushed chunk by chunk computes every position once, with the same kernels and the same bits as the whole clip.  The 24 kHz
// model is causal: its convolutions reflect-pad on the left only (and on the right once, at the end of an encode, where the strided
// ones pad to whole frames), the transposed convolutions trim on the right and the LSTMs run forwards.  So a layer's output is final as
// soon as the inputs it reads have arrived, and the layer keeps the last few of them, the LSTMs their (h, c).
#include "codec_kernels.h"
#include "codec_layers.h"
#include "context.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <string>
#include <vector>

namespace bark {

long long codec_stream_ready(int direction, long long n) {
    // encode: latent frame j reads samples up to kCodecHop (j + 1) - 1 through the four strided convs, and the final k = 7 conv reflects
    // frame 0 onto frames 1..6, so nothing is final before 7 frames.  decode: the first k = 7 conv waits for 7 frames; after it nothing
    // looks ahead except at the start of the signal (DESIGN.md §19).
    if (direction == kStreamEncode) return n >= (long long) kCodecMinFrames * kCodecHop ? n / kCodecHop : 0;
    return n >= kCodecMinFrames ? n * kCodecHop : 0;
}

long long codec_stream_ready_resampled(int direction, int sample_rate, long long n) {
    // encode: the resampler's final outputs feed the encoder; decode: the decoder's final samples feed the resampler (DESIGN.md §20)
    if (direction == kStreamEncode) return codec_stream_ready(kStreamEncode, resample_ready(n, sample_rate, kCodecSampleRate));
    const long long samples = n < kCodecMinFrames ? 0 : n > LLONG_MAX / kCodecHop ? LLONG_MAX : n * kCodecHop;
    return resample_ready(samples, kCodecSampleRate, sample_rate);
}

namespace {

// the outputs of a stream's resampler final once `in` frames have arrived; at finish every output, the signal ending there
long long resampler_target(const StreamResampler & rs, long long in, bool finish) {
    return finish ? resample_len(in, rs.t.sr, rs.t.new_sr) : resample_ready(in, rs.t.sr, rs.t.new_sr);
}

// The resampler step of a pass over the resampled streams among st (DESIGN.md §20).  Stream i's n[i] new frames come from the host at
// host[i] (an encode's interleaved source) or from the device at dev[i] (a decode's 24 kHz samples); one copy launch gathers them after
// its history into `gather`, one launch of resample_kernel computes the out[i] outputs that became final into y[i], and a second copy
// launch keeps the frames from the next block's first read on.  Every output released before finish has an index below the clip's
// L = ceil(q n / o): block k is released once n >= (k + 1) o + w, and then its last output k q + q - 1 < q n / o.  It reads no frame
// past n, so the frames that arrive later, and the zeros past the end at finish, cannot change it.
void resample_step(cudaStream_t s, CodecStream * const * st, int count, const int * n, const void * const * host, const float * const * dev,
                   float * gather, float * const * y, const int * out, bool finish) {
    ColumnCopies g, back;
    auto job = [](ColumnCopies & c, const float * src, float * dst, long long floats) {
        if (floats <= 0) return;
        c.src[c.n] = src; c.dst[c.n] = dst; c.src_ld[c.n] = c.dst_ld[c.n] = c.cols[c.n] = (int) floats; c.n++;
    };
    ResampleWindow w[kCodecMaxItems];
    int m = 0;
    size_t off = 0;
    for (int i = 0; i < count; i++) {
        if (!st[i]->resampled) continue;
        StreamResampler & rs = st[i]->rs;
        const int C = rs.channels, len = rs.h + n[i];
        const long long in = rs.in + n[i], org = rs.in - rs.h, target = resampler_target(rs, in, finish);
        if (target - rs.out != out[i]) throw std::runtime_error("stream resampler: outputs differ from the plan");
        float * x = gather + off;
        job(g, rs.hist, x, (long long) rs.h * C);
        if (n[i] && host) {
            BARK_CUDA_CHECK(cudaMemcpyAsync(x + (size_t) rs.h * C, host[i], (size_t) n[i] * C * sizeof(float), cudaMemcpyHostToDevice, s));
            g_h2d_bytes += (size_t) n[i] * C * sizeof(float);
        } else if (n[i]) job(g, dev[i], x + rs.h, n[i]);
        if (out[i]) {
            ResampleWindow & v = w[m++];
            v.t = rs.t; v.x = x; v.y = y[i]; v.org = org; v.len = len; v.C = C; v.first = rs.out; v.n_out = out[i]; v.end = finish ? in : LLONG_MAX;
        }
        const long long keep = finish ? in : std::max(org, target / rs.t.q * rs.t.o - rs.t.w);
        const int h = (int)(in - keep);
        if (h > rs.cap) throw std::runtime_error("stream resampler history overflow");
        job(back, x + (size_t)(keep - org) * C, rs.hist, (long long) h * C);
        rs.in = in; rs.out = target; rs.h = h;
        off += (size_t) len * C;
    }
    copy_columns(g, 1, s);
    if (m) resample_windows(w, m, s);
    copy_columns(back, 1, s);
}

// A layer over windows.  Output t reads input positions t stride - pad .. t stride - pad + k - 1, pad = k - stride.  A convolution
// reflects those below 0, so its output 0 waits for its largest reflected read; the transposed convolution (k = 2, stride 1: frames
// t - 1 and t) reads nothing below 0.
struct LayerShape { int k, stride; bool reflect; };

// the outputs of `shape` final after `in` inputs; at the end of an encode the strided convolutions pad to whole frames as the whole clip
// does (get_extra_padding_for_conv_1d, evaluated in float)
long long layer_ready(const LayerShape & l, long long in, long long out, bool finish) {
    if (!l.reflect) return in;
    if (l.stride == 1) return in >= l.k ? in : 0;
    if (finish) return std::max(out, in <= INT_MAX ? (long long) conv1d_out_len((int) in, l.k, l.stride) : (in + l.stride - 1) / l.stride);
    return in >= l.stride + 1 ? in / l.stride : 0;       // output 0 reads the reflected position `stride`
}

// The windows and LSTM states of a stream, in list order: a convolution keeps up to k - 1 input columns (k - 1 before its first output;
// after it, the k - stride its next output reads before its first new position plus at most stride - 1 unconsumed), a transposed
// convolution one frame.
struct LayoutRunner {
    int C; std::vector<std::pair<int, int>> win; int lstm_C = 0;
    void conv(const ConvW & cv, bool, int) { win.emplace_back(C, cv.k - 1); C = cv.cout; }
    template <class B> void resblock(const B & blk) { win.emplace_back(C, blk.c1.k - 1); }
    void convtr(const ConvW & cv, int) { win.emplace_back(C, 1); C = cv.cout; }
    void lstm2(const CodecLSTM &) { lstm_C = C; }
};

// One pass of the layer lists over n streams.  cur holds every item's N[b] new columns of C channels, item-major; a layer gathers each
// item's window into `a`, runs over the items with outputs to compute (in that order, so their outputs stay item-major in `b`), saves the
// columns the next push needs and leaves its outputs in cur.  An item without new outputs appends its new columns to its history.
struct StreamRunner {
    CodecScratch & sc; cudaStream_t s; int n; CodecStream * const * st; bool finish;
    int C; std::vector<int> N; float * cur, * a, * b;
    int wi = 0, li = 0;                                  // the next window and LSTM layer

    struct Launch { int n = 0; int L[kCodecMaxItems]; CodecWindow w; int item[kCodecMaxItems]; long long ready[kCodecMaxItems]; size_t off[kCodecMaxItems]; };

    Launch open(const LayerShape & shape) {
        Launch l;
        ColumnCopies g;
        auto job = [&](const float * src, int src_ld, float * dst, int dst_ld, int cols) {
            if (cols <= 0) return;
            g.src[g.n] = src; g.src_ld[g.n] = src_ld; g.dst[g.n] = dst; g.dst_ld[g.n] = dst_ld; g.cols[g.n] = cols; g.n++;
        };
        size_t src = 0, dst = 0;
        for (int i = 0; i < n; src += (size_t) C * N[(size_t) i], i++) {
            CodecStream::Window & w = st[i]->win[(size_t) wi];
            const long long in = w.in + N[(size_t) i], R = layer_ready(shape, in, w.out, finish);
            if (R == w.out) {                            // nothing new is final: the new columns join the history
                if (w.h + N[(size_t) i] > w.cap) throw std::runtime_error("stream history overflow");
                job(cur + src, N[(size_t) i], w.hist + w.h, w.cap, N[(size_t) i]);
                w.h += N[(size_t) i]; w.in = in;
                continue;
            }
            const int W = w.h + N[(size_t) i], j = l.n++;
            job(w.hist, w.cap, a + dst, W, w.h);
            job(cur + src, N[(size_t) i], a + dst + w.h, W, N[(size_t) i]);
            l.L[j] = W; l.item[j] = i; l.ready[j] = R; l.off[j] = dst;
            l.w.org[j] = w.in - w.h; l.w.first[j] = w.out; l.w.n_out[j] = (int)(R - w.out);
            dst += (size_t) C * W;
        }
        copy_columns(g, C, s);
        return l;
    }

    // after the launches on window `a`: each launched item keeps the columns from its next output's first read on
    void close(const Launch & l, const LayerShape & shape) {
        ColumnCopies g;
        for (int j = 0; j < l.n; j++) {
            CodecStream::Window & w = st[l.item[j]]->win[(size_t) wi];
            const long long in = l.w.org[j] + l.L[j], keep = std::max(l.w.org[j], l.ready[j] * shape.stride - (shape.k - shape.stride));
            const int h = (int)(in - keep);
            g.src[g.n] = a + l.off[j] + (l.L[j] - h); g.src_ld[g.n] = l.L[j]; g.dst[g.n] = w.hist; g.dst_ld[g.n] = w.cap; g.cols[g.n] = h;
            g.n += h > 0;
            w.in = in; w.out = l.ready[j]; w.h = h;
        }
        copy_columns(g, C, s);
        wi++;
    }

    // the new columns of the next layer: the launched items' outputs, times `per` (a transposed conv's samples per frame)
    void outputs(const Launch & l, int per) {
        std::fill(N.begin(), N.end(), 0);
        for (int j = 0; j < l.n; j++) N[(size_t) l.item[j]] = l.w.n_out[j] * per;
    }

    void conv(const ConvW & cv, bool elu_in, int stride) {
        const LayerShape shape{cv.k, stride, true};
        const Launch l = open(shape);
        if (l.n) conv1d(a, C, l.L, l.n, cv, elu_in, nullptr, b, s, stride, &l.w);
        close(l, shape);
        outputs(l, 1);
        C = cv.cout; std::swap(cur, b);
    }
    template <class B> void resblock(const B & blk) {
        const LayerShape shape{blk.c1.k, 1, true};
        const Launch l = open(shape);                    // the shortcut reads the k3 conv's window, so both give the same outputs
        if (l.n) {
            conv1d(a, C, l.L, l.n, blk.sc, false, nullptr, b, s, 1, &l.w);
            conv1d(a, C, l.L, l.n, blk.c1, true, nullptr, cur, s, 1, &l.w);
        }
        close(l, shape);
        if (l.n) conv1d(cur, C / 2, l.w.n_out, l.n, blk.c2, true, b, a, s);
        outputs(l, 1);
        std::swap(cur, a);
    }
    void convtr(const ConvW & cv, int stride) {
        const LayerShape shape{2, 1, false};
        const Launch l = open(shape);
        if (l.n) convtr1d(a, C, l.L, l.n, cv, stride, b, s, &l.w);
        close(l, shape);
        outputs(l, stride);
        C = cv.cout; std::swap(cur, b);
    }
    void lstm2(const CodecLSTM & w) {
        int T[kCodecMaxItems], m = 0;
        float * h0[kCodecMaxItems], * h1[kCodecMaxItems];
        for (int i = 0; i < n; i++)
            if (N[(size_t) i]) { T[m] = N[(size_t) i]; h0[m] = st[i]->lstm[li]; h1[m] = st[i]->lstm[li + 1]; m++; }
        li += 2;
        if (!m) return;
        lstm_layer(cur, C, T, m, w.ih_w[0], w.hh_w[0], w.Kp, w.ih_b[0], w.hh_b[0], nullptr, sc.gi, sc.hbuf, sc.counter, a, s, h0);
        lstm_layer(a, C, T, m, w.ih_w[1], w.hh_w[1], w.Kp, w.ih_b[1], w.hh_b[1], cur, sc.gi, sc.hbuf, sc.counter, b, s, h1);
        std::swap(cur, b);
    }
};

// the items of `N` with columns: their count, lengths and stream indices
int present(const std::vector<int> & N, int * T, int * item) {
    int m = 0;
    for (size_t i = 0; i < N.size(); i++) if (N[i]) { T[m] = N[i]; item[m] = (int) i; m++; }
    return m;
}

// One pass: n[i] new inputs of stream i at in[i] (with finish, none); the outputs that became final go to the streams' pending outputs.
bool stream_pass(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, CodecStream * const * st, const void * const * in, const int * n, int count,
                 bool finish, const char * fn) {
    const int dir = st[0]->direction, n_q = st[0]->n_q;
    // per stream: the codec's new inputs N (a resampled encode's are its resampler's new outputs) and the resampler's new outputs.
    // Frames of scratch per stream: its new frames, one more held by the strided convs, and the kCodecMinFrames the first k = 7 conv of
    // a direction releases at once when a stream reaches them; a resampled decode's resampler gathers and writes its samples there too.
    std::vector<int> N(n, n + count), out((size_t) count, 0);
    size_t frames = 0, stage = 0;
    for (int i = 0; i < count; i++) {
        const CodecStream & t = *st[i];
        if (t.resampled) {
            const long long rin = dir == kStreamEncode ? t.rs.in + n[i] : codec_stream_ready(kStreamDecode, t.n_in + n[i]);
            out[(size_t) i] = (int)(resampler_target(t.rs, rin, finish) - t.rs.out);
            if (dir == kStreamEncode) { N[(size_t) i] = out[(size_t) i]; stage += (size_t)(t.rs.h + n[i]) * t.rs.channels; }
            else frames += (size_t)(t.rs.h + (rin - t.rs.in) + out[(size_t) i]) / 10240 + 2;
        }
        frames += (size_t)(dir == kStreamEncode ? (N[(size_t) i] + kCodecHop - 1) / kCodecHop : N[(size_t) i]) + kCodecMinFrames + 1;
    }
    if (!codec_scratch(sc, frames, n_q, fn) || !stage_scratch(sc, stage, fn)) return false;
    StreamRunner r{sc, s, count, st, finish, dir == kStreamEncode ? 1 : cm.hidden_dim, N, sc.buf[0], sc.buf[1], sc.buf[2]};
    std::vector<float *> y((size_t) count, nullptr);
    int T[kCodecMaxItems], item[kCodecMaxItems];
    if (dir == kStreamEncode) {
        // the source frames through the resamplers, straight into the encoder's input; mono 24 kHz samples copied there
        size_t off = 0;
        for (int i = 0; i < count; off += (size_t) N[(size_t) i], i++) y[(size_t) i] = r.cur + off;
        resample_step(s, st, count, n, in, nullptr, sc.stage, y.data(), out.data(), finish);
        off = 0;
        for (int i = 0; i < count; off += (size_t) N[(size_t) i], i++)
            if (n[i] && !st[i]->resampled) { BARK_CUDA_CHECK(cudaMemcpyAsync(r.cur + off, in[i], (size_t) n[i] * sizeof(float), cudaMemcpyHostToDevice, s)); g_h2d_bytes += (size_t) n[i] * sizeof(float); }
        encoder_layers(cm.enc, r);
        const int m = present(r.N, T, item);
        if (m && !rvq_encode(cm.embed, cm.embed_norm, n_q, cm.n_bins, cm.hidden_dim, r.cur, T, m, sc.codes, s)) {
            fprintf(stderr, "%s: unsupported codebook shape (%d bins of %d)\n", fn, cm.n_bins, cm.hidden_dim); return false;
        }
    } else {
        size_t off = 0;
        for (int i = 0; i < count; off += (size_t) n_q * n[i], i++)
            if (n[i]) { BARK_CUDA_CHECK(cudaMemcpyAsync(sc.codes + off, in[i], (size_t) n_q * n[i] * sizeof(int32_t), cudaMemcpyHostToDevice, s)); g_h2d_bytes += (size_t) n_q * n[i] * sizeof(int32_t); }
        const int m = present(r.N, T, item);
        if (m) rvq_decode(cm, sc.codes, n_q, T, m, r.cur, s);
        decoder_layers(cm, r);
        // the decoder's new samples through the resamplers, after its last layer: gathered in r.a, resampled into r.b
        std::vector<const float *> dev((size_t) count, nullptr);
        size_t yoff = 0;
        off = 0;
        for (int i = 0; i < count; off += (size_t) r.N[(size_t) i], i++) {
            dev[(size_t) i] = r.cur + off;
            if (st[i]->resampled) { y[(size_t) i] = r.b + yoff; yoff += (size_t) out[(size_t) i]; }
        }
        resample_step(s, st, count, r.N.data(), nullptr, dev.data(), r.a, y.data(), out.data(), finish);
    }
    // the outputs back, one synchronisation: codes, or samples (a resampled decode's from its resampler)
    std::vector<std::vector<int32_t>> codes((size_t) count);
    std::vector<std::vector<float>> audio((size_t) count);
    size_t off = 0;
    for (int i = 0; i < count; i++) {
        const size_t k = (size_t) r.N[(size_t) i];
        if (dir == kStreamEncode) {
            if (!k) continue;
            codes[(size_t) i].resize(k * n_q);
            BARK_CUDA_CHECK(cudaMemcpyAsync(codes[(size_t) i].data(), sc.codes + off, k * n_q * sizeof(int32_t), cudaMemcpyDeviceToHost, s)); g_d2h_bytes += k * n_q * sizeof(int32_t);
            off += k * n_q;
            continue;
        }
        const float * src = st[i]->resampled ? y[(size_t) i] : r.cur + off;
        const size_t ks = st[i]->resampled ? (size_t) out[(size_t) i] : k;
        off += k;
        if (!ks) continue;
        audio[(size_t) i].resize(ks);
        BARK_CUDA_CHECK(cudaMemcpyAsync(audio[(size_t) i].data(), src, ks * sizeof(float), cudaMemcpyDeviceToHost, s)); g_d2h_bytes += ks * sizeof(float);
    }
    BARK_CUDA_CHECK(cudaStreamSynchronize(s));
    for (int i = 0; i < count; i++) {
        CodecStream & t = *st[i];
        const int k = r.N[(size_t) i];
        t.n_in += dir == kStreamEncode ? N[(size_t) i] : n[i];
        t.n_out += k;
        if (dir == kStreamDecode) { t.audio.insert(t.audio.end(), audio[(size_t) i].begin(), audio[(size_t) i].end()); continue; }
        for (int f = 0; f < k; f++)                      // pending codes are frame-major
            for (int q = 0; q < n_q; q++) t.codes.push_back(codes[(size_t) i][(size_t) q * k + f]);
    }
    return true;
}

}  // namespace

bool codec_stream_init(const CodecModel & cm, CodecStream & st, int direction, int n_q, int channels, int sample_rate) {
    LayoutRunner l{direction == kStreamEncode ? 1 : cm.hidden_dim, {}};
    if (direction == kStreamEncode) encoder_layers(cm.enc, l); else decoder_layers(cm, l);
    size_t floats = (size_t) 4 * 2 * l.lstm_C;
    for (const auto & w : l.win) floats += (size_t) w.first * w.second;
    BARK_CUDA_CHECK(cudaMalloc((void **) &st.mem, floats * sizeof(float)));
    BARK_CUDA_CHECK(cudaMemset(st.mem, 0, floats * sizeof(float)));
    st.direction = direction; st.n_q = n_q;
    float * p = st.mem;
    for (int i = 0; i < 4; i++, p += 2 * l.lstm_C) st.lstm[i] = p;
    for (const auto & w : l.win) {
        CodecStream::Window x;
        x.C = w.first; x.cap = w.second; x.hist = p;
        st.win.push_back(x);
        p += (size_t) w.first * w.second;
    }
    if (channels == 1 && sample_rate == kCodecSampleRate) return true;
    // the resampler: its own copy of the rate pair's taps, and room for 2w + o - 1 frames, the most it keeps
    StreamResampler & rs = st.rs;
    st.resampled = true; rs.channels = channels; rs.rate = sample_rate;
    const std::vector<unsigned char> bytes = direction == kStreamEncode ? resample_table(sample_rate, kCodecSampleRate, &rs.t)
                                                                        : resample_table(kCodecSampleRate, sample_rate, &rs.t);
    if (!bytes.empty()) {
        BARK_CUDA_CHECK(cudaMalloc(&rs.taps, bytes.size()));
        BARK_CUDA_CHECK(cudaMemcpy(rs.taps, bytes.data(), bytes.size(), cudaMemcpyHostToDevice)); g_h2d_bytes += bytes.size();
        resample_bind(rs.t, rs.taps);
    }
    rs.cap = 2 * rs.t.w + rs.t.o - 1;
    if (rs.cap > 0) BARK_CUDA_CHECK(cudaMalloc((void **) &rs.hist, (size_t) rs.cap * channels * sizeof(float)));
    return true;
}

void CodecStream::release() {
    for (void * p : {(void *) mem, rs.taps, (void *) rs.hist}) if (p) cudaFree(p);
    mem = nullptr; rs.taps = nullptr; rs.hist = nullptr;
}

// the outputs a stream hands back: frames, or samples (at its own rate on a resampled decode)
static long long outputs(const CodecStream & t) { return t.resampled && t.direction == kStreamDecode ? t.rs.out : t.n_out; }

int codec_stream_run(const CodecModel & cm, CodecScratch & sc, cudaStream_t s, CodecStream * const * st, const void * const * in, const int * n, int count,
                     bool finish, const char * fn) {
    const int dir = st[0]->direction;
    std::vector<long long> before((size_t) count);
    for (int i = 0; i < count; i++) before[(size_t) i] = outputs(*st[i]);
    // a long push runs in passes of a bounded size per stream (the outputs do not depend on the chunks), a finish in one pass of none.
    // A resampled encode's pass takes the frames of about as many 24 kHz samples, and at most as many floats.
    const int per_frames = std::max(1, kCodecLaunchFrames / count - 2), per = dir == kStreamEncode ? per_frames * kCodecHop : per_frames;
    std::vector<int> done((size_t) count, 0), take((size_t) count), step((size_t) count, per), width((size_t) count, 1);
    for (int i = 0; i < count; i++)
        if (dir == kStreamEncode && st[i]->resampled) {
            const StreamResampler & rs = st[i]->rs;
            width[(size_t) i] = rs.channels;
            step[(size_t) i] = (int) std::max<long long>(1, std::min<long long>((long long) per * rs.t.o / rs.t.q, per / rs.channels));
        }
    std::vector<const void *> ptr((size_t) count);
    for (bool more = true; more;) {
        more = false;
        for (int i = 0; i < count; i++) {
            take[(size_t) i] = finish ? 0 : std::min(n[i] - done[(size_t) i], step[(size_t) i]);
            ptr[(size_t) i] = dir == kStreamEncode ? (const void *)((const float *) in[i] + (size_t) width[(size_t) i] * done[(size_t) i])
                                                   : (const void *)((const int32_t *) in[i] + (size_t) st[i]->n_q * done[(size_t) i]);
            more |= take[(size_t) i] > 0;
        }
        if (!more && !finish) break;
        for (int i = 0; i < count; i++) st[i]->failed = true;                          // until the pass completes
        // decode codes [n_q][n] are codebook-major: a pass of part of them goes through a contiguous copy
        std::vector<std::vector<int32_t>> part;
        if (dir == kStreamDecode && !finish)
            for (int i = 0; i < count; i++) {
                if (take[(size_t) i] == n[i]) continue;
                part.emplace_back((size_t) st[i]->n_q * take[(size_t) i]);
                for (int q = 0; q < st[i]->n_q; q++)
                    std::copy_n((const int32_t *) in[i] + (size_t) q * n[i] + done[(size_t) i], take[(size_t) i], part.back().data() + (size_t) q * take[(size_t) i]);
                ptr[(size_t) i] = part.back().data();
            }
        if (!stream_pass(cm, sc, s, st, ptr.data(), take.data(), count, finish, fn)) return -1;
        for (int i = 0; i < count; i++) { st[i]->failed = false; done[(size_t) i] += take[(size_t) i]; }
        if (finish) break;
    }
    long long added = 0;
    for (int i = 0; i < count; i++) {
        CodecStream & t = *st[i];
        if (finish) t.finished = true;
        const long long want = finish ? (dir == kStreamEncode ? (t.n_in - 1) / kCodecHop + 1 : t.n_in * kCodecHop) : codec_stream_ready(dir, t.n_in);
        // a resampler's outputs by its own rule, and the codec's inputs or outputs are its outputs or inputs
        const StreamResampler & rs = t.rs;
        const bool rs_ok = !t.resampled || (rs.out == resampler_target(rs, rs.in, finish) && (dir == kStreamEncode ? t.n_in == rs.out : rs.in == t.n_out));
        if (t.n_out != want || !rs_ok) {
            fprintf(stderr, "%s: internal error: %lld outputs after %lld inputs, the rule says %lld", fn, t.n_out, t.n_in, want);
            if (t.resampled) fprintf(stderr, "; resampler: %lld outputs after %lld frames, the rule says %lld", rs.out, rs.in, resampler_target(rs, rs.in, finish));
            fprintf(stderr, "\n");
            t.failed = true;
            return -1;
        }
        added += outputs(t) - before[(size_t) i];
    }
    return (int) std::min<long long>(added, INT_MAX);
}

}  // namespace bark
