/* TEST INFRASTRUCTURE — CPU restatement of the EnCodec encoder and of the RVQ encode.  NOT product code.
 *
 * The arithmetic the reference executes for encodec_compress_audio (encodec.cpp/encodec.cpp:878-900) at 6 kbps:
 *   encodec_forward_encoder (encoder.h:39-109) with strided_conv_1d (ops.cpp:8-75) at every conv, then
 *   encodec_forward_quantizer_encode (quantizer.h:20-76) over codebooks 0..7.
 * It is built on the decoder oracle's restated ggml kernels (oracle/bark_oracle.c, compiled into this translation unit so its
 * file-static vec_dot / LSTM / ELU are shared rather than copied): f16 dots in the AVX2/FMA lane order, glibc activations.
 * tests/encoder_oracle.py compiles it with the oracle's flags (no FP contraction) into a temporary directory.
 * Pinned against the unmodified reference's stored outputs (tests/golden/ref_pairs/encoder.npz, tests/test_encoder.py). */
#include "../oracle/bark_oracle.c"

typedef struct {
    conv_t init, final;
    struct { conv_t sc, c1, c2, ds; } blk[4];
    tensor_t ih_w[2], hh_w[2], ih_b[2], hh_b[2];
    tensor_t embed[8];
    int n_bins, hidden;
} oenc_t;

/* skip one GPT section of the file (bark.cpp:692-1078): 10-int header, tensor count, tensors */
static int skip_gpt(FILE * f) {
    int32_t hdr[10], n_tensors;
    if (!rd(f, hdr, 40) || !rd(f, &n_tensors, 4)) return 0;
    for (int i = 0; i < n_tensors; i++) {
        tensor_t t; char name[256];
        if (read_tensor_hdr(f, &t, name, sizeof name) != 1) return 0;
        free(t.data);
    }
    return 1;
}

/* the encoder tensors and codebooks 0..7 of a ggml_weights.bin; NULL when the file has no encoder */
oenc_t * oenc_load(const char * path) {
    init_f16_lut();
    FILE * f = fopen(path, "rb");
    if (!f) return NULL;
    oenc_t * m = calloc(1, sizeof(*m));
    uint32_t magic; int32_t n_vocab;
    if (!rd(f, &magic, 4) || magic != 0x67676d6cu || !rd(f, &n_vocab, 4)) goto fail;
    for (int i = 0; i < n_vocab; i++) {
        uint32_t len; char buf[1 << 12];
        if (!rd(f, &len, 4) || len > sizeof buf || (len && !rd(f, buf, len))) goto fail;
    }
    for (int g = 0; g < 3; g++) if (!skip_gpt(f)) goto fail;
    int32_t hp[9];
    if (!rd(f, &magic, 4) || magic != 0x67676d6cu || !rd(f, hp, 36)) goto fail;
    m->hidden = hp[1]; m->n_bins = hp[5];
    int n_enc = 0;
    for (;;) {
        tensor_t t; char name[256], tail[64];
        const int r = read_tensor_hdr(f, &t, name, sizeof name);
        if (r == 0) break;
        if (r < 0) goto fail;
        int i, q, keep = 1;
        if (sscanf(name, "quantizer.vq.layers.%d._codebook.embed", &q) == 1 && q < 8) m->embed[q] = t;
        else if (!strcmp(name, "encoder.model.0.conv.conv.weight")) m->init.w = t;
        else if (!strcmp(name, "encoder.model.0.conv.conv.bias")) m->init.b = t;
        else if (!strcmp(name, "encoder.model.15.conv.conv.weight")) m->final.w = t;
        else if (!strcmp(name, "encoder.model.15.conv.conv.bias")) m->final.b = t;
        else if (sscanf(name, "encoder.model.13.lstm.%63s", tail) == 1) {
            const int l = tail[strlen(tail) - 1] - '0';
            if      (!strncmp(tail, "weight_ih", 9)) m->ih_w[l] = t;
            else if (!strncmp(tail, "weight_hh", 9)) m->hh_w[l] = t;
            else if (!strncmp(tail, "bias_ih", 7))   m->ih_b[l] = t;
            else                                      m->hh_b[l] = t;
        } else if (sscanf(name, "encoder.model.%d.%63s", &i, tail) == 2) {
            /* blocks: model.{3b+1} resblock (block.1 = conv_1, block.3 = conv_2, shortcut), model.{3(b+1)} down-sampling conv */
            const int isw = strstr(tail, "weight") != NULL;
            conv_t * cv = i % 3 == 0 ? &m->blk[i / 3 - 1].ds
                        : !strncmp(tail, "block.1", 7) ? &m->blk[(i - 1) / 3].c1 : !strncmp(tail, "block.3", 7) ? &m->blk[(i - 1) / 3].c2 : &m->blk[(i - 1) / 3].sc;
            if (isw) cv->w = t; else cv->b = t;
        } else { free(t.data); keep = 0; }
        n_enc += keep && !strncmp(name, "encoder.", 8);
    }
    fclose(f);
    if (n_enc == 0) { free(m); return NULL; }
    return m;
fail:
    fclose(f); free(m); return NULL;
}

/* strided_conv_1d (ops.cpp:59-75) on x [Cin][L]: reflect-pad k - stride left and `extra` right (ggml.c:15581-15589), im2col to f16
 * at the stride (ggml.c:14892-14960), f16 dot over c*k + j, bias added in f32.  Returns [Cout][*T_out]. */
static float * conv_strided(const float * x, int Cin, int L, const conv_t * cv, int stride, int * T_out) {
    const int k = cv->w.ne[0], Cout = cv->w.ne[2], padl = k - stride;
    assert(cv->w.ne[1] == Cin);
    /* get_extra_padding_for_conv_1d (ops.cpp:10-16), in float as there */
    const float length = (float) L, ks = (float) k, st = (float) stride, pt = (float) padl;
    const float n_frames = (length - ks + pt) / st + 1.0f;
    const int ideal_length = (int)((ceilf(n_frames) - 1.0f) * st + (ks - pt));
    const int extra = (int)((float) ideal_length - length);
    const int Lp = L + padl + extra, T = (Lp - k) / stride + 1;
    assert(padl < L && extra < L);
    uint16_t * xp = malloc((size_t) Cin * Lp * 2);
    for (int c = 0; c < Cin; c++) {
        uint16_t * row = xp + (size_t) c * Lp;
        for (int t = 0; t < L; t++) row[padl + t] = orc_f32_to_f16(x[(size_t) c * L + t]);
        for (int i = 1; i <= padl; i++) row[padl - i] = row[padl + i];
        for (int i = 1; i <= extra; i++) row[padl + L - 1 + i] = row[padl + L - 1 - i];
    }
    float * y = malloc((size_t) Cout * T * 4);
    #pragma omp parallel
    {
        uint16_t * col = malloc((size_t) Cin * k * 2);
        #pragma omp for schedule(static)
        for (int t = 0; t < T; t++) {
            for (int c = 0; c < Cin; c++) for (int j = 0; j < k; j++) col[c * k + j] = xp[(size_t) c * Lp + (size_t) t * stride + j];
            for (int o = 0; o < Cout; o++) {
                const float v = orc_vec_dot_f16(Cin * k, col, (const uint16_t *) cv->w.data + (size_t) o * Cin * k);
                y[(size_t) o * T + t] = ((const float *) cv->b.data)[o] + v;
            }
        }
        free(col);
    }
    free(xp);
    *T_out = T;
    return y;
}

/* encodec_forward_quantizer_encode (quantizer.h:20-76) for one frame at a time; codebooks cb[q] [n_bins][hidden] */
static void rvq_core(const float * latent, int T, const float * const * cb, int hidden, int n_bins, int n_q, int32_t * codes) {
    float * nrm = malloc((size_t) n_q * n_bins * 4);
    for (int q = 0; q < n_q; q++)
        for (int j = 0; j < n_bins; j++) {                       /* sum_rows(sqr(embed)): ggml_vec_sum_f32 sums in double */
            double s = 0.0;
            for (int i = 0; i < hidden; i++) { const float e = cb[q][(size_t) j * hidden + i]; const float p = e * e; s += (double) p; }
            nrm[(size_t) q * n_bins + j] = (float) s;
        }
    #pragma omp parallel
    {
        float * r = malloc((size_t) hidden * 4);
        #pragma omp for schedule(static)
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < hidden; i++) r[i] = latent[(size_t) i * T + t];
            for (int q = 0; q < n_q; q++) {
                double s = 0.0;
                for (int i = 0; i < hidden; i++) { const float p = r[i] * r[i]; s += (double) p; }
                const float sf = (float) s;
                float max = -INFINITY; int idx = 0;
                for (int j = 0; j < n_bins; j++) {
                    const float dot = orc_vec_dot_f32(hidden, cb[q] + (size_t) j * hidden, r);
                    const float dp = dot * -2.0f;                /* ggml_scale */
                    const float a = sf + dp;                     /* add(repeat(sqr_inp_nrm), dp) */
                    const float b = nrm[(size_t) q * n_bins + j] + a;   /* add(repeat(sqr_embed_nrm^T), dist) */
                    const float v = -b;                          /* neg */
                    max = max > v ? max : v;                     /* ggml_vec_argmax_f32 (ggml.c:2965-2973), literally */
                    if (max == v) idx = j;
                }
                codes[(size_t) q * T + t] = idx;
                for (int i = 0; i < hidden; i++) r[i] = r[i] - cb[q][(size_t) idx * hidden + i];
            }
        }
        free(r);
    }
    free(nrm);
}

/* codebooks [n_q][n_bins][hidden] contiguous; codes [n_q][T] */
void orc_rvq_encode(const float * latent, int T, const float * codebooks, int hidden, int n_bins, int n_q, int32_t * codes) {
    const float * cb[32];
    for (int q = 0; q < n_q && q < 32; q++) cb[q] = codebooks + (size_t) q * n_bins * hidden;
    rvq_core(latent, T, cb, hidden, n_bins, n_q, codes);
}

/* encodec_compress_audio at 6 kbps: audio [n] -> codes [8][T] and latent [hidden][T] (either may be NULL); returns T or -1 */
int orc_encodec_encode(oenc_t * m, const float * audio, int n, int32_t * codes, float * latent) {
    static const int ratios[4] = {8, 5, 4, 2};
    if (!m || n < 1921) return -1;
    int L = n, C = m->init.w.ne[2], T;
    float * y = conv_strided(audio, 1, n, &m->init, 1, &L);                   /* encoder.h:49 */
    for (int b = 0; b < 4; b++) {                                              /* encoder.h:52-83 */
        int Ls;
        float * sc = conv_strided(y, C, L, &m->blk[b].sc, 1, &Ls);
        elu_inplace(y, (size_t) C * L);
        float * r1 = conv_strided(y, C, L, &m->blk[b].c1, 1, &Ls); free(y);
        elu_inplace(r1, (size_t)(C / 2) * L);
        float * r2 = conv_strided(r1, C / 2, L, &m->blk[b].c2, 1, &Ls); free(r1);
        for (size_t i = 0; i < (size_t) C * L; i++) r2[i] = r2[i] + sc[i];  /* add(current, shortcut) */
        free(sc);
        elu_inplace(r2, (size_t) C * L);
        y = conv_strided(r2, C, L, &m->blk[b].ds, ratios[3 - b], &L); free(r2);
        C *= 2;
    }
    T = L;
    float * h1 = lstm_layer(y, C, T, &m->ih_w[0], &m->hh_w[0], &m->ih_b[0], &m->hh_b[0]);
    float * h2 = lstm_layer(h1, C, T, &m->ih_w[1], &m->hh_w[1], &m->ih_b[1], &m->hh_b[1]);
    for (size_t i = 0; i < (size_t) C * T; i++) y[i] = y[i] + h2[i];         /* encoder.h:98 inpL + out */
    free(h1); free(h2);
    elu_inplace(y, (size_t) C * T);
    int T2;
    float * lat = conv_strided(y, C, T, &m->final, 1, &T2); free(y);
    if (latent) memcpy(latent, lat, (size_t) m->hidden * T * 4);
    if (codes) {
        const float * cb[8];
        for (int q = 0; q < 8; q++) cb[q] = m->embed[q].data;
        rvq_core(lat, T, cb, m->hidden, m->n_bins, 8, codes);
    }
    free(lat);
    return T;
}

/* ------------------------------------------------------------------------------------------ */
/* The EnCodec ops one at a time on raw arrays, for the kernel-by-kernel GPU tests: thin wrappers around the static cores above, */
/* one item each.  tests/test_codec_oracle_ops.py chains them into orc_encodec_decode and this file's encoder latent.          */
/* ------------------------------------------------------------------------------------------ */
static float * elu_copy(const float * x, size_t n, int elu_in) {
    float * y = malloc(n * 4);
    memcpy(y, x, n * 4);
    if (elu_in) elu_inplace(y, n);
    return y;
}

/* strided_conv_1d on x [Cin][L], w [Cout][Cin][k] f16: ELU on the input when elu_in, stride 1 through the decoder's conv1d, else
 * conv_strided; resid [Cout][T] (may be NULL) added to the result.  Returns T, y [Cout][T]. */
int orc_codec_conv1d(const float * x, int Cin, int L, const uint16_t * w, const float * bias, int Cout, int k, int stride, int elu_in,
                     const float * resid, float * y) {
    conv_t cv = {{1, {k, Cin, Cout}, 3, (void *) w}, {0, {Cout, 1, 1}, 1, (void *) bias}};
    float * xin = elu_copy(x, (size_t) Cin * L, elu_in), * out;
    int T = L;
    if (stride == 1) out = conv1d(xin, Cin, L, &cv);
    else             out = conv_strided(xin, Cin, L, &cv, stride, &T);
    if (resid) for (size_t i = 0; i < (size_t) Cout * T; i++) out[i] = out[i] + resid[i];
    memcpy(y, out, (size_t) Cout * T * 4);
    free(xin); free(out);
    return T;
}

/* ELU, then strided_conv_transpose_1d with k = 2 stride (right trim, bias): x [Cin][T], w [Cin][Cout][k] f16 -> y [Cout][T stride] */
int orc_codec_convtr1d(const float * x, int Cin, int T, const uint16_t * w, const float * bias, int Cout, int stride, float * y) {
    conv_t cv = {{1, {2 * stride, Cout, Cin}, 3, (void *) w}, {0, {Cout, 1, 1}, 1, (void *) bias}};
    float * xin = elu_copy(x, (size_t) Cin * T, 1);
    int L;
    float * out = convtr1d(xin, Cin, T, &cv, stride, &L);
    memcpy(y, out, (size_t) Cout * L * 4);
    free(xin); free(out);
    return L;
}

/* one LSTM layer: x [C][T], wih / whh [4C][C] f16, bih / bhh [4C] -> out [C][T], plus skip [C][T] (decoder.h:72) when not NULL */
void orc_codec_lstm(const float * x, int C, int T, const uint16_t * wih, const uint16_t * whh, const float * bih, const float * bhh, const float * skip,
                    float * out) {
    const tensor_t ih = {1, {C, 4 * C, 1}, 2, (void *) wih}, hh = {1, {C, 4 * C, 1}, 2, (void *) whh};
    const tensor_t bi = {0, {4 * C, 1, 1}, 1, (void *) bih}, bh = {0, {4 * C, 1, 1}, 1, (void *) bhh};
    float * h = lstm_layer(x, C, T, &ih, &hh, &bi, &bh);
    for (size_t i = 0; i < (size_t) C * T; i++) out[i] = skip ? skip[i] + h[i] : h[i];
    free(h);
}

/* the quantizer decode over codebooks [n_q][n_bins][hidden]: codes [n_q][T] -> x [hidden][T] */
void orc_codec_rvq_decode(const int32_t * codes, int n_q, int T, const float * codebooks, int hidden, int n_bins, float * x) {
    const float * cb[32];
    for (int q = 0; q < n_q && q < 32; q++) cb[q] = codebooks + (size_t) q * n_bins * hidden;
    quantizer_decode(codes, n_q, T, cb, hidden, x);
}

/* The host libm under the codec and soft_max, as the oracle calls it, on the floats of bit patterns x[0..n): fn 0 expm1f, 1 tanhf,
 * 2 expf, 3 ggml_v_expf, 4 ELU, 5 the LSTM's sigmoid, 6 the f16 round trip (bark_b200_device_math's order). */
void orc_libm(int fn, const uint32_t * x, long long n, float * out) {
    #pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; i++) {
        const float v = u2f(x[i]);
        float r;
        switch (fn) {
        case 0:  r = expm1f(v); break;
        case 1:  r = tanhf(v); break;
        case 2:  r = expf(v); break;
        case 3:  r = orc_v_expf(v); break;
        case 4:  r = (v > 0.f) ? v : expm1f(v); break;
        case 5:  r = 1.f / (1.f + expf(-v)); break;
        default: r = orc_f16_to_f32(orc_f32_to_f16(v)); break;
        }
        out[i] = r;
    }
}
