/* TEST INFRASTRUCTURE — CPU oracle for the bark.cpp hot path.  NOT product code.
 * See bark_oracle.h for scope, pinning and who may load it.
 *
 * Everything is written as scalar C with explicit fmaf()/separate mul+add so that the result does
 * not depend on how this file is compiled (oracle/Makefile passes -ffp-contract=off).  "Lane
 * order" comments describe the accumulation structure of the pinned reference build
 * (gcc 13 -O3 -mavx2 -mfma -mf16c): GGML_F32_STEP = GGML_F16_STEP = 32, 4 accumulators x 8 lanes
 * (ggml.c:1384-1480).
 */
#define _GNU_SOURCE
#include "bark_oracle.h"

#include <assert.h>
#include <ctype.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------ */
/* fp16 <-> fp32 (IEEE binary16, round-to-nearest-even; what F16C vcvtps2ph/vcvtph2ps do,      */
/* ggml.c:538 ggml_fp32_to_fp16_row / ggml-impl.h GGML_COMPUTE_FP32_TO_FP16)                   */
/* ------------------------------------------------------------------------------------------ */
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float    u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

float orc_f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp  = (h >> 10) & 0x1f;
    uint32_t man  = h & 0x3ffu;
    if (exp == 0) {
        if (man == 0) return u2f(sign);
        /* subnormal: value = man * 2^-24 */
        float v = (float) man * 0x1p-24f;
        return u2f(f2u(v) | sign);
    }
    if (exp == 31) return u2f(sign | 0x7f800000u | (man << 13));
    return u2f(sign | ((exp + 112) << 23) | (man << 13));
}

uint16_t orc_f32_to_f16(float f) {
    uint32_t x = f2u(f);
    uint32_t sign = (x >> 16) & 0x8000u;
    uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (ax > 0x7f800000u ? (0x200u | ((ax >> 13) & 0x3ffu)) : 0));
    if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);          /* >= 65520 rounds to inf */
    if (ax < 0x33000001u) return (uint16_t) sign;                      /* <= 2^-25 rounds to 0 (ties-to-even) */
    int e = (int)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7fffffu) | 0x800000u;                         /* 24-bit significand */
    int shift;                                                         /* bits to drop */
    uint32_t base;
    if (e < -14) { shift = 13 + (-14 - e); base = 0; }                 /* subnormal half */
    else         { shift = 13;             base = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
    uint32_t q = m >> shift;
    uint32_t rem = m & ((1u << shift) - 1u);
    uint32_t half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1u))) q++;
    return (uint16_t)(sign | (base + q));                              /* carry into exponent is correct */
}

/* ------------------------------------------------------------------------------------------ */
/* dot products (ggml.c:2144 ggml_vec_dot_f32, ggml.c:2251 ggml_vec_dot_f16)                   */
/* ------------------------------------------------------------------------------------------ */
static inline float reduce32(const float * a) {
    /* GGML_F32x8_REDUCE (ggml.c:1405-1422): x0+=x2; x1+=x3; x0+=x1; t[l]=x0[l]+x0[l+4];
     * (t0+t1)+(t2+t3) */
    float x0[8], x1[8], t[4];
    for (int l = 0; l < 8; l++) x0[l] = a[l] + a[16 + l];
    for (int l = 0; l < 8; l++) x1[l] = a[8 + l] + a[24 + l];
    for (int l = 0; l < 8; l++) x0[l] = x0[l] + x1[l];
    for (int l = 0; l < 4; l++) t[l] = x0[l] + x0[l + 4];
    return (t[0] + t[1]) + (t[2] + t[3]);
}

float orc_vec_dot_f32(int n, const float * x, const float * y) {
    const int np = n & ~31;
    float acc[32];
    for (int v = 0; v < 32; v++) acc[v] = 0.0f;
    for (int i = 0; i < np; i += 32)
        for (int v = 0; v < 32; v++) acc[v] = fmaf(x[i + v], y[i + v], acc[v]);
    float sumf = reduce32(acc);
    /* leftovers (ggml.c:2172-2174 `sumf += x[i]*y[i]` in float).  As compiled in the pinned build
     * (objdump of ggml_vec_dot_f32 in oracle/_ref/ggml.o) gcc vectorises the products: full
     * groups of 8, then one group of 4, use a rounded vmulps followed by sequential vaddss; the
     * final <=3 elements are contracted to vfmadd231ss. */
    int i = np;
    int r = n - np;
    while (r >= 8) { for (int k = 0; k < 8; k++) { float p = x[i + k] * y[i + k]; sumf = sumf + p; } i += 8; r -= 8; }
    if (r >= 4)    { for (int k = 0; k < 4; k++) { float p = x[i + k] * y[i + k]; sumf = sumf + p; } i += 4; r -= 4; }
    for (; r > 0; r--, i++) sumf = fmaf(x[i], y[i], sumf);
    return sumf;
}

/* strided variant: x has element stride sx (used for V^T columns out of the KV cache) */
static float vec_dot_f32_sx(int n, const float * x, int sx, const float * y) {
    const int np = n & ~31;
    float acc[32];
    for (int v = 0; v < 32; v++) acc[v] = 0.0f;
    for (int i = 0; i < np; i += 32)
        for (int v = 0; v < 32; v++) acc[v] = fmaf(x[(size_t)(i + v) * sx], y[i + v], acc[v]);
    float sumf = reduce32(acc);
    int i = np, r = n - np;
    while (r >= 8) { for (int k = 0; k < 8; k++) { float p = x[(size_t)(i + k) * sx] * y[i + k]; sumf = sumf + p; } i += 8; r -= 8; }
    if (r >= 4)    { for (int k = 0; k < 4; k++) { float p = x[(size_t)(i + k) * sx] * y[i + k]; sumf = sumf + p; } i += 4; r -= 4; }
    for (; r > 0; r--, i++) sumf = fmaf(x[(size_t) i * sx], y[i], sumf);
    return sumf;
}

static float f16_lut[65536];
static int   f16_lut_ready = 0;
static void  init_f16_lut(void) { if (!f16_lut_ready) { for (int i = 0; i < 65536; i++) f16_lut[i] = orc_f16_to_f32((uint16_t) i); f16_lut_ready = 1; } }

float orc_vec_dot_f16(int n, const uint16_t * x, const uint16_t * y) {
    init_f16_lut();
    const int np = n & ~31;
    float acc[32];
    for (int v = 0; v < 32; v++) acc[v] = 0.0f;
    for (int i = 0; i < np; i += 32)
        for (int v = 0; v < 32; v++) acc[v] = fmaf(f16_lut[x[i + v]], f16_lut[y[i + v]], acc[v]);
    double sumf = (double) reduce32(acc);
    for (int i = np; i < n; i++) { float p = f16_lut[x[i]] * f16_lut[y[i]]; sumf += (double) p; }   /* ggml.c:2281-2283 */
    return (float) sumf;
}

/* ------------------------------------------------------------------------------------------ */
/* LayerNorm (ggml.c:11964-12013), GELU table (ggml.c:2546-2571, 3795-3810)                    */
/* ------------------------------------------------------------------------------------------ */
void orc_norm(int n, const float * x, float * y, float eps) {
    double sum = 0.0;
    for (int i = 0; i < n; i++) sum += (double) x[i];
    float mean = (float)(sum / (double) n);
    double sum2 = 0.0;
    for (int i = 0; i < n; i++) { float v = x[i] - mean; y[i] = v; float vv = v * v; sum2 += (double) vv; }
    float variance = (float)(sum2 / (double) n);
    const float scale = 1.0f / sqrtf(variance + eps);
    for (int i = 0; i < n; i++) y[i] = y[i] * scale;
}

static uint16_t gelu_tab[65536];
static int      gelu_ready = 0;
static void init_gelu(void) {
    if (gelu_ready) return;
    init_f16_lut();
    /* ggml_gelu_f32 (ggml.c:2546): 0.5f*x*(1.0f + tanhf(SQRT_2_OVER_PI*x*(1.0f + GELU_COEF_A*x*x)))
     * The pinned build contracts `1.0f + (GELU_COEF_A*x)*x` into one fma (checked against the
     * table dumped from the reference, tests/golden/gelu_table_f16.bin); the other products are
     * plain rounded multiplies. */
    const float A = 0.044715f, S = 0.79788456080286535587989211986876f;
    for (int i = 0; i < 65536; i++) {
        float x = f16_lut[i];
        float inner = fmaf(A * x, x, 1.0f);
        float t = tanhf((S * x) * inner);
        float g = (0.5f * x) * (1.0f + t);
        gelu_tab[i] = orc_f32_to_f16(g);
    }
    gelu_ready = 1;
}
static inline float gelu_f32(float x) {           /* ggml_vec_gelu_f32, GGML_GELU_FP16 branch */
    if (x <= -10.0f) return 0.0f;
    if (x >= 10.0f) return x;
    return f16_lut[gelu_tab[orc_f32_to_f16(x)]];
}
/* gelu evaluated at every f16 input, result rounded to f16 (what a one-op ggml_gelu graph returns) */
void orc_gelu_table(uint16_t * out) { init_gelu(); for (int i = 0; i < 65536; i++) out[i] = orc_f32_to_f16(gelu_f32(f16_lut[i])); }

/* ------------------------------------------------------------------------------------------ */
/* soft_max row (ggml.c:13953-14042, ggml_vec_soft_max_f32 ggml.c:2826-2888, AVX2 ggml_v_expf   */
/* ggml.c:2706-2746)                                                                           */
/* ------------------------------------------------------------------------------------------ */
float orc_v_expf(float x) {
    const float r = 0x1.8p23f;
    const float z = fmaf(x, 0x1.715476p+0f, r);
    const float n = z - r;
    const float b = fmaf(-n, 0x1.7f7d1cp-20f, fmaf(-n, 0x1.62e4p-1f, x));
    const uint32_t e = f2u(z) << 23;
    const float k = u2f(e + f2u(1.0f));
    const float an = fabsf(n);
    const float u = b * b;
    const float j = fmaf(fmaf(fmaf(0x1.0e4020p-7f, b, 0x1.573e2ep-5f), u, fmaf(0x1.555e66p-3f, b, 0x1.fffdb6p-2f)), u,
                         0x1.ffffecp-1f * b);
    if (!(an > 126.0f)) return fmaf(j, k, k);
    const uint32_t g = (n <= 0.0f) ? 0x82000000u : 0u;
    const float s1 = u2f(g + 0x7f000000u);
    const float s2 = u2f(e - g);
    if (an > 192.0f) return s1 * s1;
    return fmaf(s2, j, s2) * s1;
}

void orc_soft_max(int n, const float * x, float * y) {
    float max = -INFINITY;
    for (int i = 0; i < n; i++) max = x[i] > max ? x[i] : max;      /* ggml_vec_max_f32 */
    double sum = 0.0;
    int i = 0;
    for (; i + 7 < n; i += 8) {
        float v[8];
        for (int l = 0; l < 8; l++) { v[l] = orc_v_expf(x[i + l] - max); y[i + l] = v[l]; }
        float t0 = v[4] + v[0], t1 = v[5] + v[1], t2 = v[6] + v[2], t3 = v[7] + v[3];   /* hi128 + lo128 */
        float s0 = t0 + t2, s1 = t1 + t3;                                               /* + movehl */
        float s = s0 + s1;                                                              /* add_ss movehdup */
        sum += (double) s;
    }
    for (; i < n; i++) { float val = expf(x[i] - max); sum += (double) val; y[i] = val; }
    sum = 1.0 / sum;
    const float sc = (float) sum;                                    /* ggml_vec_scale_f32(nc, dp, sum) */
    for (int k = 0; k < n; k++) y[k] = y[k] * sc;
}

/* ------------------------------------------------------------------------------------------ */
/* mt19937 + libstdc++ discrete_distribution (bits/random.tcc:2657-2730, 3349-3384)            */
/* ------------------------------------------------------------------------------------------ */
void orc_mt_seed(uint32_t * st, uint32_t seed) {
    st[0] = seed;
    for (int i = 1; i < 624; i++) st[i] = 1812433253u * (st[i - 1] ^ (st[i - 1] >> 30)) + (uint32_t) i;
    st[624] = 624;
}
uint32_t orc_mt_next(uint32_t * st) {
    if (st[624] >= 624) {
        for (int i = 0; i < 624; i++) {
            uint32_t y = (st[i] & 0x80000000u) | (st[(i + 1) % 624] & 0x7fffffffu);
            st[i] = st[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        st[624] = 0;
    }
    uint32_t y = st[st[624]++];
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}
static double mt_canonical(uint32_t * st) {        /* generate_canonical<double,53>: two draws */
    double sum = 0.0, tmp = 1.0;
    for (int k = 0; k < 2; k++) { sum += (double) orc_mt_next(st) * tmp; tmp *= 4294967296.0; }
    double ret = sum / tmp;
    if (ret >= 1.0) ret = nextafter(1.0, 0.0);
    return ret;
}

/* ------------------------------------------------------------------------------------------ */
/* model container + loader (file format: SURVEY.md App. A; bark.cpp:664-1163,                 */
/* encodec.cpp/encodec.cpp:141-502)                                                            */
/* ------------------------------------------------------------------------------------------ */
typedef struct { int type; int ne[3]; int n_dims; void * data; } tensor_t;   /* type: 0 f32, 1 f16, 2 q4_0 */

typedef struct {
    int32_t n_layer, n_head, n_embd, block_size, bias, n_in_vocab, n_out_vocab, n_lm_heads, n_wtes, ftype;
    tensor_t wte[8], lm_head[8], wpe, ln_f_g, ln_f_b;
    struct { tensor_t ln_1_g, ln_1_b, ln_2_g, ln_2_b, c_attn, c_proj, fc, proj; } * layers;
    float * mem_k, * mem_v;      /* [n_layer][block_size][n_embd] f32 (bark.cpp:980-981) */
} gpt_t;

typedef struct { tensor_t w, b; } conv_t;
typedef struct {
    conv_t init, final;
    tensor_t lstm_ih_w[2], lstm_hh_w[2], lstm_ih_b[2], lstm_hh_b[2];
    struct { conv_t us, c1, c2, sc; } blk[4];
    tensor_t embed[32];
    int hidden_dim, n_filters, kernel_size, res_kernel, n_bins;
} codec_t;

struct orc_ctx {
    int n_vocab; char ** vocab;        /* id = index */
    gpt_t gpt[3];
    codec_t codec;
    uint32_t rng[625];
    float temp, fine_temp, min_eos_p;
    int n_steps_text_encoder;
};

static int rd(FILE * f, void * p, size_t n) { return fread(p, 1, n, f) == n; }

static size_t tensor_bytes(int type, size_t nel) {
    if (type == 0) return nel * 4;
    if (type == 1) return nel * 2;
    if (type == 2) return nel / 32 * 18;      /* q4_0 */
    if (type == 3) return nel / 32 * 20;      /* q4_1 */
    if (type == 6) return nel / 32 * 22;      /* q5_0 */
    if (type == 7) return nel / 32 * 24;      /* q5_1 */
    if (type == 8) return nel / 32 * 34;      /* q8_0 */
    return 0;
}

static int read_tensor_hdr(FILE * f, tensor_t * t, char * name, int name_cap) {
    int32_t n_dims, len, ttype;
    if (!rd(f, &n_dims, 4)) return 0;
    if (!rd(f, &len, 4) || !rd(f, &ttype, 4)) return -1;
    if (n_dims < 1 || n_dims > 3 || len <= 0 || len >= name_cap) return -1;
    t->ne[0] = t->ne[1] = t->ne[2] = 1;
    for (int i = 0; i < n_dims; i++) if (!rd(f, &t->ne[i], 4)) return -1;
    if (!rd(f, name, len)) return -1;
    name[len] = 0;
    t->type = ttype; t->n_dims = n_dims;
    size_t nb = tensor_bytes(ttype, (size_t) t->ne[0] * t->ne[1] * t->ne[2]);
    if (nb == 0) return -1;
    t->data = malloc(nb);
    if (!t->data || !rd(f, t->data, nb)) return -1;
    return 1;
}

static int load_gpt(FILE * f, gpt_t * m) {
    if (!rd(f, &m->n_layer, 40)) return 0;       /* 10 int32 in header order */
    m->ftype %= 1000;
    m->layers = calloc(m->n_layer, sizeof(*m->layers));
    int32_t n_tensors;
    if (!rd(f, &n_tensors, 4)) return 0;
    for (int i = 0; i < n_tensors; i++) {
        tensor_t t; char name[256];
        if (read_tensor_hdr(f, &t, name, sizeof name) != 1) return 0;
        int l, k;
        if (sscanf(name, "model/wte/%d", &k) == 1) m->wte[k] = t;
        else if (sscanf(name, "model/lm_head/%d", &k) == 1) m->lm_head[k] = t;
        else if (!strcmp(name, "model/wpe")) m->wpe = t;
        else if (!strcmp(name, "model/ln_f/g")) m->ln_f_g = t;
        else if (!strcmp(name, "model/ln_f/b")) m->ln_f_b = t;
        else if (sscanf(name, "model/h%d/", &l) == 1 && l >= 0 && l < m->n_layer) {
            const char * s = strchr(name + 7, '/') + 1;
            if      (!strcmp(s, "ln_1/g")) m->layers[l].ln_1_g = t;
            else if (!strcmp(s, "ln_1/b")) m->layers[l].ln_1_b = t;
            else if (!strcmp(s, "ln_2/g")) m->layers[l].ln_2_g = t;
            else if (!strcmp(s, "ln_2/b")) m->layers[l].ln_2_b = t;
            else if (!strcmp(s, "attn/c_attn/w")) m->layers[l].c_attn = t;
            else if (!strcmp(s, "attn/c_proj/w")) m->layers[l].c_proj = t;
            else if (!strcmp(s, "mlp/c_fc/w")) m->layers[l].fc = t;
            else if (!strcmp(s, "mlp/c_proj/w")) m->layers[l].proj = t;
            else return 0;
        } else return 0;
    }
    if (m->n_lm_heads == 1 && m->n_wtes == 1) {
        size_t n = (size_t) m->n_layer * m->block_size * m->n_embd;
        m->mem_k = calloc(n, 4); m->mem_v = calloc(n, 4);
    }
    return 1;
}

static int load_codec(FILE * f, codec_t * c) {
    uint32_t magic; int32_t hp[9];
    if (!rd(f, &magic, 4) || magic != 0x67676d6cu || !rd(f, hp, 36)) return 0;
    c->hidden_dim = hp[1]; c->n_filters = hp[2]; c->kernel_size = hp[3]; c->res_kernel = hp[4]; c->n_bins = hp[5];
    for (;;) {
        tensor_t t; char name[256];
        int r = read_tensor_hdr(f, &t, name, sizeof name);
        if (r == 0) break;
        if (r < 0) return 0;
        int i, q; char tail[64];
        if (!strncmp(name, "encoder.", 8)) { free(t.data); continue; }          /* never used by decode */
        if (!strcmp(name, "decoder.model.0.conv.conv.weight")) c->init.w = t;
        else if (!strcmp(name, "decoder.model.0.conv.conv.bias")) c->init.b = t;
        else if (!strcmp(name, "decoder.model.15.conv.conv.weight")) c->final.w = t;
        else if (!strcmp(name, "decoder.model.15.conv.conv.bias")) c->final.b = t;
        else if (sscanf(name, "decoder.model.1.lstm.%63s", tail) == 1) {
            int l = tail[strlen(tail) - 1] - '0';
            if      (!strncmp(tail, "weight_ih", 9)) c->lstm_ih_w[l] = t;
            else if (!strncmp(tail, "weight_hh", 9)) c->lstm_hh_w[l] = t;
            else if (!strncmp(tail, "bias_ih", 7))   c->lstm_ih_b[l] = t;
            else if (!strncmp(tail, "bias_hh", 7))   c->lstm_hh_b[l] = t;
            else return 0;
        } else if (sscanf(name, "quantizer.vq.layers.%d._codebook.embed", &q) == 1) c->embed[q] = t;
        else if (sscanf(name, "decoder.model.%d.%63s", &i, tail) == 2) {
            int isw = strstr(tail, "weight") != NULL;
            if (i % 3 == 0) { int b = i / 3 - 1; if (isw) c->blk[b].us.w = t; else c->blk[b].us.b = t; }
            else {
                int b = (i - 1) / 3 - 1;
                conv_t * cv = !strncmp(tail, "block.1", 7) ? &c->blk[b].c1 : !strncmp(tail, "block.3", 7) ? &c->blk[b].c2 : &c->blk[b].sc;
                if (isw) cv->w = t; else cv->b = t;
            }
        } else return 0;
    }
    return 1;
}

orc_ctx * orc_load(const char * path, uint32_t seed) {
    init_f16_lut(); init_gelu();
    FILE * f = fopen(path, "rb");
    if (!f) return NULL;
    orc_ctx * c = calloc(1, sizeof(*c));
    uint32_t magic;
    if (!rd(f, &magic, 4) || magic != 0x67676d6cu) goto fail;
    if (!rd(f, &c->n_vocab, 4)) goto fail;
    c->vocab = calloc(c->n_vocab, sizeof(char *));
    for (int i = 0; i < c->n_vocab; i++) {
        uint32_t len; if (!rd(f, &len, 4)) goto fail;
        c->vocab[i] = calloc(len + 1, 1);
        if (len && !rd(f, c->vocab[i], len)) goto fail;
    }
    for (int g = 0; g < 3; g++) if (!load_gpt(f, &c->gpt[g])) goto fail;
    if (!load_codec(f, &c->codec)) goto fail;
    fclose(f);
    orc_mt_seed(c->rng, seed);
    c->temp = 0.7f; c->fine_temp = 0.5f; c->min_eos_p = 0.2f; c->n_steps_text_encoder = 768;   /* bark.cpp:2202-2232 */
    return c;
fail:
    fclose(f); free(c); return NULL;
}

void orc_free(orc_ctx * c) { free(c); /* fixtures are short-lived processes; tensors are left to exit */ }
void orc_reseed(orc_ctx * c, uint32_t seed) { orc_mt_seed(c->rng, seed); }
void orc_hparams(orc_ctx * c, int which, int32_t * out) { memcpy(out, &c->gpt[which].n_layer, 40); }
void orc_set_params(orc_ctx * c, float temp, float fine_temp, float min_eos_p, int n_steps) {
    c->temp = temp; c->fine_temp = fine_temp; c->min_eos_p = min_eos_p; if (n_steps > 0) c->n_steps_text_encoder = n_steps;
}

/* ------------------------------------------------------------------------------------------ */
/* q4_0 (ggml-common.h:144-148, ggml-quants.c:848-871 quantize_row_q8_0, :3921 vec_dot)        */
/* ------------------------------------------------------------------------------------------ */
typedef struct { uint16_t d; int8_t qs[32]; } q8_0_t;

/* _mm256_round_ps(nearest-even) then _mm256_cvtps_epi32: a non-finite or out-of-range value becomes INT_MIN (the "integer
 * indefinite"); the saturating packs (packs_epi32, packs_epi16) then clamp the int32 to a byte */
static int32_t cvt_epi32(float v) { return isfinite(v) && fabsf(v) < 2147483648.0f ? (int32_t) nearbyintf(v) : INT32_MIN; }
static int8_t packs8(int32_t i) { return (int8_t)(i < -128 ? -128 : i > 127 ? 127 : i); }

static void quantize_row_q8_0(const float * x, q8_0_t * y, int k) {
    /* AVX2 branch: amax over the block, d = amax/127, id = 127/amax, q = round-to-nearest(x*id)
     * (ggml-quants.c:895-960: _mm256_round_ps nearest-even on x*id) */
    for (int b = 0; b < k / 32; b++) {
        float amax = 0.0f;
        for (int j = 0; j < 32; j++) { float a = fabsf(x[b * 32 + j]); amax = a > amax ? a : amax; }
        const float d = amax / 127.0f;
        const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
        y[b].d = orc_f32_to_f16(d);
        for (int j = 0; j < 32; j++) y[b].qs[j] = packs8(cvt_epi32(x[b * 32 + j] * id));
    }
}

static float vec_dot_q4_0_q8_0(int n, const uint8_t * vx, const q8_0_t * y) {
    /* AVX2 branch (ggml-quants.c:4191-4214): per block acc8 = fma(d_x*d_y, (float)int-dot lanes, acc8)
     * where the 8 int lanes are sums of 4 consecutive products (maddubs + madd); final hsum_float_8. */
    float acc[8] = {0};
    const int nb = n / 32;
    for (int b = 0; b < nb; b++) {
        const uint8_t * blk = vx + (size_t) b * 18;
        uint16_t dh; memcpy(&dh, blk, 2);
        const float d = f16_lut[dh] * f16_lut[y[b].d];
        int q[32];
        for (int j = 0; j < 16; j++) { q[j] = (blk[2 + j] & 0x0f) - 8; q[j + 16] = (blk[2 + j] >> 4) - 8; }
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int k = 0; k < 4; k++) s += q[4 * l + k] * (int) y[b].qs[4 * l + k];
            acc[l] = fmaf(d, (float) s, acc[l]);
        }
    }
    /* hsum_float_8: hi128+lo128, then movehl add, then movehdup add_ss */
    float t0 = acc[4] + acc[0], t1 = acc[5] + acc[1], t2 = acc[6] + acc[2], t3 = acc[7] + acc[3];
    float s0 = t0 + t2, s1 = t1 + t3;
    return s0 + s1;
}

/* q8_1 activation blocks (quantize_row_q8_1, AVX2 branch, ggml-quants.c:1305-1345): q as q8_0, plus s = f16(d * sum(q)), where the
 * sum adds the int32 values before the packs (hsum_i32_8 of _mm256_add_epi32: wraps modulo 2^32) */
typedef struct { uint16_t d, s; int8_t qs[32]; } q8_1_t;
static void quantize_row_q8_1(const float * x, q8_1_t * y, int k) {
    for (int b = 0; b < k / 32; b++) {
        float amax = 0.0f;
        for (int j = 0; j < 32; j++) { float a = fabsf(x[b * 32 + j]); amax = a > amax ? a : amax; }
        const float d = amax / 127.0f;
        const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
        y[b].d = orc_f32_to_f16(d);
        uint32_t sum = 0;
        for (int j = 0; j < 32; j++) { const int32_t q = cvt_epi32(x[b * 32 + j] * id); y[b].qs[j] = packs8(q); sum += (uint32_t) q; }
        y[b].s = orc_f32_to_f16(d * (float)(int32_t) sum);
    }
}

static float hsum8(const float * acc) {      /* hsum_float_8 (ggml-quants.c:48-54) */
    float t0 = acc[4] + acc[0], t1 = acc[5] + acc[1], t2 = acc[6] + acc[2], t3 = acc[7] + acc[3];
    float s0 = t0 + t2, s1 = t1 + t3;
    return s0 + s1;
}
/* the 8 int32 lanes of mul_sum_*_pairs_float: lane l = sum of products 4l..4l+3 */
static void lanes8(const int * qx, const int8_t * qy, float scale, float * acc) {
    for (int l = 0; l < 8; l++) {
        int sm = 0;
        for (int k = 0; k < 4; k++) sm += qx[4 * l + k] * (int) qy[4 * l + k];
        acc[l] = fmaf(scale, (float) sm, acc[l]);
    }
}
static uint32_t rd_u32(const uint8_t * p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint16_t rd_u16(const uint8_t * p) { uint16_t v; memcpy(&v, p, 2); return v; }

/* ggml_vec_dot_q4_1_q8_1, AVX2 branch (ggml-quants.c:4635-4667); `summs += m*s` is a fused multiply-add in the pinned build */
static float vec_dot_q4_1_q8_1(int n, const uint8_t * vx, const q8_1_t * y) {
    float acc[8] = {0}, summs = 0.0f;
    for (int b = 0; b < n / 32; b++) {
        const uint8_t * blk = vx + (size_t) b * 20;
        const float d0 = f16_lut[rd_u16(blk)], d1 = f16_lut[y[b].d];
        summs = fmaf(f16_lut[rd_u16(blk + 2)], f16_lut[y[b].s], summs);
        int q[32];
        for (int j = 0; j < 16; j++) { q[j] = blk[4 + j] & 0x0f; q[j + 16] = blk[4 + j] >> 4; }
        lanes8(q, y[b].qs, d0 * d1, acc);
    }
    return hsum8(acc) + summs;
}
/* ggml_vec_dot_q5_0_q8_0, AVX2 branch (ggml-quants.c:4935-4957): code = (nibble | fifth bit << 4) - 16 */
static float vec_dot_q5_0_q8_0(int n, const uint8_t * vx, const q8_0_t * y) {
    float acc[8] = {0};
    for (int b = 0; b < n / 32; b++) {
        const uint8_t * blk = vx + (size_t) b * 22;
        const float d = f16_lut[rd_u16(blk)] * f16_lut[y[b].d];
        const uint32_t qh = rd_u32(blk + 2);
        int q[32];
        for (int j = 0; j < 16; j++) {
            q[j]      = ((blk[6 + j] & 0x0f) | (((qh >> j) & 1) << 4)) - 16;
            q[j + 16] = ((blk[6 + j] >> 4)   | (((qh >> (j + 16)) & 1) << 4)) - 16;
        }
        lanes8(q, y[b].qs, d, acc);
    }
    return hsum8(acc);
}
/* ggml_vec_dot_q5_1_q8_1, AVX2 branch (ggml-quants.c:5300-5325) */
static float vec_dot_q5_1_q8_1(int n, const uint8_t * vx, const q8_1_t * y) {
    float acc[8] = {0}, summs = 0.0f;
    for (int b = 0; b < n / 32; b++) {
        const uint8_t * blk = vx + (size_t) b * 24;
        const float dx = f16_lut[rd_u16(blk)], dy = f16_lut[y[b].d];
        summs = fmaf(f16_lut[rd_u16(blk + 2)], f16_lut[y[b].s], summs);
        const uint32_t qh = rd_u32(blk + 4);
        int q[32];
        for (int j = 0; j < 16; j++) {
            q[j]      = (blk[8 + j] & 0x0f) | (((qh >> j) & 1) << 4);
            q[j + 16] = (blk[8 + j] >> 4)   | (((qh >> (j + 16)) & 1) << 4);
        }
        lanes8(q, y[b].qs, dx * dy, acc);
    }
    return hsum8(acc) + summs;
}
/* ggml_vec_dot_q8_0_q8_0, AVX2 branch (ggml-quants.c:5747-5768) */
static float vec_dot_q8_0_q8_0(int n, const uint8_t * vx, const q8_0_t * y) {
    float acc[8] = {0};
    for (int b = 0; b < n / 32; b++) {
        const uint8_t * blk = vx + (size_t) b * 34;
        const float d = f16_lut[rd_u16(blk)] * f16_lut[y[b].d];
        int q[32];
        for (int j = 0; j < 32; j++) q[j] = (int8_t) blk[2 + j];
        lanes8(q, y[b].qs, d, acc);
    }
    return hsum8(acc);
}

/* Exported for the kernel tests (oracle/bindings.py).  The activation quantisers on k floats (k % 32 == 0) into the reference's block
 * layouts (block_q8_0: 34 bytes, block_q8_1: 36 bytes); one dot of n elements of weight blocks of wtype (enum ggml_type: 2 q4_0, 3 q4_1,
 * 6 q5_0, 7 q5_1, 8 q8_0) against the blocks of its vec_dot_type; and out[m][o] = that dot of weight row o against row m of A [M][K]
 * quantised, for W [N] rows of K/32 blocks. */
void orc_quantize_row_q8_0(const float * x, void * y, int k) { quantize_row_q8_0(x, (q8_0_t *) y, k); }
void orc_quantize_row_q8_1(const float * x, void * y, int k) { quantize_row_q8_1(x, (q8_1_t *) y, k); }
static int q_block_bytes(int wtype) { return wtype == 2 ? 18 : wtype == 3 ? 20 : wtype == 6 ? 22 : wtype == 7 ? 24 : wtype == 8 ? 34 : 0; }
float orc_vec_dot_q(int wtype, int n, const void * vx, const void * vy) {
    init_f16_lut();
    switch (wtype) {
        case 2: return vec_dot_q4_0_q8_0(n, vx, vy);
        case 3: return vec_dot_q4_1_q8_1(n, vx, vy);
        case 6: return vec_dot_q5_0_q8_0(n, vx, vy);
        case 7: return vec_dot_q5_1_q8_1(n, vx, vy);
        case 8: return vec_dot_q8_0_q8_0(n, vx, vy);
        default: return NAN;
    }
}
int orc_quant_matmul(int wtype, const void * W, const float * A, int M, int N, int K, float * out) {
    const int bb = q_block_bytes(wtype), nb = K / 32;
    if (!bb || K % 32) return 0;
    init_f16_lut();
    const int q81 = wtype == 3 || wtype == 7;
    const size_t ab = q81 ? sizeof(q8_1_t) : sizeof(q8_0_t);
    unsigned char * aq = malloc((size_t) M * nb * ab);
    for (int m = 0; m < M; m++) {
        if (q81) quantize_row_q8_1(A + (size_t) m * K, (q8_1_t *) (aq + (size_t) m * nb * ab), K);
        else     quantize_row_q8_0(A + (size_t) m * K, (q8_0_t *) (aq + (size_t) m * nb * ab), K);
    }
    #pragma omp parallel for schedule(static) collapse(2)
    for (int m = 0; m < M; m++)
        for (int o = 0; o < N; o++)
            out[(size_t) m * N + o] = orc_vec_dot_q(wtype, K, (const unsigned char *) W + (size_t) o * nb * bb, aq + (size_t) m * nb * ab);
    free(aq);
    return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* mul_mat: dst[r][o] = vec_dot(W[o][:], act[r][:]) (ggml.c:12369-12457, 12530-12558)          */
/* ------------------------------------------------------------------------------------------ */
static void mul_mat(const tensor_t * W, const float * act, int rows, float * dst, int n_out_limit) {
    const int K = W->ne[0];
    const int O = n_out_limit > 0 ? n_out_limit : W->ne[1];
    if (W->type == 0) {
        const float * w = W->data;
        #pragma omp parallel for schedule(static) collapse(2)
        for (int r = 0; r < rows; r++)
            for (int o = 0; o < O; o++) dst[(size_t) r * O + o] = orc_vec_dot_f32(K, w + (size_t) o * K, act + (size_t) r * K);
    } else if (W->type == 1) {
        uint16_t * a16 = malloc((size_t) rows * K * 2);
        for (size_t i = 0; i < (size_t) rows * K; i++) a16[i] = orc_f32_to_f16(act[i]);
        const uint16_t * w = W->data;
        #pragma omp parallel for schedule(static) collapse(2)
        for (int r = 0; r < rows; r++)
            for (int o = 0; o < O; o++) dst[(size_t) r * O + o] = orc_vec_dot_f16(K, w + (size_t) o * K, a16 + (size_t) r * K);
        free(a16);
    } else if (W->type == 2 || W->type == 6 || W->type == 8) {          /* vec_dot_type q8_0 (ggml.c type_traits) */
        const int nbk = K / 32, bb = W->type == 2 ? 18 : W->type == 6 ? 22 : 34;
        q8_0_t * a8 = malloc((size_t) rows * nbk * sizeof(q8_0_t));
        for (int r = 0; r < rows; r++) quantize_row_q8_0(act + (size_t) r * K, a8 + (size_t) r * nbk, K);
        const uint8_t * w = W->data;
        const int wt = W->type;
        #pragma omp parallel for schedule(static) collapse(2)
        for (int r = 0; r < rows; r++)
            for (int o = 0; o < O; o++) {
                const uint8_t * wr = w + (size_t) o * nbk * bb; const q8_0_t * ar = a8 + (size_t) r * nbk;
                dst[(size_t) r * O + o] = wt == 2 ? vec_dot_q4_0_q8_0(K, wr, ar) : wt == 6 ? vec_dot_q5_0_q8_0(K, wr, ar) : vec_dot_q8_0_q8_0(K, wr, ar);
            }
        free(a8);
    } else {                                                               /* q4_1, q5_1: vec_dot_type q8_1 */
        const int nbk = K / 32, bb = W->type == 3 ? 20 : 24;
        q8_1_t * a8 = malloc((size_t) rows * nbk * sizeof(q8_1_t));
        for (int r = 0; r < rows; r++) quantize_row_q8_1(act + (size_t) r * K, a8 + (size_t) r * nbk, K);
        const uint8_t * w = W->data;
        const int wt = W->type;
        #pragma omp parallel for schedule(static) collapse(2)
        for (int r = 0; r < rows; r++)
            for (int o = 0; o < O; o++) {
                const uint8_t * wr = w + (size_t) o * nbk * bb; const q8_1_t * ar = a8 + (size_t) r * nbk;
                dst[(size_t) r * O + o] = wt == 3 ? vec_dot_q4_1_q8_1(K, wr, ar) : vec_dot_q5_1_q8_1(K, wr, ar);
            }
        free(a8);
    }
}

/* get_rows into f32 (ggml.c:13455-13620) */
static void get_row(const tensor_t * T, int row, float * out) {
    const int K = T->ne[0];
    if (T->type == 0) memcpy(out, (const float *) T->data + (size_t) row * K, (size_t) K * 4);
    else if (T->type == 1) { const uint16_t * p = (const uint16_t *) T->data + (size_t) row * K; for (int i = 0; i < K; i++) out[i] = f16_lut[p[i]]; }
    else if (T->type != 2) {   /* dequantize_row_q4_1 / q5_0 / q5_1 / q8_0 (ggml-quants.c:1542-1630); x*d + m is one fused multiply-add in the pinned build */
        const int bb = T->type == 3 ? 20 : T->type == 6 ? 22 : T->type == 7 ? 24 : 34;
        const uint8_t * p = (const uint8_t *) T->data + (size_t) row * (K / 32) * bb;
        for (int b = 0; b < K / 32; b++) {
            const uint8_t * blk = p + (size_t) b * bb;
            const float d = f16_lut[rd_u16(blk)];
            float * o = out + b * 32;
            if (T->type == 8) { for (int j = 0; j < 32; j++) o[j] = (float)(int8_t) blk[2 + j] * d; continue; }
            const float m = (T->type == 3 || T->type == 7) ? f16_lut[rd_u16(blk + 2)] : 0.0f;
            const uint8_t * qs = blk + (T->type == 3 ? 4 : T->type == 6 ? 6 : 8);
            const uint32_t qh = T->type == 3 ? 0u : rd_u32(blk + (T->type == 6 ? 2 : 4));
            for (int j = 0; j < 16; j++) {
                int x0 = (qs[j] & 0x0f) | (int)(((qh >> j) & 1) << 4), x1 = (qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1) << 4);
                if (T->type == 6) { o[j] = (float)(x0 - 16) * d; o[j + 16] = (float)(x1 - 16) * d; }
                else              { o[j] = fmaf((float) x0, d, m); o[j + 16] = fmaf((float) x1, d, m); }
            }
        }
    }
    else {   /* dequantize_row_q4_0 (ggml-quants.c:1515): (nibble-8)*d */
        const uint8_t * p = (const uint8_t *) T->data + (size_t) row * (K / 32) * 18;
        for (int b = 0; b < K / 32; b++) {
            uint16_t dh; memcpy(&dh, p + b * 18, 2); const float d = f16_lut[dh];
            for (int j = 0; j < 16; j++) {
                out[b * 32 + j]      = (float)((p[b * 18 + 2 + j] & 0x0f) - 8) * d;
                out[b * 32 + j + 16] = (float)((p[b * 18 + 2 + j] >> 4) - 8) * d;
            }
        }
    }
}

static void layer_norm_rows(const float * x, float * y, int rows, int E, const tensor_t * g, const tensor_t * b) {
    #pragma omp parallel for schedule(static)
    for (int r = 0; r < rows; r++) {
        float * yr = y + (size_t) r * E;
        orc_norm(E, x + (size_t) r * E, yr, 1e-5f);
        const float * gg = g->data;
        for (int i = 0; i < E; i++) yr[i] = yr[i] * gg[i];                     /* ggml_mul */
        if (b && b->data) { const float * bb = b->data; for (int i = 0; i < E; i++) yr[i] = yr[i] + bb[i]; }
    }
}

/* attention over `n_kv` keys for `N` queries; K/V rows have stride E floats.
 * causal != 0: mask k > n_past + q (ggml_diag_mask_inf, ggml.c:13865-13915). */
static void attention(const float * Q, const float * Kc, const float * Vc, int N, int n_kv, int n_past,
                      int E, int H, int causal, float * out) {
    const int D = E / H;
    const float scale = 1.0f / sqrtf((float) E / (float) H);                   /* bark.cpp:1318 */
    #pragma omp parallel for schedule(dynamic) collapse(2)
    for (int h = 0; h < H; h++) {
        for (int q = 0; q < N; q++) {
            float * s = malloc((size_t) n_kv * 4), * p = malloc((size_t) n_kv * 4);
            const float * qv = Q + (size_t) q * E + h * D;
            for (int k = 0; k < n_kv; k++) {
                float v = orc_vec_dot_f32(D, Kc + (size_t) k * E + h * D, qv);
                v = v * scale;                                                 /* ggml_scale_inplace */
                if (causal && k > n_past + q) v = -INFINITY;
                s[k] = v;
            }
            orc_soft_max(n_kv, s, p);
            for (int d = 0; d < D; d++) out[(size_t) q * E + h * D + d] = vec_dot_f32_sx(n_kv, Vc + h * D + d, E, p);
            free(s); free(p);
        }
    }
}

/* transformer body shared by the causal and fine graphs.  x: [N][E] in/out. */
static void gpt_body(gpt_t * m, float * x, int N, int n_past, int causal) {
    const int E = m->n_embd, H = m->n_head;
    float * cur = malloc((size_t) N * E * 4), * qkv = malloc((size_t) N * 3 * E * 4), * att = malloc((size_t) N * E * 4);
    float * ff = malloc((size_t) N * 4 * E * 4), * tmp = malloc((size_t) N * E * 4);
    float * kbuf = NULL, * vbuf = NULL;
    if (!causal) { kbuf = malloc((size_t) N * E * 4); vbuf = malloc((size_t) N * E * 4); }
    for (int il = 0; il < m->n_layer; il++) {
        layer_norm_rows(x, cur, N, E, &m->layers[il].ln_1_g, m->bias ? &m->layers[il].ln_1_b : NULL);
        mul_mat(&m->layers[il].c_attn, cur, N, qkv, 0);
        const float * Kc, * Vc; int n_kv;
        if (causal) {                                                          /* bark.cpp:1294-1300 */
            float * mk = m->mem_k + ((size_t) il * m->block_size + n_past) * E;
            float * mv = m->mem_v + ((size_t) il * m->block_size + n_past) * E;
            for (int r = 0; r < N; r++) { memcpy(mk + (size_t) r * E, qkv + (size_t) r * 3 * E + E, (size_t) E * 4);
                                          memcpy(mv + (size_t) r * E, qkv + (size_t) r * 3 * E + 2 * E, (size_t) E * 4); }
            Kc = m->mem_k + (size_t) il * m->block_size * E; Vc = m->mem_v + (size_t) il * m->block_size * E; n_kv = n_past + N;
        } else {
            for (int r = 0; r < N; r++) { memcpy(kbuf + (size_t) r * E, qkv + (size_t) r * 3 * E + E, (size_t) E * 4);
                                          memcpy(vbuf + (size_t) r * E, qkv + (size_t) r * 3 * E + 2 * E, (size_t) E * 4); }
            Kc = kbuf; Vc = vbuf; n_kv = N;
        }
        for (int r = 0; r < N; r++) memcpy(tmp + (size_t) r * E, qkv + (size_t) r * 3 * E, (size_t) E * 4);   /* Q */
        attention(tmp, Kc, Vc, N, n_kv, n_past, E, H, causal, att);
        mul_mat(&m->layers[il].c_proj, att, N, cur, 0);
        for (size_t i = 0; i < (size_t) N * E; i++) x[i] = cur[i] + x[i];      /* inpFF = cur + inpL */
        layer_norm_rows(x, cur, N, E, &m->layers[il].ln_2_g, m->bias ? &m->layers[il].ln_2_b : NULL);
        mul_mat(&m->layers[il].fc, cur, N, ff, 0);
        for (size_t i = 0; i < (size_t) N * 4 * E; i++) ff[i] = gelu_f32(ff[i]);
        mul_mat(&m->layers[il].proj, ff, N, cur, 0);
        for (size_t i = 0; i < (size_t) N * E; i++) x[i] = cur[i] + x[i];      /* inpL = cur + inpFF */
    }
    free(cur); free(qkv); free(att); free(ff); free(tmp); free(kbuf); free(vbuf);
}

int orc_gpt_eval(orc_ctx * c, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits) {
    gpt_t * m = &c->gpt[which];
    const int E = m->n_embd;
    int N = n;
    float * x;
    merge_ctx = merge_ctx && *n_past == 0;                                     /* bark.cpp:1230: the merged prompt only exists at n_past == 0 */
    if (*n_past + (merge_ctx ? 257 : N) > m->block_size) return 0;
    if (merge_ctx) {                                                    /* bark.cpp:1230-1248 */
        if (N != 513) return 0;
        N = 257;
        x = malloc((size_t) N * E * 4);
        float * a = malloc((size_t) E * 4), * b = malloc((size_t) E * 4);
        for (int i = 0; i < 256; i++) {
            get_row(&m->wte[0], tokens[i], a); get_row(&m->wte[0], tokens[256 + i], b);
            for (int k = 0; k < E; k++) x[(size_t) i * E + k] = a[k] + b[k];
        }
        get_row(&m->wte[0], tokens[512], x + (size_t) 256 * E);
        free(a); free(b);
    } else {
        if (N > m->block_size) return 0;
        x = malloc((size_t) N * E * 4);
        for (int i = 0; i < N; i++) get_row(&m->wte[0], tokens[i], x + (size_t) i * E);
    }
    const float * wpe = m->wpe.data;
    for (int i = 0; i < N; i++) for (int k = 0; k < E; k++) x[(size_t) i * E + k] = x[(size_t) i * E + k] + wpe[(size_t)(i + *n_past) * E + k];
    gpt_body(m, x, N, *n_past, 1);
    float * last = malloc((size_t) E * 4);
    layer_norm_rows(x + (size_t)(N - 1) * E, last, 1, E, &m->ln_f_g, m->bias ? &m->ln_f_b : NULL);
    mul_mat(&m->lm_head[0], last, 1, logits, 0);
    free(last); free(x);
    *n_past += N;
    return 1;
}

int orc_fine_eval(orc_ctx * c, const int32_t * in, int nn, float * logits) {
    gpt_t * m = &c->gpt[2];
    const int E = m->n_embd, N = 1024;
    float * x = calloc((size_t) N * E, 4), * row = malloc((size_t) E * 4);
    for (int w = 0; w <= nn; w++)                                              /* bark.cpp:1457-1463 */
        for (int i = 0; i < N; i++) { get_row(&m->wte[w], in[w * 1024 + i], row); for (int k = 0; k < E; k++) x[(size_t) i * E + k] = x[(size_t) i * E + k] + row[k]; }
    const float * wpe = m->wpe.data;
    for (size_t i = 0; i < (size_t) N * E; i++) x[i] = x[i] + wpe[i];
    gpt_body(m, x, N, 0, 0);
    float * fin = malloc((size_t) N * E * 4);
    layer_norm_rows(x, fin, N, E, &m->ln_f_g, &m->ln_f_b);
    mul_mat(&m->lm_head[nn - 1], fin, N, logits, 0);                           /* n_codes_given = 1, bark.cpp:1573 */
    free(fin); free(row); free(x);
    return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* sampling (bark.cpp:184-270)                                                                 */
/* ------------------------------------------------------------------------------------------ */
/* gpt_sample with the uniform draw u already made (u is not used when temp == 0) */
int orc_sample_u(const float * logits_in, int n, float temp, double u, float * eos_p) {
    float * l = malloc((size_t) n * 4);
    const float t = (temp == 0.0f) ? 0.7f : temp;                              /* bark.cpp:226-228 quirk */
    for (int i = 0; i < n; i++) l[i] = logits_in[i] / t;
    float maxl = -INFINITY;
    for (int i = 0; i < n; i++) maxl = l[i] > maxl ? l[i] : maxl;
    float sum = 0.0f;
    for (int i = 0; i < n; i++) { l[i] = (float) exp((double)(l[i] - maxl)); sum += l[i]; }   /* `exp` resolves to the double overload */
    for (int i = 0; i < n; i++) l[i] = l[i] / sum;
    int next = 0;
    if (temp == 0.0f) {
        float mx = -INFINITY;
        for (int i = 0; i < n; i++) if (l[i] > mx) { mx = l[i]; next = i; }
    } else {
        double s = 0.0;
        for (int i = 0; i < n; i++) s += (double) l[i];
        double * cp = malloc((size_t) n * 8);
        double run = 0.0;
        for (int i = 0; i < n; i++) { double p = (double) l[i] / s; run = (i == 0) ? p : run + p; cp[i] = run; }
        cp[n - 1] = 1.0;
        int lo = 0, hi = n;                                                    /* lower_bound: first cp[i] >= u */
        while (lo < hi) { int mid = lo + (hi - lo) / 2; if (cp[mid] < u) lo = mid + 1; else hi = mid; }
        next = lo;
        free(cp);
    }
    if (eos_p) *eos_p = l[n - 1];
    free(l);
    return next;
}
int orc_sample(orc_ctx * c, const float * logits_in, int n, float temp, float * eos_p) {
    return orc_sample_u(logits_in, n, temp, temp == 0.0f ? 0.0 : mt_canonical(c->rng), eos_p);   /* one draw per sample, none for argmax */
}

/* ------------------------------------------------------------------------------------------ */
/* tokenizer (bark.cpp:480-662)                                                                */
/* ------------------------------------------------------------------------------------------ */
static int vocab_find(orc_ctx * c, const char * s) {
    /* std::map insert semantics: duplicates keep the LAST id (token_to_id[word] = i, bark.cpp:685) */
    for (int i = c->n_vocab - 1; i >= 0; i--) if (!strcmp(c->vocab[i], s)) return i;
    return -1;
}

static const struct { const char * utf8; char ascii; } ACCENTS[] = {
    {"\xc3\x80",'A'},{"\xc3\x81",'A'},{"\xc3\x82",'A'},{"\xc3\x83",'A'},{"\xc3\x84",'A'},{"\xc3\x85",'A'},
    {"\xc3\xa0",'a'},{"\xc3\xa1",'a'},{"\xc3\xa2",'a'},{"\xc3\xa3",'a'},{"\xc3\xa4",'a'},{"\xc3\xa5",'a'},
    {"\xc3\x88",'E'},{"\xc3\x89",'E'},{"\xc3\x8a",'E'},{"\xc3\x8b",'E'},{"\xc3\xa8",'e'},{"\xc3\xa9",'e'},{"\xc3\xaa",'e'},{"\xc3\xab",'e'},
    {"\xc3\x8c",'I'},{"\xc3\x8d",'I'},{"\xc3\x8e",'I'},{"\xc3\x8f",'I'},{"\xc3\xac",'i'},{"\xc3\xad",'i'},{"\xc3\xae",'i'},{"\xc3\xaf",'i'},
    {"\xc3\x92",'O'},{"\xc3\x93",'O'},{"\xc3\x94",'O'},{"\xc3\x95",'O'},{"\xc3\x96",'O'},{"\xc3\xb2",'o'},{"\xc3\xb3",'o'},{"\xc3\xb4",'o'},{"\xc3\xb5",'o'},{"\xc3\xb6",'o'},
    {"\xc3\x99",'U'},{"\xc3\x9a",'U'},{"\xc3\x9b",'U'},{"\xc3\x9c",'U'},{"\xc3\xb9",'u'},{"\xc3\xba",'u'},{"\xc3\xbb",'u'},{"\xc3\xbc",'u'},
    {"\xc3\x9d",'Y'},{"\xc3\xbd",'y'},{"\xc3\x87",'C'},{"\xc3\xa7",'c'},{"\xc3\x91",'N'},{"\xc3\xb1",'n'},
};

void orc_tokenize(orc_ctx * c, const char * text, int32_t * out) {
    /* strip_accents (bark.cpp:486-556) */
    size_t L = strlen(text);
    char * s = malloc(L + 1); size_t o = 0;
    for (size_t i = 0; i < L;) {
        static const int lookup[16] = {1,1,1,1,1,1,1,1,1,1,1,1,2,2,3,4};
        int len = lookup[((unsigned char) text[i]) >> 4];
        if ((size_t) len > L - i) len = (int)(L - i);
        int hit = 0;
        if (len == 2) for (size_t a = 0; a < sizeof(ACCENTS) / sizeof(ACCENTS[0]); a++)
            if (!memcmp(text + i, ACCENTS[a].utf8, 2)) { s[o++] = ACCENTS[a].ascii; hit = 1; break; }
        if (!hit) { memcpy(s + o, text + i, len); o += len; }
        i += len;
    }
    s[o] = 0;
    /* word split: [[:punct:]]|[[:alpha:]]+|[[:digit:]]+ in the classic locale (bark.cpp:575-584), then
     * greedy longest-match WordPiece (bark.cpp:588-617) */
    int32_t toks[256]; int t = 0; const int n_max = 256;
    size_t i = 0;
    while (i < o) {
        unsigned char ch = (unsigned char) s[i];
        size_t j = i;
        if (ch < 128 && ispunct(ch)) j = i + 1;
        else if (ch < 128 && isalpha(ch)) { while (j < o && (unsigned char) s[j] < 128 && isalpha((unsigned char) s[j])) j++; }
        else if (ch < 128 && isdigit(ch)) { while (j < o && (unsigned char) s[j] < 128 && isdigit((unsigned char) s[j])) j++; }
        else { i++; continue; }
        /* wordpiece on s[i..j) */
        int n = (int)(j - i), p = 0; const char * prefix = "";
        while (p < n) {
            if (t >= n_max - 1) break;
            int e = n, found = 0;
            while (e > p) {
                char buf[600]; snprintf(buf, sizeof buf, "%s%.*s", prefix, e - p, s + i + p);
                int id = vocab_find(c, buf);
                if (id >= 0) { toks[t++] = id; p = e; prefix = "##"; found = 1; break; }
                e--;
            }
            if (!found) { prefix = "##"; p++; }
        }
        i = j;
    }
    free(s);
    /* bark_tokenize_input (bark.cpp:622-662): +10048 on all 256 slots (unset slots are 0), then pad */
    for (int k = 0; k < 256; k++) out[k] = (k < t ? toks[k] : 0) + 10048;
    for (int k = t; k < 256; k++) out[k] = 129595;
    for (int k = 0; k < 256; k++) out[256 + k] = 10000;
    out[512] = 129599;
}

/* ------------------------------------------------------------------------------------------ */
/* stage loops                                                                                 */
/* ------------------------------------------------------------------------------------------ */
int orc_semantic(orc_ctx * c, const int32_t * prompt, int32_t * out) {       /* bark.cpp:1645-1701 */
    gpt_t * m = &c->gpt[0];
    float * logits = malloc((size_t) m->n_out_vocab * 4);
    int n_past = 0, n_out = 0; float eos_p = 0;
    int32_t in[513]; int n_in = 513; memcpy(in, prompt, sizeof in);
    for (int i = 0; i < c->n_steps_text_encoder; i++) {
        orc_gpt_eval(c, 0, in, n_in, &n_past, 1, logits);
        int next = orc_sample(c, logits, m->n_out_vocab, c->temp, &eos_p);  /* all logits: quirk D.1 */
        if (next == 10000 || eos_p >= c->min_eos_p) break;
        in[0] = next; n_in = 1; out[n_out++] = next;
    }
    free(logits);
    return n_out;
}

int orc_coarse(orc_ctx * c, const int32_t * sem, int n_sem, int32_t * out_Tx2) {   /* bark.cpp:1745-1863 */
    gpt_t * m = &c->gpt[1];
    float * logits = malloc((size_t) m->n_out_vocab * 4);
    const int max_coarse_history = 630, sliding_window_size = 60, n_cb = 2, sem_vocab = 10000, cb_size = 1024;
    const float stc_ratio = 75.0f / 49.9f * (float) n_cb;
    const int max_semantic_history = (int) floorf((float) max_coarse_history / stc_ratio);
    const int n_steps = (int)(floorf((float) n_sem * stc_ratio / (float) n_cb) * (float) n_cb);
    const int n_window_steps = (int) ceilf((float) n_steps / (float) sliding_window_size);
    int32_t * out = malloc((size_t)(n_steps + 1) * 4); int n_out = 0;
    int32_t * in = malloc(2048 * 4);
    int step_idx = 0;
    for (int w = 0; w < n_window_steps; w++) {
        const int semantic_idx = (int) roundf((float) step_idx / stc_ratio);
        int start = semantic_idx - max_semantic_history; if (start < 0) start = 0;
        int n_in = 0;
        for (int k = start; k < n_sem && n_in < 256; k++) in[n_in++] = sem[k];
        while (n_in < 256) in[n_in++] = 12048;
        in[n_in++] = 12050;
        int hist = n_out < max_coarse_history ? n_out : max_coarse_history;
        for (int k = n_out - hist; k < n_out; k++) in[n_in++] = out[k];
        int n_past = 0;
        for (int j = 0; j < sliding_window_size; j++) {
            if (step_idx >= n_steps) continue;
            orc_gpt_eval(c, 1, in, n_in, &n_past, 0, logits);
            const int is_major = step_idx % n_cb == 0;
            const int start_idx = sem_vocab + (1 - is_major) * cb_size;
            int next = orc_sample(c, logits + start_idx, cb_size, c->temp, NULL) + start_idx;
            in[0] = next; n_in = 1; out[n_out++] = next; step_idx++;
        }
    }
    for (int i = 0; i < n_out; i += 2) { out_Tx2[i] = out[i] - sem_vocab; out_Tx2[i + 1] = out[i + 1] - sem_vocab - cb_size; }
    free(out); free(in); free(logits);
    return n_out / 2;
}

int orc_fine(orc_ctx * c, const int32_t * coarse, int T, int32_t * out_Tx8) {       /* bark.cpp:1961-2059 */
    assert(T <= 1024);                     /* beyond that the reference writes out of bounds (bark.cpp:2037) */
    gpt_t * m = &c->gpt[2];
    const int V = m->n_out_vocab;
    float * logits = malloc((size_t) 1024 * V * 4);
    int32_t * in = malloc(8 * 1024 * 4);
    for (int cb = 0; cb < 8; cb++) for (int t = 0; t < 1024; t++) in[cb * 1024 + t] = (cb < 2 && t < T) ? coarse[t * 2 + cb] : 1024;
    for (int nn = 2; nn < 8; nn++) {
        orc_fine_eval(c, in, nn, logits);
        for (int i = 0; i < 1024; i++) in[nn * 1024 + i] = orc_sample(c, logits + (size_t) i * V, 1024, c->fine_temp, NULL);
    }
    for (int t = 0; t < T; t++) for (int cb = 0; cb < 8; cb++) out_Tx8[t * 8 + cb] = in[cb * 1024 + t];
    free(in); free(logits);
    return T;
}

/* ------------------------------------------------------------------------------------------ */
/* EnCodec decoder.  Activations are [C][T] (channel-major, time contiguous) like the          */
/* reference's [T, C] ggml tensors.                                                            */
/* ------------------------------------------------------------------------------------------ */
static void elu_inplace(float * x, size_t n) { for (size_t i = 0; i < n; i++) x[i] = (x[i] > 0.f) ? x[i] : expm1f(x[i]); }

/* strided_conv_1d, stride 1 (ops.cpp:59-75): reflect-pad left by k-1, im2col to f16 (ggml.c:14954),
 * f16 x f16 vec_dot over [Cin][k], bias added in f32 */
/* ggml_conv_1d core (ggml.c:6641-6660 = im2col to f16 + mul_mat): xp is the already padded f16 input [Cin][Tp], T = Tp - k + 1 outputs */
static void conv1d_core(const uint16_t * xp, int Cin, int Tp, int k, const uint16_t * w, int Cout, const float * bias, float * y) {
    const int T = Tp - k + 1;
    #pragma omp parallel
    {
        uint16_t * col = malloc((size_t) Cin * k * 2);
        #pragma omp for schedule(static)
        for (int t = 0; t < T; t++) {
            for (int c = 0; c < Cin; c++) for (int j = 0; j < k; j++) col[c * k + j] = xp[(size_t) c * Tp + t + j];
            for (int o = 0; o < Cout; o++) {
                float v = orc_vec_dot_f16(Cin * k, col, w + (size_t) o * Cin * k);
                y[(size_t) o * T + t] = bias ? bias[o] + v : v;                  /* ops.cpp:72 add(repeat(b), dst) */
            }
        }
        free(col);
    }
}
static float * conv1d(const float * x, int Cin, int T, const conv_t * cv) {
    const int k = cv->w.ne[0], Cout = cv->w.ne[2], pad = k - 1;
    assert(cv->w.ne[1] == Cin && T > pad);
    uint16_t * xp = malloc((size_t) Cin * (T + pad) * 2);           /* padded, f16 */
    for (int c = 0; c < Cin; c++) {
        uint16_t * row = xp + (size_t) c * (T + pad);
        for (int t = 0; t < T; t++) row[pad + t] = orc_f32_to_f16(x[(size_t) c * T + t]);
        for (int i = 1; i <= pad; i++) row[pad - i] = row[pad + i];            /* ggml.c:15589 */
    }
    float * y = malloc((size_t) Cout * T * 4);
    conv1d_core(xp, Cin, T + pad, k, cv->w.data, Cout, cv->b.data, y);
    free(xp);
    return y;
}

/* strided_conv_transpose_1d (ops.cpp:77-98, ggml.c:14614-14700): kernel [k][Cout][Cin] f16 */
/* ggml_conv_transpose_1d core (ggml.c:14614-14700): full-length output [(T-1)*stride + k] per channel, kernel [Cin][Cout][k] f16 */
static float * convtr1d_full(const float * x, int Cin, int T, const uint16_t * w, int k, int Cout, int stride) {
    const int Lfull = (T - 1) * stride + k;
    uint16_t * xs = malloc((size_t) T * Cin * 2);                   /* [T][Cin] f16 */
    for (int c = 0; c < Cin; c++) for (int t = 0; t < T; t++) xs[(size_t) t * Cin + c] = orc_f32_to_f16(x[(size_t) c * T + t]);
    float * full = calloc((size_t) Cout * Lfull, 4);
    #pragma omp parallel
    {
        uint16_t * wk = malloc((size_t) k * Cin * 2);
        #pragma omp for schedule(static)
        for (int o = 0; o < Cout; o++) {
            for (int ci = 0; ci < Cin; ci++) for (int j = 0; j < k; j++) wk[(size_t) j * Cin + ci] = w[((size_t) ci * Cout + o) * k + j];
            for (int t = 0; t < T; t++) for (int j = 0; j < k; j++) {
                float v = orc_vec_dot_f16(Cin, xs + (size_t) t * Cin, wk + (size_t) j * Cin);
                full[(size_t) o * Lfull + t * stride + j] += v;
            }
        }
        free(wk);
    }
    free(xs);
    return full;
}
static float * convtr1d(const float * x, int Cin, int T, const conv_t * cv, int stride, int * T_out) {
    const int k = cv->w.ne[0], Cout = cv->w.ne[1];
    assert(cv->w.ne[2] == Cin);
    const float * bias = cv->b.data;
    const int Lfull = (T - 1) * stride + k;
    float * full = convtr1d_full(x, Cin, T, cv->w.data, k, Cout, stride);
    const int L = Lfull - (k - stride);                             /* unpad right (ops.cpp:89-95) */
    float * y = malloc((size_t) Cout * L * 4);
    for (int o = 0; o < Cout; o++) for (int t = 0; t < L; t++) y[(size_t) o * L + t] = bias[o] + full[(size_t) o * Lfull + t];
    free(full);
    *T_out = L;
    return y;
}

/* Test hooks for the known-answer vectors of the reference's own op tests (ggml/tests/test-conv1d.cpp:233-281,
 * test-conv-transpose-1d.cpp:415-560).  Kernels arrive as f32 and are rounded to f16 like the codec's weights; the vectors are
 * small integers / halves, exact in f16.  conv1d: ggml_conv_1d(a, b, s0 = 1, p0, d0 = 1), zero padding p0 on both sides. */
void orc_test_conv1d(const float * w, int k, int Cin, int Cout, const float * x, int T, int p0, float * y /*[Cout][T + 2 p0 - k + 1]*/) {
    const int Tp = T + 2 * p0;
    uint16_t * w16 = malloc((size_t) k * Cin * Cout * 2), * xp = calloc((size_t) Cin * Tp, 2);
    for (int i = 0; i < k * Cin * Cout; i++) w16[i] = orc_f32_to_f16(w[i]);
    for (int c = 0; c < Cin; c++) for (int t = 0; t < T; t++) xp[(size_t) c * Tp + p0 + t] = orc_f32_to_f16(x[(size_t) c * T + t]);
    conv1d_core(xp, Cin, Tp, k, w16, Cout, NULL, y);
    free(w16); free(xp);
}
void orc_test_convtr1d(const float * w /*[Cin][Cout][k]*/, int k, int Cout, int Cin, const float * x /*[Cin][T]*/, int T, int stride, float * y /*[Cout][(T-1)*stride + k]*/) {
    uint16_t * w16 = malloc((size_t) k * Cin * Cout * 2);
    for (int i = 0; i < k * Cin * Cout; i++) w16[i] = orc_f32_to_f16(w[i]);
    float * full = convtr1d_full(x, Cin, T, w16, k, Cout, stride);
    memcpy(y, full, (size_t) Cout * ((T - 1) * stride + k) * 4);
    free(full); free(w16);
}

/* forward_pass_lstm_unilayer (lstm.h:22-78).  x: [C][T] -> returns [H][T] */
static float * lstm_layer(const float * x, int C, int T, const tensor_t * wih, const tensor_t * whh, const tensor_t * bih, const tensor_t * bhh) {
    const int H = wih->ne[1] / 4;
    float * hs = malloc((size_t) H * T * 4);
    float * h = calloc(H, 4), * cst = calloc(H, 4), * xt = malloc((size_t) C * 4);
    float * gi = malloc((size_t) 4 * H * 4), * gh = malloc((size_t) 4 * H * 4);
    const float * bi = bih->data, * bh = bhh->data;
    for (int t = 0; t < T; t++) {
        for (int c = 0; c < C; c++) xt[c] = x[(size_t) c * T + t];
        mul_mat(wih, xt, 1, gi, 0);
        mul_mat(whh, h, 1, gh, 0);
        for (int g = 0; g < 4 * H; g++) { float a = gi[g] + bi[g]; float b = gh[g] + bh[g]; gi[g] = a + b; }
        for (int j = 0; j < H; j++) {
            float it = 1.f / (1.f + expf(-gi[j]));
            float ft = 1.f / (1.f + expf(-gi[H + j]));
            float gt = tanhf(gi[2 * H + j]);
            float ot = 1.f / (1.f + expf(-gi[3 * H + j]));
            float a = ft * cst[j]; float b = it * gt;
            cst[j] = a + b;
            h[j] = ot * tanhf(cst[j]);
            hs[(size_t) j * T + t] = h[j];
        }
    }
    free(h); free(cst); free(xt); free(gi); free(gh);
    return hs;
}

/* quantizer decode (quantizer.h:78-111): zero-initialised accumulator, q = 0..n_q-1 in order; cb[q] [n_bins][Hd], codes [n_q][T] */
static void quantizer_decode(const int32_t * codes, int n_q, int T, const float * const * cb, int Hd, float * x) {
    memset(x, 0, (size_t) Hd * T * 4);
    for (int q = 0; q < n_q; q++)
        for (int t = 0; t < T; t++) for (int d = 0; d < Hd; d++) x[(size_t) d * T + t] = x[(size_t) d * T + t] + cb[q][(size_t) codes[q * T + t] * Hd + d];
}

int orc_encodec_decode(orc_ctx * c, const int32_t * codes, int T, float * out) {
    codec_t * cd = &c->codec;
    const int Hd = cd->hidden_dim;
    static const int ratios[4] = {8, 5, 4, 2};
    const float * cb[8];
    for (int q = 0; q < 8; q++) cb[q] = cd->embed[q].data;
    float * x = malloc((size_t) Hd * T * 4);
    quantizer_decode(codes, 8, T, cb, Hd, x);
    float * y = conv1d(x, Hd, T, &cd->init); free(x);
    int C = cd->init.w.ne[2];
    float * h1 = lstm_layer(y, C, T, &cd->lstm_ih_w[0], &cd->lstm_hh_w[0], &cd->lstm_ih_b[0], &cd->lstm_hh_b[0]);
    float * h2 = lstm_layer(h1, C, T, &cd->lstm_ih_w[1], &cd->lstm_hh_w[1], &cd->lstm_ih_b[1], &cd->lstm_hh_b[1]);
    for (size_t i = 0; i < (size_t) C * T; i++) y[i] = y[i] + h2[i];           /* decoder.h:72 */
    free(h1); free(h2);
    int L = T;
    for (int b = 0; b < 4; b++) {
        elu_inplace(y, (size_t) C * L);
        int L2; float * u = convtr1d(y, C, L, &cd->blk[b].us, ratios[b], &L2); free(y);
        C /= 2; L = L2;
        float * sc = conv1d(u, C, L, &cd->blk[b].sc);
        elu_inplace(u, (size_t) C * L);
        float * r1 = conv1d(u, C, L, &cd->blk[b].c1); free(u);
        elu_inplace(r1, (size_t)(C / 2) * L);
        float * r2 = conv1d(r1, C / 2, L, &cd->blk[b].c2); free(r1);
        for (size_t i = 0; i < (size_t) C * L; i++) r2[i] = r2[i] + sc[i];     /* decoder.h:101 */
        free(sc); y = r2;
    }
    elu_inplace(y, (size_t) C * L);
    float * wav = conv1d(y, C, L, &cd->final); free(y);
    memcpy(out, wav, (size_t) L * 4); free(wav);
    return L;
}

int orc_generate(orc_ctx * c, const char * text, int32_t * semantic, int * n_semantic, int32_t * coarse, int32_t * fine,
                 int * n_frames, float * audio) {
    int32_t prompt[513];
    orc_tokenize(c, text, prompt);
    /* 1024 semantic ids make at most 1539 coarse frames (orc_coarse) */
    int32_t * sem = malloc(1024 * 4), * co = malloc(2 * 2048 * 4), * fi = malloc(8 * 1024 * 4), * codes = malloc(8 * 1024 * 4);
    int ns = orc_semantic(c, prompt, sem);
    int T = orc_coarse(c, sem, ns, co);
    if (T > 1024) {                        /* the reference's fine stage writes out of bounds there (orc_fine) */
        free(sem); free(co); free(fi); free(codes);
        return -1;
    }
    orc_fine(c, co, T, fi);
    for (int cb = 0; cb < 8; cb++) for (int t = 0; t < T; t++) codes[cb * T + t] = fi[t * 8 + cb];   /* bark.cpp:2151-2159 */
    int n = orc_encodec_decode(c, codes, T, audio);
    if (semantic) memcpy(semantic, sem, (size_t) ns * 4);
    if (coarse) memcpy(coarse, co, (size_t) T * 2 * 4);
    if (fine) memcpy(fine, fi, (size_t) T * 8 * 4);
    if (n_semantic) *n_semantic = ns;
    if (n_frames) *n_frames = T;
    free(sem); free(co); free(fi); free(codes);
    return n;
}
