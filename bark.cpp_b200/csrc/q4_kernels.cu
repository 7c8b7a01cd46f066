// q4_0 GPT weights (BASELINE configs[3]): the reference's quantised mul_mat, bit for bit.
//
// ggml turns the f32 activation row into q8_0 blocks (quantize_row_q8_0, AVX2 flavour, ggml-quants.c:944-1000: d = amax/127,
// q = round-to-nearest-even(x * (127/amax)), d kept as f16) and calls ggml_vec_dot_q4_0_q8_0 (AVX2 flavour,
// ggml-quants.c:4191-4214): per 32-element block EIGHT int32 lanes, lane l = sum of products 4l..4l+3, folded into eight
// float accumulators with one fused multiply-add by d_w * d_a, then hsum_float_8.  Eight CUDA lanes own those eight
// accumulators of one output (a warp = 4 outputs): each takes one 32-bit word of nibbles and one of int8 activations per
// block, one dp4a, one fma; the final tree is three xor-shuffles (4, 2, 1).  oracle/bark_oracle.c vec_dot_q4_0_q8_0 is the
// executable spec, pinned against the reference in tests/test_quantize.py.
//
// Layout: the 18-byte blocks of the file are split at load into qs [n_out][K/32] x 16 B (aligned 16-byte words) and
// scales [n_out][K/32] f16.  Activations arrive as f32 rows (store_act, W_Q4_0) and are quantised by quantize_q8_kernel into
// int8 [rows][K] + f32 scales [rows][K/32] (the f16-rounded d, widened back).
#include "epilogue.cuh"
#include "gpt_kernels.h"

namespace bark {

namespace {

// one thread per block: file layout {f16 d; u8 qs[16]} (18 B, unaligned) -> separate aligned arrays
__global__ void split_q4_kernel(const unsigned char * __restrict__ raw, size_t n_blocks, uint4 * __restrict__ qs, __half * __restrict__ scales) {
    const size_t b = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const unsigned char * p = raw + b * 18;
    scales[b] = __ushort_as_half((unsigned short)(p[0] | (p[1] << 8)));
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) w[i] = (uint32_t) p[2 + 4 * i] | ((uint32_t) p[3 + 4 * i] << 8) | ((uint32_t) p[4 + 4 * i] << 16) | ((uint32_t) p[5 + 4 * i] << 24);
    qs[b] = make_uint4(w[0], w[1], w[2], w[3]);
}

// one warp per (row, block), lane j = element j.  A non-finite product (a block holding an inf, or 0 < amax < 127 / FLT_MAX where
// id = 127 / amax overflows) becomes -128: cvtps_epi32 turns it into INT_MIN and the saturating packs into -128.
__global__ void quantize_q8_kernel(const float * __restrict__ x, int ldx, int rows, int K, int8_t * __restrict__ q, float * __restrict__ d_out) {
    const int nb = K >> 5;
    const size_t w = ((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= (size_t) rows * nb) return;
    const int r = (int)(w / nb), b = (int)(w % nb);
    const float v = x[(size_t) r * ldx + b * 32 + lane];
    float amax = fabsf(v);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = __fdiv_rn(amax, 127.0f);
    const float id = amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f;
    const float p = __fmul_rn(v, id);
    q[(size_t) r * K + b * 32 + lane] = (int8_t)(isfinite(p) ? __float2int_rn(p) : -128);   // _mm256_round_ps(nearest) + cvtps_epi32 + packs
    if (lane == 0) d_out[(size_t) r * nb + b] = __half2float(__float2half_rn(d));          // y[i].d = GGML_FP32_TO_FP16(d)
}

// out[m][o] = vec_dot_q4_0_q8_0(W[o], A[m]).  Eight lanes own the eight float accumulators of one output; an 8-lane group walks OPW
// outputs against MT activation rows (MT x OPW accumulators per lane), so one load of an activation word serves OPW outputs: with
// one output per group the kernel was bound by the activation-load instructions (37 M per fc pass).  MT = 8, OPW = 4 for the
// multi-row passes (warp = 16 outputs x 8 rows, block = 128 outputs); MT = 1, OPW = 1 for a single decode row.
template <int kQ4MT, int OPW>
__global__ void __launch_bounds__(256) q4_matmul_kernel(const uint4 * __restrict__ qs, const __half * __restrict__ scales, int K, int O,
                                                        const int8_t * __restrict__ aq, const float * __restrict__ ad, int M, MatmulEpilogue ep) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int l = lane & 7, grp = lane >> 3;
    const int o0 = ((blockIdx.x * 8 + warp) * 4 + grp) * OPW;      // first output of this 8-lane group
    const int m0 = blockIdx.y * kQ4MT;
    const int nb = K >> 5;
    const bool high = l >= 4;                                     // lanes 4..7: elements 16..31 = high nibbles of the same bytes
    const uint32_t * wq[OPW]; const __half * ws[OPW];
#pragma unroll
    for (int oo = 0; oo < OPW; oo++) {
        const int oc = min(o0 + oo, O - 1);                       // keep every lane in the shuffles; out-of-range outputs are not stored
        wq[oo] = reinterpret_cast<const uint32_t *>(qs + (size_t) oc * nb) + (l & 3); ws[oo] = scales + (size_t) oc * nb;
    }
    float acc[OPW][kQ4MT];
#pragma unroll
    for (int oo = 0; oo < OPW; oo++)
#pragma unroll
        for (int mi = 0; mi < kQ4MT; mi++) acc[oo][mi] = 0.0f;
    for (int b = 0; b < nb; b++) {
        int yi[kQ4MT]; float da[kQ4MT];
#pragma unroll
        for (int mi = 0; mi < kQ4MT; mi++) {
            const int m = min(m0 + mi, M - 1);
            yi[mi] = __ldg(reinterpret_cast<const int *>(aq + (size_t) m * K + b * 32) + l);
            da[mi] = __ldg(ad + (size_t) m * nb + b);
        }
#pragma unroll
        for (int oo = 0; oo < OPW; oo++) {
            uint32_t w = __ldg(wq[oo] + (size_t) b * 4);
            w = (high ? (w >> 4) : w) & 0x0f0f0f0fu;
            const int wi = (int) __vsub4(w, 0x08080808u);         // nibble - 8 per byte
            const float dw = __half2float(__ldg(ws[oo] + b));
#pragma unroll
            for (int mi = 0; mi < kQ4MT; mi++) acc[oo][mi] = __fmaf_rn(__fmul_rn(dw, da[mi]), (float) __dp4a(wi, yi[mi], 0), acc[oo][mi]);
        }
    }
#pragma unroll
    for (int oo = 0; oo < OPW; oo++)
#pragma unroll
        for (int mi = 0; mi < kQ4MT; mi++) {
            float t = acc[oo][mi];                                // hsum_float_8 (ggml-quants.c:48-54)
            t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 4));
            t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 2));
            t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 1));
            if (l == 0 && o0 + oo < O && m0 + mi < M) matmul_epilogue(ep, m0 + mi, o0 + oo, t);
        }
}

thread_local int8_t * g_q8 = nullptr; thread_local float * g_q8d = nullptr;   // per host thread: one thread drives one context

}  // namespace

void q4_split(const void * raw_blocks, size_t n_blocks, void * qs, void * scales, cudaStream_t s) {
    BARK_LAUNCH(split_q4_kernel, (unsigned)((n_blocks + 255) / 256), 256, 0, s, (const unsigned char *) raw_blocks, n_blocks, (uint4 *) qs, (__half *) scales);
}

void q4_set_scratch(void * q8, void * q8_scales) { g_q8 = (int8_t *) q8; g_q8d = (float *) q8_scales; }
void q4_get_scratch(void ** q8, void ** q8_scales) { *q8 = g_q8; *q8_scales = g_q8d; }

// act: f32 rows [rows][ld_act] as store_act(W_Q4_0) leaves them
void q4_matmul(const DMat & W, const void * act, int ld_act, int rows, const MatmulEpilogue & ep, cudaStream_t s) {
    if (!g_q8 || !g_q8d) { fprintf(stderr, "bark_b200: q4_0 scratch buffers are not set\n"); throw std::runtime_error("unsupported configuration (see the message above)"); }
    const int nb = W.K / 32;
    const size_t warps = (size_t) rows * nb;
    BARK_LAUNCH(quantize_q8_kernel, (unsigned)((warps * 32 + 255) / 256), 256, 0, s, (const float *) act, ld_act, rows, W.K, g_q8, g_q8d);
    g_next_bytes = (double) W.n_out * nb * 18.0 + (double) rows * (W.K * 1.0 + nb * 4.0 + W.n_out * 4.0);
    g_next_flops = 2.0 * rows * (double) W.n_out * W.K;
    if (rows == 1) BARK_LAUNCH((q4_matmul_kernel<1, 1>), dim3((W.n_out + 31) / 32, 1), 256, 0, s, (const uint4 *) W.p, (const __half *) W.scales, W.K, W.n_out, g_q8, g_q8d, rows, ep);
    else           BARK_LAUNCH((q4_matmul_kernel<8, 4>), dim3((W.n_out + 127) / 128, (rows + 7) / 8), 256, 0, s, (const uint4 *) W.p, (const __half *) W.scales, W.K, W.n_out, g_q8, g_q8d, rows, ep);
}

}  // namespace bark
