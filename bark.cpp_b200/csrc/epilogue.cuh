// Device-side pieces shared by the mat-mul kernels: activation-operand writers, operand unpacking, GELU table lookup
// and the mat-mul epilogues.
#pragma once
#include "gpt_kernels.h"

namespace bark {

// ------------------------------------------------------------------------------------------------
// activation operand writers: an activation value for column k of row m, in the format the next
// mul_mat consumes (the reference converts src1 to the weight's vec_dot_type, ggml.c:12530-12558)
// ------------------------------------------------------------------------------------------------
// activations are written in the group-major layout (common.cuh), gs = group stride in elements (= row capacity * 128)
// (q4_0 weights: plain f32 rows, gs = row stride; quantize_q8_kernel turns them into q8_0 blocks in front of the mat-mul)
__device__ __forceinline__ void store_act(void * act, int wt, int gs, int m, int k, float v) {
    if (wt == W_Q4_0) { ((float *) act)[(size_t) m * gs + k] = v; return; }
    const size_t off = gm_offset(m, k, (size_t) gs);
    if (wt == W_F16) ((__half *) act)[off] = __float2half_rn(v);
    else             ((float *) act)[off] = v;
}

template <typename T> __device__ __forceinline__ void unpack16(const uint4 & u, float (&f)[16 / sizeof(T)]);
template <> __device__ __forceinline__ void unpack16<__half>(const uint4 & u, float (&f)[8]) {
    const __half2 * h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
    for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
template <> __device__ __forceinline__ void unpack16<float>(const uint4 & u, float (&f)[4]) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
}

__device__ __forceinline__ float gelu_lookup(const __half * __restrict__ tab, float x) {   // ggml_vec_gelu_f32, ggml.c:2557-2571
    if (x <= -10.0f) return 0.0f;
    if (x >= 10.0f) return x;
    return __half2float(tab[__half_as_ushort(__float2half_rn(x))]);
}

// P.V: the columns past the last full round of 32 lane chains (n_kv & ~31 .. n_kv), folded into the chains' reduced sum in the order
// the pinned build compiles vec_dot_f32's leftovers (oracle/bark_oracle.c orc_vec_dot_f32): runs of 8 and 4 multiply-then-add, then
// fused multiply-adds.  v: the V column (stride E), p: the probability row.
__device__ __forceinline__ float pv_leftovers(float sum, const float * __restrict__ v, const float * __restrict__ p, int np, int n_kv, int E) {
    int i = np, r = n_kv - np;
    while (r >= 8) { for (int l = 0; l < 8; l++) sum = __fadd_rn(sum, __fmul_rn(__ldg(v + (size_t)(i + l) * E), __ldg(p + i + l))); i += 8; r -= 8; }
    if (r >= 4)    { for (int l = 0; l < 4; l++) sum = __fadd_rn(sum, __fmul_rn(__ldg(v + (size_t)(i + l) * E), __ldg(p + i + l))); i += 4; r -= 4; }
    for (; r > 0; r--, i++) sum = __fmaf_rn(__ldg(v + (size_t) i * E), __ldg(p + i), sum);
    return sum;
}

__device__ __forceinline__ void matmul_epilogue(const MatmulEpilogue & ep, int m, int o, float r) {
    switch (ep.mode) {
        case EPI_STORE: ep.out[(size_t) m * ep.ldo + o] = r; break;
        case EPI_RESID: { float * p = ep.out + (size_t) m * ep.ldo + o; *p = __fadd_rn(r, *p); } break;
        case EPI_GELU_ACT: store_act(ep.act_out, ep.act_wt, ep.act_Kp, m, o, gelu_lookup(ep.gelu_tab, r)); break;
        case EPI_QKV: {
            const int E = ep.ldo;
            if (o < E)          ep.out[(size_t) m * E + o] = r;
            else if (o < 2 * E) { ep.k_out[(size_t) m * E + (o - E)] = r;     for (int p = 0; p < ep.n_peer; p++) ep.k_peer[p][(size_t) m * E + (o - E)] = r; }
            else                { ep.v_out[(size_t) m * E + (o - 2 * E)] = r; for (int p = 0; p < ep.n_peer; p++) ep.v_peer[p][(size_t) m * E + (o - 2 * E)] = r; }
        } break;
    }
}


}  // namespace bark
