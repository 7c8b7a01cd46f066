// Device-side pieces shared by the mat-mul and attention kernels: activation-operand writers, operand unpacking, GELU table lookup,
// the attention soft_max and P.V leftovers, and the mat-mul epilogues.
#pragma once
#include "gpt_kernels.h"

namespace bark {

// ------------------------------------------------------------------------------------------------
// activation operand writers: an activation value for column k of row m, in the format the next
// mul_mat consumes (the reference converts src1 to the weight's vec_dot_type, ggml.c:12530-12558)
// ------------------------------------------------------------------------------------------------
// activations are written in the group-major layout (common.cuh), gs = group stride in elements (= row capacity * 128)
// (q4_0 weights: plain f32 rows, gs = row stride; quantize_q8x_kernel turns them into q8_0 blocks in front of the mat-mul)
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

// soft_max over one row of n_kv <= 1024 by one warp (ggml.c:13953-14042 + ggml_vec_soft_max_f32 AVX2 branch ggml.c:2845-2888): in place.
// replays (optional): counts the rows whose 1/sum needed the sequential replay (the row tests; the attention kernels pass none).
__device__ __forceinline__ void softmax_row(float * __restrict__ p, int n_kv, unsigned * replays = nullptr) {
    const int lane = threadIdx.x & 31;
    float mx = __int_as_float(0xff800000);
    for (int i = lane; i < n_kv; i += 32) mx = fmaxf(mx, p[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const int nchunks = n_kv >> 3;
    float csum[4] = {0.f, 0.f, 0.f, 0.f};                                    // chunk c is owned by lane c%32, slot c/32 (n_kv <= 1024)
#pragma unroll
    for (int slot = 0; slot < 4; slot++) {
        const int c = slot * 32 + lane;
        if (c < nchunks) {
            float v[8];
#pragma unroll
            for (int l = 0; l < 8; l++) { v[l] = ggml_v_expf_dev(__fsub_rn(p[c * 8 + l], mx)); }
#pragma unroll
            for (int l = 0; l < 8; l++) p[c * 8 + l] = v[l];
            const float t0 = __fadd_rn(v[4], v[0]), t1 = __fadd_rn(v[5], v[1]), t2 = __fadd_rn(v[6], v[2]), t3 = __fadd_rn(v[7], v[3]);
            csum[slot] = __fadd_rn(__fadd_rn(t0, t2), __fadd_rn(t1, t3));
        }
    }
    // The reference accumulates the chunk sums sequentially in double, then the tail (ggml.c:2845-2888).  All terms are positive, so a
    // tree sum S brackets the sequential one within +-2n*2^-53*S: if 1/sum rounds to the same float at both ends of the bracket the
    // order cannot matter (the persistent decode step decides the same way); otherwise replay the sequential chain (128 dependent
    // shuffle + add steps per row: it used to run for every row).
    for (int i = nchunks * 8; i < n_kv; i++) {                                // scalar tail through libm expf
        const float val = glibc_expf_dev(__fsub_rn(p[i], mx));
        if (lane == 0) p[i] = val;
    }
    __syncwarp();
    double tsum = 0.0;
#pragma unroll
    for (int slot = 0; slot < 4; slot++) tsum += (double) csum[slot];         // (zero where this lane owns no chunk)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
    float sc;
    {
        const double dl = 2.0 * (double)(nchunks + 8) * 0x1p-53 * tsum * (1.0 + 1e-6);
        double lo = tsum - dl, hi = tsum + dl;
        for (int i = nchunks * 8; i < n_kv; i++) { const double tl = (double) p[i]; lo = __dadd_rn(lo, tl); hi = __dadd_rn(hi, tl); }
        const double mid = 0.5 * (lo + hi);
        double y = (double) __frcp_rn((float) mid);                          // 1/mid to ~2^-50: float seed + 2 Newton steps
        double e = __fma_rn(-mid, y, 1.0); y = __fma_rn(y, e, y);
        e = __fma_rn(-mid, y, 1.0);        y = __fma_rn(y, e, y);
        const double rw = (hi - lo) * y * 0.5 + 0x1p-48;
        sc = __double2float_rn(y * (1.0 - rw));
        if (sc != __double2float_rn(y * (1.0 + rw))) {                        // rare: the reference's own order
            double sum = 0.0;
#pragma unroll
            for (int slot = 0; slot < 4; slot++) {
                const int base = slot * 32;
                if (base < nchunks) {
                    const int cnt = min(32, nchunks - base);
                    for (int l = 0; l < cnt; l++) sum = __dadd_rn(sum, (double) __shfl_sync(0xffffffffu, csum[slot], l));
                }
            }
            for (int i = nchunks * 8; i < n_kv; i++) sum = __dadd_rn(sum, (double) p[i]);
            sc = __double2float_rn(__ddiv_rn(1.0, sum));
            if (replays && lane == 0) atomicAdd(replays, 1u);
        }
    }
    __syncwarp();
    for (int i = lane; i < n_kv; i += 32) p[i] = __fmul_rn(p[i], sc);
}

// P.V: the columns past the last full round of 32 lane chains (n_kv & ~31 .. n_kv), folded into the chains' reduced sum in the order
// the pinned build compiles vec_dot_f32's leftovers (oracle/bark_oracle.c orc_vec_dot_f32): runs of 8 and 4 multiply-then-add, then
// fused multiply-adds.  v: the V column (stride E), p: the probability row (global or shared memory: plain loads, never __ldg).
__device__ __forceinline__ float pv_leftovers(float sum, const float * __restrict__ v, const float * __restrict__ p, int np, int n_kv, int E) {
    int i = np, r = n_kv - np;
    while (r >= 8) { for (int l = 0; l < 8; l++) sum = __fadd_rn(sum, __fmul_rn(v[(size_t)(i + l) * E], p[i + l])); i += 8; r -= 8; }
    if (r >= 4)    { for (int l = 0; l < 4; l++) sum = __fadd_rn(sum, __fmul_rn(v[(size_t)(i + l) * E], p[i + l])); i += 4; r -= 4; }
    for (; r > 0; r--, i++) sum = __fmaf_rn(v[(size_t) i * E], p[i], sum);
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
