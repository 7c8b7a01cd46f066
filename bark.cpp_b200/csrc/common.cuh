// Shared device/host helpers for the H100-native bark hot path (sm_90a only).
//
// "Lane order": the reference's CPU dot products (ggml.c:2144 ggml_vec_dot_f32, ggml.c:2251
// ggml_vec_dot_f16, pinned AVX2/FMA build) keep 32 independent float accumulators — element k goes
// to virtual lane v = k % 32 and is folded in with one fused multiply-add, in increasing k — and
// then add the 32 partials in a fixed tree (GGML_F32x8_REDUCE, ggml.c:1405-1422).  A CUDA warp has
// exactly 32 lanes, so lane v of a warp owns virtual lane v: the serial chain lives in one thread,
// the tree is five xor-shuffles.  Every bit-exact kernel in this library is built on that mapping.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <atomic>
#include <exception>
#include <stdexcept>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

// A failed CUDA call is reported on stderr and thrown; every extern "C" entry point catches it and returns its failure value
// (nullptr / false / 0), as bark.h's contract says (bark.cpp:1174-1177, 2126-2141) — a drop-in library must not abort() its host.
namespace bark { struct CudaFailure { cudaError_t err; const char * file; int line; }; }
#define BARK_CUDA_CHECK(expr)                                                                         \
    do {                                                                                              \
        cudaError_t err__ = (expr);                                                                   \
        if (err__ != cudaSuccess) {                                                                   \
            fprintf(stderr, "bark_b200: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(err__), __FILE__, __LINE__, \
                    cudaGetErrorString(err__));                                                       \
            throw ::bark::CudaFailure{err__, __FILE__, __LINE__};                                     \
        }                                                                                             \
    } while (0)

namespace bark {

// run `f`; a CUDA failure (already reported) or any other exception becomes the entry point's failure value
template <typename R, typename F> inline R guarded(R fail, F && f) {
    try { return f(); }
    catch (const CudaFailure &) { return fail; }
    catch (const std::exception & e) { fprintf(stderr, "bark_b200: %s\n", e.what()); return fail; }
    catch (...) { fprintf(stderr, "bark_b200: unexpected exception\n"); return fail; }
}

// Process-wide state is limited to counters (atomic) and per-thread annotations (thread_local), so that one host thread per GPU can
// drive its own bark_context inside one process (SURVEY.md §5; tests/test_parity_gpu.py two-thread case).
// number of kernels this library launched (bench.py reports it as gpu_launches)
extern std::atomic<unsigned long long> g_kernel_launches;
// host<->device traffic issued by the library (bench.py: e2e.h2d_bytes_per_step / d2h_bytes_per_step)
extern std::atomic<unsigned long long> g_h2d_bytes, g_d2h_bytes;
// Kernel attributes (cudaFuncSetAttribute) are per DEVICE: true exactly once per (call site's mask, current device).
inline bool first_use_on_this_device(std::atomic<unsigned long long> & mask) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev > 63) return true;
    return !(mask.fetch_or(1ull << dev) >> dev & 1ull);
}
// optional per-launch device timing (prof.cu): CUDA events on the launching stream around every kernel
extern bool g_prof_on;
void prof_begin(const char * name, cudaStream_t s, double bytes, double flops);
void prof_end(cudaStream_t s);
// annotate the NEXT launch with its algorithmic HBM bytes and/or flops for the roofline report
extern thread_local double g_next_bytes, g_next_flops;
#define BARK_LAUNCH(kernel, grid, block, smem, stream, ...)                                           \
    do {                                                                                              \
        if (::bark::g_prof_on) ::bark::prof_begin(#kernel, (stream), ::bark::g_next_bytes, ::bark::g_next_flops);            \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                                   \
        if (::bark::g_prof_on) ::bark::prof_end((stream));                                            \
        ::bark::g_next_bytes = ::bark::g_next_flops = 0.0;                                                                    \
        ++::bark::g_kernel_launches;                                                                  \
    } while (0)

// Same, with programmatic dependent launch (PDL): the kernel may start while its predecessor in the stream is still draining and
// runs its own prologue (barrier init, TMEM allocation, tensor-map prefetch) meanwhile; it MUST execute griddepcontrol.wait before it
// touches anything the predecessor wrote.  Used by the fast-mode chain of 2-20 us kernels (fast_kernels.cu).
#define BARK_LAUNCH_PDL(kernel, grid, block, smem, strm__, ...)                                       \
    do {                                                                                              \
        if (::bark::g_prof_on) ::bark::prof_begin(#kernel, (strm__), ::bark::g_next_bytes, ::bark::g_next_flops);            \
        cudaLaunchConfig_t cfg__ = {};                                                                \
        cfg__.gridDim = (grid); cfg__.blockDim = (block); cfg__.dynamicSmemBytes = (smem); cfg__.stream = (strm__);          \
        cudaLaunchAttribute at__[1];                                                                  \
        at__[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at__[0].val.programmaticStreamSerializationAllowed = 1; \
        cfg__.attrs = at__; cfg__.numAttrs = 1;                                                       \
        BARK_CUDA_CHECK(cudaLaunchKernelEx(&cfg__, kernel, __VA_ARGS__));                             \
        if (::bark::g_prof_on) ::bark::prof_end((strm__));                                            \
        ::bark::g_next_bytes = ::bark::g_next_flops = 0.0;                                                                    \
        ++::bark::g_kernel_launches;                                                                  \
    } while (0)

// weight element types as stored in ggml_weights.bin (ggml_type values, SURVEY App. A)
enum WType : int { W_F32 = 0, W_F16 = 1, W_Q4_0 = 2, W_Q4_1 = 3, W_Q5_0 = 6, W_Q5_1 = 7, W_Q8_0 = 8 };   // 3..8: qx_kernels.cu
inline bool is_quant(WType t) { return t != W_F32 && t != W_F16; }

// Element e of a quantised matrix kept in the file's blocks (rows are whole blocks of 32): the f32 that dequantize_row_<t>
// (ggml-quants.c:1522-1630) computes.  q5 codes take their fifth bit from bit j of qh.  x*d + m of q4_1 / q5_1 is one fused
// multiply-add in the pinned build (vfmadd132ps); x*d is exact in f32 (a code below 32 times an f16), so a separate product and sum
// would give the same value (tests/test_fast_weights.py checks both forms against tests/golden/ref_pairs/dequant.npz).
__device__ __forceinline__ float dequant_element(const unsigned char * blocks, WType t, size_t e) {
    const int bytes = t == W_Q4_0 ? 18 : t == W_Q4_1 ? 20 : t == W_Q5_0 ? 22 : t == W_Q5_1 ? 24 : 34;
    const unsigned char * b = blocks + (e >> 5) * bytes;
    const int j = (int)(e & 31);
    const float d = __half2float(__ushort_as_half((unsigned short)(b[0] | (b[1] << 8))));
    if (t == W_Q8_0) return __fmul_rn((float)(signed char) b[2 + j], d);
    const bool has_m = t == W_Q4_1 || t == W_Q5_1, q5 = t == W_Q5_0 || t == W_Q5_1;
    const unsigned char * qs = b + 2 + (has_m ? 2 : 0) + (q5 ? 4 : 0);
    int q = j < 16 ? (qs[j] & 0x0f) : (qs[j - 16] >> 4);
    if (q5) q |= ((b[2 + (has_m ? 2 : 0) + (j >> 3)] >> (j & 7)) & 1) << 4;
    if (has_m) return __fmaf_rn((float) q, d, __half2float(__ushort_as_half((unsigned short)(b[2] | (b[3] << 8)))));
    return __fmul_rn((float)(q - (q5 ? 16 : 8)), d);
}

// ---------------------------------------------------------------------------------------------
// Lane-interleaved ("LI") matrix layout.
// A row of K elements (K % 32 == 0) is cut into chain steps c = k / 32 for virtual lane v = k % 32.
// G consecutive chain steps of one lane are stored contiguously as one 16-byte vector
// (G = 8 for f16, 4 for f32), vectors of the 32 lanes are adjacent:
//     offset(k) = ((c / G) * 32 + v) * G + (c % G)          [elements, within the row]
// so one warp-wide 16-byte load fetches G chain steps for all 32 lanes, fully coalesced (512 B).
// Rows are padded to a multiple of 32*G elements; kernels never touch chain steps >= K/32.
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline int li_group(int elem_bytes) { return 16 / elem_bytes; }
__host__ __device__ inline int li_padded_k(int K, int elem_bytes) { const int q = 32 * li_group(elem_bytes); return (K + q - 1) / q * q; }
__host__ __device__ inline int li_offset(int k, int G) { const int v = k & 31, c = k >> 5; return ((c / G) * 32 + v) * G + (c % G); }

// Group-major ("GM") operand layout of the multi-row mat-muls.  A k-group is 128 consecutive columns = 4 chain steps of
// every lane; element (row r, column k) lives at  (k/128) * gs + r * 128 + (k%32) * 4 + (k/32)%4  with gs = rows_cap * 128.
// For a fixed group the rows are contiguous, so a block tile of R rows x 128 columns is ONE contiguous R*128-element span
// (one bulk copy), and lane v's 4 elements of a row are one 8-byte (f16) / 16-byte (f32) word at stride = word size:
// bank-conflict free in shared memory.
constexpr int kGmGroup = 128;
__host__ __device__ inline size_t gm_offset(int r, int k, size_t gs) { return (size_t)(k >> 7) * gs + (size_t) r * kGmGroup + (size_t)((k & 31) << 2) + (size_t)((k >> 5) & 3); }
__host__ __device__ inline int gm_groups(int K) { return (K + kGmGroup - 1) / kGmGroup; }

#ifdef __CUDACC__
// GGML_F32x8_REDUCE (ggml.c:1405-1422) over the 32 lane partials; every lane returns the result.
// x0+=x2, x1+=x3 (xor 16); x0+=x1 (xor 8); t[l]=x0[l]+x0[l+4] (xor 4); (t0+t1)+(t2+t3) (xor 1, xor 2).
__device__ __forceinline__ float lane_tree_reduce(float a) {
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 16));
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 8));
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 4));
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 1));
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 2));
    return a;
}

// same tree, over a 32-entry array held by ONE thread (index = virtual lane)
__device__ __forceinline__ float lane_tree_reduce_local(const float (&a)[32]) {
    float x0[8];
#pragma unroll
    for (int l = 0; l < 8; l++) x0[l] = __fadd_rn(__fadd_rn(a[l], a[16 + l]), __fadd_rn(a[8 + l], a[24 + l]));
    float t0 = __fadd_rn(x0[0], x0[4]), t1 = __fadd_rn(x0[1], x0[5]), t2 = __fadd_rn(x0[2], x0[6]), t3 = __fadd_rn(x0[3], x0[7]);
    return __fadd_rn(__fadd_rn(t0, t1), __fadd_rn(t2, t3));
}

// f32 -> f16 -> f32 round trip (what converting an activation row to the f16 vec_dot_type does,
// ggml.c:12551-12555 + ggml_fp32_to_fp16_row RNE)
__device__ __forceinline__ float round_f16(float x) { return __half2float(__float2half_rn(x)); }

// ggml_v_expf, AVX2+FMA flavour (ggml.c:2706-2746), one lane
__device__ __forceinline__ float ggml_v_expf_dev(float x) {
    const float r = 0x1.8p23f;
    const float z = __fmaf_rn(x, 0x1.715476p+0f, r);
    const float n = __fsub_rn(z, r);
    const float b = __fmaf_rn(-n, 0x1.7f7d1cp-20f, __fmaf_rn(-n, 0x1.62e4p-1f, x));
    const uint32_t e = __float_as_uint(z) << 23;
    const float k = __uint_as_float(e + 0x3f800000u);
    const float an = fabsf(n);
    const float u = __fmul_rn(b, b);
    const float j = __fmaf_rn(__fmaf_rn(__fmaf_rn(0x1.0e4020p-7f, b, 0x1.573e2ep-5f), u, __fmaf_rn(0x1.555e66p-3f, b, 0x1.fffdb6p-2f)), u,
                              __fmul_rn(0x1.ffffecp-1f, b));
    if (!(an > 126.0f)) return __fmaf_rn(j, k, k);
    const uint32_t g = (n <= 0.0f) ? 0x82000000u : 0u;
    const float s1 = __uint_as_float(g + 0x7f000000u);
    const float s2 = __uint_as_float(e - g);
    if (an > 192.0f) return __fmul_rn(s1, s1);
    return __fmul_rn(__fmaf_rn(s2, j, s2), s1);
}

// glibc 2.39 expf (sysdeps/ieee754/flt-32/e_expf.c; table = 2^(i/32) with the exponent folded out),
// used by the soft_max tail columns (ggml.c:2880-2884).  Verified against host expf over 3.2e8
// inputs on the build host (DESIGN.md, "libm on the device").
__device__ __constant__ uint64_t c_exp2f_tab[32] = {
    0x3ff0000000000000ULL, 0x3fefd9b0d3158574ULL, 0x3fefb5586cf9890fULL, 0x3fef9301d0125b51ULL,
    0x3fef72b83c7d517bULL, 0x3fef54873168b9aaULL, 0x3fef387a6e756238ULL, 0x3fef1e9df51fdee1ULL,
    0x3fef06fe0a31b715ULL, 0x3feef1a7373aa9cbULL, 0x3feedea64c123422ULL, 0x3feece086061892dULL,
    0x3feebfdad5362a27ULL, 0x3feeb42b569d4f82ULL, 0x3feeab07dd485429ULL, 0x3feea47eb03a5585ULL,
    0x3feea09e667f3bcdULL, 0x3fee9f75e8ec5f74ULL, 0x3feea11473eb0187ULL, 0x3feea589994cce13ULL,
    0x3feeace5422aa0dbULL, 0x3feeb737b0cdc5e5ULL, 0x3feec49182a3f090ULL, 0x3feed503b23e255dULL,
    0x3feee89f995ad3adULL, 0x3feeff76f2fb5e47ULL, 0x3fef199bdd85529cULL, 0x3fef3720dcef9069ULL,
    0x3fef5818dcfba487ULL, 0x3fef7c97337b9b5fULL, 0x3fefa4afa2a490daULL, 0x3fefd0765b6e4540ULL,
};
__device__ __forceinline__ float glibc_expf_dev(float x) {
    const uint32_t ux = __float_as_uint(x);
    const uint32_t abstop = (ux >> 20) & 0x7ffu;
    if (abstop >= 0x42bu) {                        // |x| >= 88 or nan
        if (ux == 0xff800000u) return 0.0f;
        if (abstop >= 0x7f8u) return x + x;
        if (x > 0x1.62e42ep6f) return __int_as_float(0x7f800000);
        if (x < -0x1.9fe368p6f) return 0.0f;
    }
    const double xd = (double) x;
    double z = __dmul_rn(0x1.71547652b82fep+0 * 32.0, xd);
    double kd = __dadd_rn(z, 0x1.8p+52);
    const uint64_t ki = (uint64_t) __double_as_longlong(kd);
    kd = __dsub_rn(kd, 0x1.8p+52);
    const double r = __dsub_rn(z, kd);
    uint64_t t = c_exp2f_tab[ki & 31];
    t += ki << 47;
    const double s = __longlong_as_double((long long) t);
    const double C0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, C1 = 0x1.ebfce50fac4f3p-3 / 32 / 32, C2 = 0x1.62e42ff0c52d6p-1 / 32;
    z = __dadd_rn(__dmul_rn(C0, r), C1);
    const double r2 = __dmul_rn(r, r);
    double y = __dadd_rn(__dmul_rn(C2, r), 1.0);
    y = __dadd_rn(__dmul_rn(z, r2), y);
    y = __dmul_rn(y, s);
    return __double2float_rn(y);
}

// glibc 2.39 expm1f / tanhf (sysdeps/ieee754/flt-32/s_expm1f.c, s_tanhf.c: the fdlibm float algorithms), restated with
// explicit IEEE single-precision operations.  ELU uses expm1f (ggml.c:2533), the LSTM gates tanhf / expf (ggml.c:2532,2536).
// The C restatement was checked against the host libm on 3.3e8 inputs spanning every float (DESIGN.md, "libm on the device").
__device__ __forceinline__ float glibc_expm1f_dev(float x) {
    const float one = 1.0f, huge = 1.0e+30f, tiny = 1.0e-30f, o_threshold = 8.8721679688e+01f, ln2_hi = 6.9313812256e-01f,
                ln2_lo = 9.0580006145e-06f, invln2 = 1.4426950216e+00f, Q1 = -3.3333335072e-02f, Q2 = 1.5873016091e-03f,
                Q3 = -7.9365076090e-05f, Q4 = 4.0082177293e-06f, Q5 = -2.0109921195e-07f;
    float y, hi, lo, c = 0.0f, t, e, hxs, hfx, r1;
    int k;
    uint32_t hx = __float_as_uint(x);
    const uint32_t xsb = hx & 0x80000000u;
    hx &= 0x7fffffffu;
    if (hx >= 0x4195b844u) {                       // |x| >= 27 ln2
        if (hx >= 0x42b17218u) {
            if (hx > 0x7f800000u) return __fadd_rn(x, x);
            if (hx == 0x7f800000u) return xsb == 0 ? x : -1.0f;
            if (x > o_threshold) return __fmul_rn(huge, huge);
        }
        if (xsb != 0) return __fsub_rn(tiny, one);
    }
    if (hx > 0x3eb17218u) {                        // |x| > 0.5 ln2
        if (hx < 0x3F851592u) {
            if (xsb == 0) { hi = __fsub_rn(x, ln2_hi); lo = ln2_lo; k = 1; }
            else          { hi = __fadd_rn(x, ln2_hi); lo = -ln2_lo; k = -1; }
        } else {
            k = __float2int_rz(__fadd_rn(__fmul_rn(invln2, x), xsb == 0 ? 0.5f : -0.5f));
            t = (float) k;
            hi = __fsub_rn(x, __fmul_rn(t, ln2_hi));
            lo = __fmul_rn(t, ln2_lo);
        }
        x = __fsub_rn(hi, lo);
        c = __fsub_rn(__fsub_rn(hi, x), lo);
    } else if (hx < 0x33000000u) {                 // |x| < 2^-25
        t = __fadd_rn(huge, x);
        return __fsub_rn(x, __fsub_rn(t, __fadd_rn(huge, x)));
    } else k = 0;
    hfx = __fmul_rn(0.5f, x);
    hxs = __fmul_rn(x, hfx);
    r1 = __fadd_rn(one, __fmul_rn(hxs, __fadd_rn(Q1, __fmul_rn(hxs, __fadd_rn(Q2, __fmul_rn(hxs, __fadd_rn(Q3, __fmul_rn(hxs, __fadd_rn(Q4, __fmul_rn(hxs, Q5)))))))))); 
    t = __fsub_rn(3.0f, __fmul_rn(r1, hfx));
    e = __fmul_rn(hxs, __fdiv_rn(__fsub_rn(r1, t), __fsub_rn(6.0f, __fmul_rn(x, t))));
    if (k == 0) return __fsub_rn(x, __fsub_rn(__fmul_rn(x, e), hxs));
    e = __fsub_rn(__fmul_rn(x, __fsub_rn(e, c)), c);
    e = __fsub_rn(e, hxs);
    if (k == -1) return __fsub_rn(__fmul_rn(0.5f, __fsub_rn(x, e)), 0.5f);
    if (k == 1) {
        if (x < -0.25f) return __fmul_rn(-2.0f, __fsub_rn(e, __fadd_rn(x, 0.5f)));
        return __fadd_rn(one, __fmul_rn(2.0f, __fsub_rn(x, e)));
    }
    if (k <= -2 || k > 56) {
        y = __fsub_rn(one, __fsub_rn(e, x));
        y = __uint_as_float(__float_as_uint(y) + ((uint32_t) k << 23));
        return __fsub_rn(y, one);
    }
    if (k < 23) {
        t = __uint_as_float(0x3f800000u - (0x1000000u >> k));
        y = __fsub_rn(t, __fsub_rn(e, x));
        y = __uint_as_float(__float_as_uint(y) + ((uint32_t) k << 23));
    } else {
        t = __uint_as_float((uint32_t)(0x7f - k) << 23);
        y = __fsub_rn(x, __fadd_rn(e, t));
        y = __fadd_rn(y, one);
        y = __uint_as_float(__float_as_uint(y) + ((uint32_t) k << 23));
    }
    return y;
}

__device__ __forceinline__ float glibc_tanhf_dev(float x) {
    const float one = 1.0f, two = 2.0f, tiny = 1.0e-30f;
    const uint32_t jx = __float_as_uint(x), ix = jx & 0x7fffffffu;
    float t, z;
    if (ix >= 0x7f800000u) return (jx & 0x80000000u) ? __fsub_rn(__fdiv_rn(one, x), one) : __fadd_rn(__fdiv_rn(one, x), one);
    if (ix < 0x41b00000u) {                        // |x| < 22
        if (ix == 0) return x;
        if (ix < 0x24000000u) return __fmul_rn(x, __fadd_rn(one, x));
        if (ix >= 0x3f800000u) { t = glibc_expm1f_dev(__fmul_rn(two, fabsf(x))); z = __fsub_rn(one, __fdiv_rn(two, __fadd_rn(t, two))); }
        else                   { t = glibc_expm1f_dev(__fmul_rn(-two, fabsf(x))); z = __fdiv_rn(-t, __fadd_rn(t, two)); }
    } else z = __fsub_rn(one, tiny);
    return (jx & 0x80000000u) ? -z : z;
}

__device__ __forceinline__ float elu_exact(float x) { return x > 0.f ? x : glibc_expm1f_dev(x); }                       // ggml.c:2533
__device__ __forceinline__ float sigmoid_exact(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, glibc_expf_dev(-x))); } // ggml.c:2536
#endif  // __CUDACC__

}  // namespace bark
