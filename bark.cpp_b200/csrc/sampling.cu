// Device-side token sampling: gpt_sample (bark.cpp:184-270) for a batch of logit rows, bit-faithful to the host path.
//
// The reference samples on the CPU: l /= temp; float softmax with the DOUBLE exp() and a SEQUENTIAL float sum; then
// libstdc++'s std::discrete_distribution (double normalisation, sequential double partial sums, last one forced to 1,
// lower_bound of one generate_canonical<double,53> draw; bits/random.tcc:2657-2730).  Doing that on the host costs a
// logits read-back per step (4.3 MB per fine pass) plus 50-190 us of scalar work per sample — ~100 ms of a 2.76 s clip.
//
// Here one CTA owns one row:
//   * divisions, max, exps: parallel over the row;
//   * the float sum: strictly sequential on one thread (the order IS the result);
//   * exp: CUDA's double exp (<= 1 ulp) rounded to float.  glibc's exp is also < 1 ulp, so the two can only round to
//     different floats when the double lies within a few ulp of a float rounding boundary: that is detected
//     (both ends of a +-2^-50 relative bracket must round to the same float) and the row is FLAGGED;
//   * the multinomial draw: the uniform u comes from the host's std::mt19937 stream (same two 32-bit draws per sample);
//     the partial sums are formed in parallel in double and compared with u * total; if any partial sum lies within the
//     rounding-error bound of the threshold the row is FLAGGED.
// Flagged rows are re-sampled on the host with the reference's exact sequence, using the same u, so the token stream is
// identical to the host path in all cases.  How often real rows are flagged has not been measured.  tests/test_sampler_orders.py
// restates both orders and brackets and builds rows on the decision edges; tests/test_sampler_gpu.py runs them through both
// instantiations (bark_b200_sample_given_u).  eps = 0 fails test_threshold_rows and test_edge_rows; `>=` in the per-thread argmax
// fails test_argmax_rows; dropping the exp check fails test_exp_rows and test_exp_rounding_against_glibc (DESIGN.md section 2).
#include "gpt_kernels.h"

namespace bark {

// gpt_sample for ONE logit row by one thread block of kSampleThreads threads.  sh: [n] floats of shared memory; lg: the n logits of the row
template <int kSampleThreads>
__device__ __forceinline__ void sample_row_body(float * sh, const float * lg, int n, float temp, double u, int32_t * out_tok, int tok_add, int32_t * feed,
                                                float * eos_p, int32_t * flags, int force_flag) {
    __shared__ float s_f[kSampleThreads / 32]; __shared__ int s_i[kSampleThreads / 32]; __shared__ double s_d[kSampleThreads / 32];
    __shared__ float s_sum; __shared__ int s_amb;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = kSampleThreads / 32;
    const float div = temp == 0.0f ? 0.7f : temp;        // the argmax path still divides by 0.7 (bark.cpp:226-228)
    bool ambiguous = force_flag != 0;
    if (tid == 0) s_amb = 0;

    float mx = __int_as_float(0xff800000);
    for (int i = tid; i < n; i += kSampleThreads) { const float l = __fdiv_rn(__ldcg(lg + i), div); sh[i] = l; mx = fmaxf(mx, l); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_f[warp] = mx;
    __syncthreads();
    mx = s_f[0];
#pragma unroll
    for (int w = 1; w < NW; w++) mx = fmaxf(mx, s_f[w]);
    for (int i = tid; i < n; i += kSampleThreads) {
        const double y = exp((double) __fsub_rn(sh[i], mx));
        if (__double2float_rn(y * (1.0 - 0x1p-50)) != __double2float_rn(y * (1.0 + 0x1p-50))) ambiguous = true;
        sh[i] = __double2float_rn(y);
    }
    __syncthreads();
    if (tid == 0) {                                      // sequential float sum (bark.cpp:191-195): the order IS the result
        float sum = 0.0f;
        int i = 0;
        for (; i + 8 <= n; i += 8) {
            const float4 a = *reinterpret_cast<const float4 *>(sh + i), b = *reinterpret_cast<const float4 *>(sh + i + 4);
            sum = __fadd_rn(sum, a.x); sum = __fadd_rn(sum, a.y); sum = __fadd_rn(sum, a.z); sum = __fadd_rn(sum, a.w);
            sum = __fadd_rn(sum, b.x); sum = __fadd_rn(sum, b.y); sum = __fadd_rn(sum, b.z); sum = __fadd_rn(sum, b.w);
        }
        for (; i < n; i++) sum = __fadd_rn(sum, sh[i]);
        s_sum = sum;
    }
    __syncthreads();
    const float sum = s_sum;
    for (int i = tid; i < n; i += kSampleThreads) sh[i] = __fdiv_rn(sh[i], sum);
    __syncthreads();

    int token = 0;
    if (temp == 0.0f) {                                  // gpt_argmax_sample: first strict maximum
        float best = __int_as_float(0xff800000); int bi = 0x7fffffff;
        for (int i = tid; i < n; i += kSampleThreads) { const float p = sh[i]; if (p > best) { best = p; bi = i; } }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (lane == 0) { s_f[warp] = best; s_i[warp] = bi; }
        __syncthreads();
        best = s_f[0]; bi = s_i[0];
#pragma unroll
        for (int w = 1; w < NW; w++) if (s_f[w] > best || (s_f[w] == best && s_i[w] < bi)) { best = s_f[w]; bi = s_i[w]; }
        token = bi;
    } else {
        // thread t owns the contiguous chunk [t*c, (t+1)*c): local sums, block scan of the chunk sums, then the crossing search
        const int c = (n + kSampleThreads - 1) / kSampleThreads, lo = min(n, tid * c), hi = min(n, lo + c);
        double part = 0.0;
        for (int i = lo; i < hi; i++) part += (double) sh[i];
        double incl = part;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) s_d[warp] = incl;
        __syncthreads();
        double before = 0.0, total = 0.0;
#pragma unroll
        for (int w = 0; w < NW; w++) { if (w < warp) before += s_d[w]; total += s_d[w]; }
        const double thr = u * total;               // cp[i] >= u  <=>  (sum_{j<=i} p_j) / total >= u, up to rounding
        const double eps = 8.0 * (double) n * 0x1p-53 * total;
        double run = before + incl - part;
        int first = 0x7fffffff;
        for (int i = lo; i < hi; i++) {
            run += (double) sh[i];
            if (i < n - 1) {                             // the last partial sum is forced to 1.0 >= u
                if (fabs(run - thr) <= eps) ambiguous = true;
                if (run >= thr && first == 0x7fffffff) first = i;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
        if (lane == 0) s_i[warp] = first;
        __syncthreads();
        first = s_i[0];
#pragma unroll
        for (int w = 1; w < NW; w++) first = min(first, s_i[w]);
        token = first == 0x7fffffff ? n - 1 : first;
    }
    if (ambiguous) s_amb = 1;
    __syncthreads();
    if (tid == 0) {
        *out_tok = token + tok_add;
        if (feed) *feed = token + tok_add;
        if (eos_p) *eos_p = sh[n - 1];                   // probability of the LAST logit (bark.cpp:216-218)
        *flags = s_amb;
    }
}

// 256 threads per row when many rows are sampled at once (fine passes: 1024 rows), 1024 threads for the single row of a decode
// step (the exp / division / scan passes of a 10 048-wide semantic row are 4x shorter; the sequential sum is unchanged)

// One CTA per row.  tok_add is added to the sampled index (coarse stage: offset of the codebook window in
// the vocabulary); feed, when set, receives the token for the NEXT decode step to read (no host round trip).
template <int kSampleThreads>
__global__ void __launch_bounds__(kSampleThreads) sample_rows_kernel(const float * __restrict__ logits, int ld, int n, int rows, float temp, const double * __restrict__ u,
                                                                     int32_t * __restrict__ out_tok, int tok_add, int32_t * __restrict__ feed,
                                                                     float * __restrict__ eos_p, int32_t * __restrict__ flags, int force_flag) {
    extern __shared__ float sh[];                        // [n] working row
    const int row = blockIdx.x;
    sample_row_body<kSampleThreads>(sh, logits + (size_t) row * ld, n, temp, temp != 0.0f ? u[row] : 0.0, out_tok + row, tok_add, feed ? feed + row : nullptr,
                                    eos_p ? eos_p + row : nullptr, flags + row, force_flag);
}

void sample_rows(const float * logits, int ld, int n, int rows, float temp, const double * d_u, int32_t * d_out_tok, int tok_add, int32_t * d_feed,
                 float * d_eos_p, int32_t * d_flags, int force_flag, cudaStream_t s) {
    const size_t smem = ((size_t) n * sizeof(float) + 15) & ~(size_t) 15;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) {
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    }
    g_next_bytes = (double) rows * n * 4.0;
    if (rows == 1) BARK_LAUNCH(sample_rows_kernel<1024>, rows, 1024, smem, s, logits, ld, n, rows, temp, d_u, d_out_tok, tok_add, d_feed, d_eos_p, d_flags, force_flag);
    else           BARK_LAUNCH(sample_rows_kernel<256>, rows, 256, smem, s, logits, ld, n, rows, temp, d_u, d_out_tok, tok_add, d_feed, d_eos_p, d_flags, force_flag);
}

// The same kernels with the instantiation chosen by the caller (bark_b200_sample_given_u, tests): threads 0 picks as sample_rows does,
// 256 or 1024 forces that one, so every row can be checked at both.  Rows are packed (ld = n), no offset, no feed, no forced flag.
void sample_rows_threads(int threads, const float * logits, int n, int rows, float temp, const double * d_u, int32_t * d_out_tok, float * d_eos_p,
                         int32_t * d_flags, cudaStream_t s) {
    const size_t smem = ((size_t) n * sizeof(float) + 15) & ~(size_t) 15;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) {
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    }
    if (threads == 0) threads = rows == 1 ? 1024 : 256;
    if (threads == 1024) BARK_LAUNCH(sample_rows_kernel<1024>, rows, 1024, smem, s, logits, n, n, rows, temp, d_u, d_out_tok, 0, nullptr, d_eos_p, d_flags, 0);
    else                 BARK_LAUNCH(sample_rows_kernel<256>, rows, 256, smem, s, logits, n, n, rows, temp, d_u, d_out_tok, 0, nullptr, d_eos_p, d_flags, 0);
}

}  // namespace bark
