// Token sampling: gpt_sample (bark.cpp:184-270) for a batch of logit rows on the device, bit-faithful to the reference's, with
// the host replay of the rows the device cannot decide.
//
// The reference samples on the CPU: l /= temp; float softmax with the DOUBLE exp() and a SEQUENTIAL float sum; then
// libstdc++'s discrete distribution (double normalisation, sequential double partial sums, last one forced to 1,
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
// Flagged rows are re-sampled on the host with the reference's exact sequence (sample_token_given_u), using the same u, so the
// token stream is the reference's in all cases.  How often real rows are flagged has not been measured.  tests/test_sampler_orders.py
// restates both orders and brackets and builds rows on the decision edges; tests/test_sampler_gpu.py runs them through both
// instantiations (bark_b200_sample_given_u).  eps = 0 fails test_threshold_rows and test_edge_rows; `>=` in the per-thread argmax
// fails test_argmax_rows; dropping the exp check fails test_exp_rows and test_exp_rounding_against_glibc (DESIGN.md section 2).
#include "context.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>

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
                 float * d_eos_p, int32_t * d_flags, int force_flag, int threads, cudaStream_t s) {
    const size_t smem = ((size_t) n * sizeof(float) + 15) & ~(size_t) 15;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) {
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSampleMaxLogits * (int) sizeof(float)));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(sample_rows_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSampleMaxLogits * (int) sizeof(float)));
    }
    // 256 threads per row when many rows are sampled at once (fine passes: 1024 rows), 1024 threads for the single row of a decode
    // step (the exp / division / scan passes of a 10 048-wide semantic row are 4x shorter; the sequential sum is unchanged)
    if (threads == 0) threads = rows == 1 ? 1024 : 256;
    g_next_bytes = (double) rows * n * 4.0;
    if (threads == 1024) BARK_LAUNCH(sample_rows_kernel<1024>, rows, 1024, smem, s, logits, ld, n, rows, temp, d_u, d_out_tok, tok_add, d_feed, d_eos_p, d_flags, force_flag);
    else                 BARK_LAUNCH(sample_rows_kernel<256>, rows, 256, smem, s, logits, ld, n, rows, temp, d_u, d_out_tok, tok_add, d_feed, d_eos_p, d_flags, force_flag);
}

// ---------------------------------------------------------------------------------------------
// top-k / top-p filter (upstream Bark's generate_text_semantic / generate_coarse, on the reference's arithmetic; DESIGN.md §14)
// ---------------------------------------------------------------------------------------------
// One CTA per row.  Every logit becomes the 64-bit key (order-preserving bits of x, -0 read as +0) << 32 | index, so a descending
// sort of the keys is "x descending, ties by descending index" (np.argsort(x, kind="stable")[::-1]).  Keys are bitonic-sorted in
// shared memory.  Sorted position j keeps its logit when j < K, so the whole filter reduces to K and the key at K - 1:
//   top-p  e_j = (float) exp((double)(y_j - y_0)) in parallel (the sampler's exp bracket flags the row), then on one thread the
//          two sequential float chains of the reference's softmax and cumsum: S = e_0 + e_1 + ..., c_j = p_0 + ... + p_j with
//          p_j = e_j / S; K_p = 1 + the first j with c_j > top_p (n if none).  Both chains stop at the first e_j < 2^-26: from
//          there on every term is below half an ulp of the running sum (S >= e_0 = 1, c >= p_0 = 1 / S), so the rest of each sum
//          is exact and changes nothing;
//   top-k  for k <= K_p, v = y_{k-1} and K = min(K_p, number of keys whose value is >= v): every tie of the k-th value stays.
// A row with a NaN or a non-finite maximum is flagged and restated on the host.
__device__ __forceinline__ unsigned long long filter_key(float x, int i) {
    const unsigned b = x == 0.0f ? 0u : __float_as_uint(x);
    return (unsigned long long)((b & 0x80000000u) ? ~b : (b | 0x80000000u)) << 32 | (unsigned) i;
}
__device__ __forceinline__ float filter_key_value(unsigned long long k) {
    const unsigned o = (unsigned)(k >> 32);
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

template <int kThreads>
__global__ void __launch_bounds__(kThreads, 1) filter_rows_kernel(const float * __restrict__ logits, int ld, int n, int P, int top_k, int use_top_p, float top_p,
                                                               float * __restrict__ out, int32_t * __restrict__ kept, int32_t * __restrict__ flags) {
    extern __shared__ unsigned long long sk[];           // [P] keys, then [P] floats (top-p: e_j, then p_j)
    float * e = reinterpret_cast<float *>(sk + P);
    __shared__ int s_amb, s_K, s_L, s_cnt; __shared__ float s_sum;
    const int tid = threadIdx.x;
    const float * lg = logits + (size_t) blockIdx.x * ld;
    if (tid == 0) { s_amb = 0; s_cnt = 0; }
    bool amb = false;
    for (int i = tid; i < P; i += kThreads) {
        if (i < n) { const float x = __ldcg(lg + i); if (x != x) amb = true; sk[i] = filter_key(x, i); }
        else sk[i] = 0ull;                               // below every real key (the key of -inf is 0x007fffff << 32)
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < P / 2; t += kThreads) {
                const int a = 2 * t - (t & (j - 1)), b = a + j;
                const unsigned long long ka = sk[a], kb = sk[b];
                if ((a & k) == 0 ? ka < kb : ka > kb) { sk[a] = kb; sk[b] = ka; }
            }
            __syncthreads();
        }
    const float m = filter_key_value(sk[0]);
    if (!isfinite(m)) amb = true;
    int Kp = n;
    if (use_top_p) {
        for (int j = tid; j < n; j += kThreads) {
            const double y = exp((double) __fsub_rn(filter_key_value(sk[j]), m));
            if (__double2float_rn(y * (1.0 - 0x1p-50)) != __double2float_rn(y * (1.0 + 0x1p-50))) amb = true;
            e[j] = __double2float_rn(y);
        }
        __syncthreads();
        if (tid == 0) {                                  // S in sorted order, up to the first group of 8 that ends below 2^-26
            float sum = 0.0f; int j = 0; bool rest_negligible = false;
            for (; j + 8 <= n && !rest_negligible; j += 8) {
                const float4 a = *reinterpret_cast<const float4 *>(e + j), b = *reinterpret_cast<const float4 *>(e + j + 4);
                sum = __fadd_rn(sum, a.x); sum = __fadd_rn(sum, a.y); sum = __fadd_rn(sum, a.z); sum = __fadd_rn(sum, a.w);
                sum = __fadd_rn(sum, b.x); sum = __fadd_rn(sum, b.y); sum = __fadd_rn(sum, b.z); sum = __fadd_rn(sum, b.w);
                rest_negligible = b.w < 0x1p-26f;
            }
            if (!rest_negligible) for (; j < n; j++) sum = __fadd_rn(sum, e[j]);
            s_sum = sum; s_L = j;
        }
        __syncthreads();
        const float S = s_sum; const int L = s_L;
        for (int j = tid; j < L; j += kThreads) e[j] = __fdiv_rn(e[j], S);
        __syncthreads();
        if (tid == 0) {                                  // c_j in sorted order until it first exceeds top_p
            float c = 0.0f; int j = 0, cut = n;
            for (; j + 8 <= L && cut == n; j += 8) {
                const float4 a = *reinterpret_cast<const float4 *>(e + j), b = *reinterpret_cast<const float4 *>(e + j + 4);
                float cc[8];
                cc[0] = __fadd_rn(c, a.x); cc[1] = __fadd_rn(cc[0], a.y); cc[2] = __fadd_rn(cc[1], a.z); cc[3] = __fadd_rn(cc[2], a.w);
                cc[4] = __fadd_rn(cc[3], b.x); cc[5] = __fadd_rn(cc[4], b.y); cc[6] = __fadd_rn(cc[5], b.z); cc[7] = __fadd_rn(cc[6], b.w);
                if (cc[7] > top_p) {                     // c is non-decreasing: the first crossing lies in this group
#pragma unroll
                    for (int q = 7; q >= 0; q--) if (cc[q] > top_p) cut = j + q + 1;
                }
                c = cc[7];
            }
            for (; j < L && cut == n; j++) { c = __fadd_rn(c, e[j]); if (c > top_p) cut = j + 1; }
            s_K = cut;
        }
        __syncthreads();
        Kp = s_K;
    }
    int K = Kp;
    if (top_k > 0 && top_k <= Kp) {
        const unsigned ov = (unsigned)(sk[top_k - 1] >> 32);
        int cnt = 0;
        for (int j = tid; j < n; j += kThreads) cnt += (unsigned)(sk[j] >> 32) >= ov;
        atomicAdd(&s_cnt, cnt);
        __syncthreads();
        K = min(Kp, s_cnt);
    }
    if (amb) s_amb = 1;
    const unsigned long long thr = sk[K - 1];
    float * o = out + (size_t) blockIdx.x * n;
    for (int i = tid; i < n; i += kThreads) { const float x = __ldcg(lg + i); o[i] = filter_key(x, i) >= thr ? x : __int_as_float(0xff800000); }
    __syncthreads();
    if (tid == 0) { flags[blockIdx.x] = s_amb; if (kept) kept[blockIdx.x] = K; }
}

bool sampling_valid(const char * fn, const bark_b200_sampling & s) {
    if (s.top_k < 0) { fprintf(stderr, "%s: top_k %d (0 for off, or k >= 1)\n", fn, s.top_k); return false; }
    if (s.use_top_p && !(std::isfinite(s.top_p) && s.top_p >= 0.0f && s.top_p <= 1.0f)) { fprintf(stderr, "%s: top_p %g is not in [0, 1]\n", fn, (double) s.top_p); return false; }
    return true;
}

static int filter_sort_width(int n) { int P = 2; while (P < n) P <<= 1; return P; }

void filter_rows(const float * logits, int ld, int n, int rows, const bark_b200_sampling & f, float * d_out, int32_t * d_kept, int32_t * d_flags, int threads,
                 cudaStream_t s) {
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) {
        const int max_smem = kSampleMaxLogits * 12;
        BARK_CUDA_CHECK(cudaFuncSetAttribute(filter_rows_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(filter_rows_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    }
    const int P = filter_sort_width(n);
    const size_t smem = (size_t) P * (f.use_top_p ? 12 : 8);
    if (threads == 0) threads = rows == 1 ? 1024 : 256;   // as sample_rows
    g_next_bytes = (double) rows * n * 12.0;
    if (threads == 1024) BARK_LAUNCH(filter_rows_kernel<1024>, rows, 1024, smem, s, logits, ld, n, P, f.top_k, f.use_top_p, f.top_p, d_out, d_kept, d_flags);
    else                 BARK_LAUNCH(filter_rows_kernel<256>, rows, 256, smem, s, logits, ld, n, P, f.top_k, f.use_top_p, f.top_p, d_out, d_kept, d_flags);
}

// The filter on the host with libm's exp, written from the rule rather than from the kernel: stable argsort, reversed; the
// reference's softmax of the sorted row; the float cumsum; torch.topk's k-th value and "<".  NaN sorts above every number, as in numpy.
int filter_row_host(float * row, int n, const bark_b200_sampling & f) {
    std::vector<int> order((size_t) n);
    for (int i = 0; i < n; i++) order[(size_t) i] = n - 1 - i;                // descending index, then a stable sort by value
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const float x = row[a], y = row[b];
        if (std::isnan(x) || std::isnan(y)) return std::isnan(x) && !std::isnan(y);
        return x > y;
    });
    std::vector<float> z((size_t) n);
    for (int j = 0; j < n; j++) z[(size_t) j] = row[order[(size_t) j]];
    std::vector<char> removed((size_t) n, 0);
    if (f.use_top_p) {
        std::vector<float> p(z);
        float mx = -INFINITY;
        for (float v : p) mx = std::max(mx, v);
        float sum = 0.0f;
        for (float & v : p) { v = (float) exp((double)(v - mx)); sum += v; }
        float c = 0.0f;
        for (int j = 0; j < n; j++) {
            if (j > 0 && c > f.top_p) removed[(size_t) j] = 1;                // c holds c_{j-1}
            c += p[(size_t) j] / sum;
        }
        for (int j = 0; j < n; j++) if (removed[(size_t) j]) z[(size_t) j] = -INFINITY;
    }
    if (f.top_k > 0) {
        std::vector<float> t(z);
        const int kk = std::min(f.top_k, n);
        std::nth_element(t.begin(), t.begin() + (kk - 1), t.end(), [](float a, float b) { return a > b; });
        const float v = t[(size_t)(kk - 1)];
        for (int j = 0; j < n; j++) if (z[(size_t) j] < v) removed[(size_t) j] = 1;
    }
    int kept = 0;
    for (int j = 0; j < n; j++) {
        if (removed[(size_t) j]) row[order[(size_t) j]] = -INFINITY;
        else kept++;
    }
    return kept;
}

// gpt_sample with the uniform draw already made: the reference's arithmetic end to end, libstdc++'s discrete distribution restated
// (bits/random.tcc: normalise in double, sequential partial sums, last one forced to 1.0, lower_bound of the draw).
int32_t sample_token_given_u(const float * logits, int n, float temp, double u, float * eos_p) {
    std::vector<float> p(logits, logits + n);
    const float div = temp == 0.0f ? 0.7f : temp;                                 // argmax path still divides by 0.7 (quirk D.3)
    for (float & v : p) v /= div;
    float mx = -INFINITY;
    for (float v : p) mx = std::max(mx, v);
    float sum = 0.0f;
    for (float & v : p) { v = (float) exp((double)(v - mx)); sum += v; }          // reference calls the double exp() on a float argument
    for (float & v : p) v /= sum;
    if (eos_p) *eos_p = p.back();                                                 // probability of the LAST logit (quirk D.2)
    if (temp == 0.0f) {
        float best = -INFINITY; int32_t next = 0;
        for (int i = 0; i < n; i++) if (p[(size_t) i] > best) { best = p[(size_t) i]; next = i; }
        return next;
    }
    std::vector<double> cp(p.begin(), p.end());
    double tot = 0.0;
    for (double v : cp) tot += v;
    for (double & v : cp) v /= tot;
    for (size_t i = 1; i < cp.size(); i++) cp[i] += cp[i - 1];
    cp.back() = 1.0;
    return (int32_t)(std::lower_bound(cp.begin(), cp.end(), u) - cp.begin());
}

void read_back_samples(bark_context * ctx, int start, int stop, bool want_eos, bool filtered) {
    cudaStream_t s = ctx->stream;
    const size_t cnt = (size_t)(stop - start);
    if (filtered) { BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_fflags + start, ctx->d_fflags + start, cnt * 4, cudaMemcpyDeviceToHost, s)); g_d2h_bytes += cnt * 4; }
    BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_stok + start, ctx->d_stok + start, cnt * 4, cudaMemcpyDeviceToHost, s));
    BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_sflags + start, ctx->d_sflags + start, cnt * 4, cudaMemcpyDeviceToHost, s));
    if (want_eos) BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_seos + start, ctx->d_seos + start, cnt * 4, cudaMemcpyDeviceToHost, s));
    g_d2h_bytes += cnt * (want_eos ? 12 : 8);
    BARK_CUDA_CHECK(cudaStreamSynchronize(s));
}

int sample_and_replay(bark_context * ctx, const float * d_logits, int ld, int lo, int n, int rows, float temp, bool want_eos, const bark_b200_sampling * f) {
    cudaStream_t s = ctx->stream;
    if (temp != 0.0f) { BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->d_u, ctx->h_u, (size_t) rows * sizeof(double), cudaMemcpyHostToDevice, s)); g_h2d_bytes += (size_t) rows * sizeof(double); }
    const int force = ctx->debug_flag_every > 0 && (ctx->n_sample_calls++ % ctx->debug_flag_every) == 0;
    const bool filtered = f && filter_on(*f);
    if (filtered) {
        if (rows > kMaxFilterRows) throw std::logic_error("sample_and_replay: more rows than the filter workspace holds");
        filter_rows(d_logits + lo, ld, n, rows, *f, ctx->d_frow, nullptr, ctx->d_fflags, 0, s);
        sample_rows(ctx->d_frow, n, n, rows, temp, ctx->d_u, ctx->d_stok, lo, nullptr, ctx->d_seos, ctx->d_sflags, force, 0, s);
    } else {
        sample_rows(d_logits + lo, ld, n, rows, temp, ctx->d_u, ctx->d_stok, lo, nullptr, ctx->d_seos, ctx->d_sflags, force, 0, s);
    }
    read_back_samples(ctx, 0, rows, want_eos, filtered);
    int replays = 0;
    std::vector<float> row;
    for (int r = 0; r < rows; r++) if (sample_flagged(ctx, r, filtered)) {
        row.resize((size_t) n);
        BARK_CUDA_CHECK(cudaMemcpy(row.data(), d_logits + (size_t) r * ld + lo, (size_t) n * 4, cudaMemcpyDeviceToHost)); g_d2h_bytes += (size_t) n * 4;
        if (filtered) filter_row_host(row.data(), n, *f);             // the raw logits are still on the device: restate the filter from them
        ctx->h_stok[r] = lo + sample_token_given_u(row.data(), n, temp, ctx->h_u[r], want_eos ? &ctx->h_seos[r] : nullptr);
        replays++;
    }
    ctx->n_sample_host_replays += replays;
    return replays;
}

// The RNG stream advances exactly as gpt_sample would advance it: one draw per row (what the discrete distribution's operator() draws),
// none on the argmax path.
bool sample_device(bark_context * ctx, GPTModel & m, std::mt19937 & rng, const float * d_logits, int ld, int n, int rows, float temp, int32_t * out_tok, float * out_eos) {
    if (rows < 1 || rows > 1024 || n < 2 || n > kSampleMaxLogits) { fprintf(stderr, "%s: unsupported shape (%d rows of %d)\n", __func__, rows, n); return false; }
    const int64_t t0 = now_us();
    if (temp != 0.0f) for (int r = 0; r < rows; r++) ctx->h_u[r] = std::generate_canonical<double, 53>(rng);
    sample_and_replay(ctx, d_logits, ld, 0, n, rows, temp, out_eos != nullptr);
    for (int r = 0; r < rows; r++) { out_tok[r] = ctx->h_stok[r]; if (out_eos) out_eos[r] = ctx->h_seos[r]; }
    m.t_sample_us += now_us() - t0;
    m.n_sample += rows;
    return true;
}

}  // namespace bark
