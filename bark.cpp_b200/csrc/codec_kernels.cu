// EnCodec kernels (24 kHz model, up to 32 codebooks, hop 320), bit-exact path.
//
// Replaces encodec_forward_quantizer_decode (encodec.cpp/quantizer.h:78-111) and
// encodec_forward_decoder (encodec.cpp/decoder.h:43-113):
//   RVQ gather-sum -> conv k7 -> 2 x LSTM(512) + skip -> 4 x [ELU, ConvT(k=2s, s), resblock] -> ELU -> conv k7,
// and their inverse, encodec_forward_encoder (encoder.h:39-109) and encodec_forward_quantizer_encode (quantizer.h:20-76):
//   conv k7 -> 4 x [resblock, ELU, conv(k=2r, stride r)] -> 2 x LSTM(512) + skip -> ELU -> conv k7 -> RVQ nearest codeword.
// Activations are [C][T] with time contiguous (the reference's [T, C] ggml tensors).
//
// Every contraction in the reference's decoder is a ggml_vec_dot_f16 (ggml.c:2251): conv1d = im2col to f16
// (ggml.c:14892-14960) x f16 kernel, conv_transpose_1d = per-tap dots over Cin (ggml.c:14688-14699), LSTM = two
// f16 mat-vecs per step (lstm.h:55-59).  They are evaluated here in the same lane order as the GPT mat-muls
// (common.cuh), with the activation functions restated from glibc (common.cuh), so the waveform comes out
// bit-identical to the CPU reference, not merely within the 1e-3 contract.
#include "codec_kernels.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace bark {

// ------------------------------------------------------------------------------------------------
// Items of one launch, passed by value (__grid_constant__: indexed in the parameter space, never copied).  Item b reads [C][L_in[b]] at
// C * base_in[b] and writes [C'][L_out[b]] at C' * base_out[b]; base_* are prefix sums of the lengths, base_*[n] their total.  Grids are
// one flattened run of tiles: item b owns tiles [tile0[b], tile0[b+1]) of the kernel's tile size, so a launch costs the sum of the
// items' tiles, not n times the longest.  Lp: the stream kernel's padded input length.
// ------------------------------------------------------------------------------------------------
struct CodecItems {
    int n;
    int L_in[kCodecMaxItems], L_out[kCodecMaxItems], Lp[kCodecMaxItems];
    int base_in[kCodecMaxItems + 1], base_out[kCodecMaxItems + 1], tile0[kCodecMaxItems + 1];
};

// tiled[b]: the positions item b's tiles of TT cover (its input or output length, as the kernel walks them)
static CodecItems codec_items(int n, const int * L_in, const int * L_out, const int * tiled, int TT) {
    if (n < 1 || n > kCodecMaxItems) { fprintf(stderr, "bark_b200: %d codec items in one launch (1 to %d)\n", n, kCodecMaxItems); throw std::runtime_error("unsupported configuration (see the message above)"); }
    CodecItems it{};
    it.n = n;
    for (int b = 0; b < n; b++) {
        it.L_in[b] = L_in[b]; it.L_out[b] = L_out[b];
        it.base_in[b + 1] = it.base_in[b] + L_in[b]; it.base_out[b + 1] = it.base_out[b] + L_out[b];
        it.tile0[b + 1] = it.tile0[b] + (tiled[b] + TT - 1) / TT;
    }
    return it;
}

// the last b in [0, n) with a[b] <= v (a ascending, a[0] = 0): the item of a flattened tile or of a concatenated position
__device__ __forceinline__ int item_at(const int * a, int n, int v) {
    int lo = 0, hi = n - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (a[mid] <= v) lo = mid; else hi = mid - 1; }
    return lo;
}

// ------------------------------------------------------------------------------------------------
// quantizer decode: x[d][t] = sum_q embed_q[codes[q][t]][d], q = 0..n_q-1 in order onto a zeroed tensor (quantizer.h:95-106)
// ------------------------------------------------------------------------------------------------
struct Codebooks { const float * e[kMaxCodebooks]; };
__global__ void rvq_decode_kernel(Codebooks cb, const int32_t * __restrict__ codes, int n_q, int Hd, float * __restrict__ x, const __grid_constant__ CodecItems it) {
    const int b = item_at(it.tile0, it.n, blockIdx.x), T = it.L_in[b];
    const int t = (blockIdx.x - it.tile0[b]) * blockDim.x + threadIdx.x, d = blockIdx.y;
    if (t >= T) return;
    codes += (size_t) n_q * it.base_in[b]; x += (size_t) Hd * it.base_in[b];
    float acc = 0.0f;
#pragma unroll
    for (int q = 0; q < kMaxCodebooks; q++)              // constant indices: the parameter struct stays in constant memory
        if (q < n_q) acc = __fadd_rn(acc, cb.e[q][(size_t) codes[q * T + t] * Hd + d]);
    x[(size_t) d * T + t] = acc;
}

void rvq_decode(const CodecModel & cm, const int32_t * d_codes, int n_q, const int * T, int n, float * x, cudaStream_t s) {
    Codebooks cb{};
    for (int q = 0; q < n_q; q++) cb.e[q] = cm.embed[q];
    const CodecItems it = codec_items(n, T, T, T, 128);
    BARK_LAUNCH(rvq_decode_kernel, dim3(it.tile0[n], cm.hidden_dim), 128, 0, s, cb, d_codes, n_q, cm.hidden_dim, x, it);
}

// ------------------------------------------------------------------------------------------------
// quantizer encode (quantizer.h:20-76), codebooks q = 0..n_q-1 in order on the residual r (initially the latent column):
//   v_j = -(e_j + (s + fl(-2 * vec_dot_f32(Hd, embed_q[j], r)))),  s = f32(sum_double fl(r_i^2)),  e_j = f32(sum_double fl(embed_q[j][i]^2))
//   code = ggml_vec_argmax_f32(v) (ggml.c:2965-2973),  r <- r - embed_q[code]
// ------------------------------------------------------------------------------------------------
// e_j: ggml_sum_rows(ggml_sqr(embed)) = sequential double sum of the f32 squares (ggml.c:2912-2922); weights only, computed at load
__global__ void rvq_norms_kernel(const float * __restrict__ e, int n_bins, int Hd, float * __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_bins) return;
    double s = 0.0;
    for (int i = 0; i < Hd; i++) { const float v = e[(size_t) j * Hd + i]; s = __dadd_rn(s, (double) __fmul_rn(v, v)); }
    out[j] = __double2float_rn(s);
}

void rvq_norms(const float * embed, int n_bins, int Hd, float * out, cudaStream_t s) {
    BARK_LAUNCH(rvq_norms_kernel, (n_bins + 127) / 128, 128, 0, s, embed, n_bins, Hd, out);
}

// One cluster of kRvqCtas CTAs per 8 frames.  CTA r owns codewords [r*S, min((r+1)*S, n_bins)), S = ceil(n_bins / kRvqCtas), and every
// CTA keeps its own copy of the 8 residuals in shared memory through all codebooks.  Per codebook, warp w of a CTA walks its codewords
// j = lo + w, lo + w + 8, ... with lane v holding virtual lane v of the dot's chain (Hd / 32 steps), so each codeword row is read once
// per 8 frames; warp f then reduces frame f's slice to (maximum, last index holding it, NaN seen).  The CTAs exchange these through
// distributed shared memory and each combines them in the same way: the last index holding the row maximum is what the reference's
// running MAX and == select for rows without NaN.  A row with a NaN goes through the reference's loop on one lane, reading the peers'
// slices in order through DSMEM, where a NaN resets the maximum.  Every CTA then applies the same residual update.
// The values and partials are double-buffered by codebook parity, so one cluster barrier per codebook orders the writes of codebook
// q + 2 after every peer's reads of codebook q.
// The 8 frames of a cluster are consecutive positions of the items' concatenated frames, so clusters fill across items: position g is
// frame g - base[b] of item b, whose latent is [Hd][T_b] at Hd * base[b] and whose codes are [n_q][T_b] at n_q * base[b].
constexpr int kRvqFrames = 8, kRvqCtas = 8, kRvqMaxBins = 1024, kRvqMaxHidden = 128, kRvqSlice = kRvqMaxBins / kRvqCtas;
__global__ void __cluster_dims__(kRvqCtas, 1, 1) __launch_bounds__(256, 4) rvq_encode_kernel(
        const float * __restrict__ latent, Codebooks cb, Codebooks norms, int n_q, int n_bins, int Hd, int32_t * __restrict__ codes,
        const __grid_constant__ CodecItems it) {
    __shared__ float vals[2][kRvqFrames][kRvqSlice];
    __shared__ float p_max[2][kRvqFrames];
    __shared__ int p_idx[2][kRvqFrames], p_nan[2][kRvqFrames];
    __shared__ float res[kRvqFrames][kRvqMaxHidden];
    __shared__ float s_nrm[kRvqFrames];
    __shared__ int s_code[kRvqFrames];
    __shared__ int s_T[kRvqFrames], s_base[kRvqFrames], s_t[kRvqFrames];   // item length, item base, frame within the item (s_T 0: no frame)
    __shared__ const float * s_cb[kMaxCodebooks], * s_cn[kMaxCodebooks];   // indexing the parameter structs by q would copy them to the stack
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int) cluster.block_rank();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, f0 = (blockIdx.x / kRvqCtas) * kRvqFrames, nc = Hd >> 5;
    const int S = (n_bins + kRvqCtas - 1) / kRvqCtas, lo = min(rank * S, n_bins), cnt = min(n_bins - lo, S);
#pragma unroll
    for (int q = 0; q < kMaxCodebooks; q++) if (threadIdx.x == q) { s_cb[q] = cb.e[q]; s_cn[q] = norms.e[q]; }
    if (threadIdx.x < kRvqFrames) {
        const int g = f0 + threadIdx.x, b = item_at(it.base_in, it.n, g);
        const bool live = g < it.base_in[it.n];
        s_T[threadIdx.x] = live ? it.L_in[b] : 0; s_base[threadIdx.x] = it.base_in[b]; s_t[threadIdx.x] = g - it.base_in[b];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kRvqFrames * Hd; i += blockDim.x) {
        const int f = i / Hd, d = i % Hd;
        res[f][d] = s_T[f] ? latent[(size_t) Hd * s_base[f] + (size_t) d * s_T[f] + s_t[f]] : 0.f;
    }
    __syncthreads();
    for (int q = 0; q < n_q; q++) {
        const int b = q & 1;
        const float * E = s_cb[q], * nrm = s_cn[q];
        if (lane == 0) {
            double s = 0.0;
            for (int d = 0; d < Hd; d++) s = __dadd_rn(s, (double) __fmul_rn(res[warp][d], res[warp][d]));
            s_nrm[warp] = __double2float_rn(s);
        }
        __syncthreads();
        float r[kRvqFrames][kRvqMaxHidden / 32], sn[kRvqFrames];
#pragma unroll
        for (int f = 0; f < kRvqFrames; f++) {
            sn[f] = s_nrm[f];
#pragma unroll
            for (int c = 0; c < kRvqMaxHidden / 32; c++) r[f][c] = c < nc ? res[f][c * 32 + lane] : 0.f;
        }
        for (int jl = warp; jl < cnt; jl += 8) {
            const int j = lo + jl;
            float ev[kRvqMaxHidden / 32];
#pragma unroll
            for (int c = 0; c < kRvqMaxHidden / 32; c++) ev[c] = c < nc ? __ldg(E + (size_t) j * Hd + c * 32 + lane) : 0.f;
            const float ej = __ldg(nrm + j);
#pragma unroll
            for (int f = 0; f < kRvqFrames; f++) {
                float acc = 0.f;
#pragma unroll
                for (int c = 0; c < kRvqMaxHidden / 32; c++) if (c < nc) acc = __fmaf_rn(ev[c], r[f][c], acc);
                const float dot = lane_tree_reduce(acc);
                if (lane == f) vals[b][f][jl] = -__fadd_rn(ej, __fadd_rn(sn[f], __fmul_rn(dot, -2.0f)));
            }
        }
        __syncthreads();
        {   // this CTA's slice of frame `warp`
            const float * v = vals[b][warp];
            float m = -INFINITY; bool nan = false;
            for (int j = lane; j < cnt; j += 32) { const float a = v[j]; nan |= a != a; m = fmaxf(m, a); }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            int idx = -1;
            for (int j = lane; j < cnt; j += 32) if (v[j] == m) idx = lo + j;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) idx = max(idx, __shfl_xor_sync(0xffffffffu, idx, o));
            const bool any_nan = __any_sync(0xffffffffu, nan);
            if (lane == 0) { p_max[b][warp] = m; p_idx[b][warp] = idx; p_nan[b][warp] = any_nan; }
        }
        cluster.sync();                                  // every CTA's partials (and values) of codebook q are visible
        {   // lane r < kRvqCtas reads rank r's partial of frame `warp`; ranks hold ascending codeword ranges
            float m = -INFINITY; int idx = -1, nan = 0;
            if (lane < kRvqCtas) {
                m = *cluster.map_shared_rank(&p_max[b][warp], lane);
                idx = *cluster.map_shared_rank(&p_idx[b][warp], lane);
                nan = *cluster.map_shared_rank(&p_nan[b][warp], lane);
            }
            float mx = m;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            int best = lane < kRvqCtas && m == mx ? idx : -1;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
            if (__any_sync(0xffffffffu, nan) && lane == 0) {
                float run = -INFINITY; best = 0;
                for (int pr = 0; pr < kRvqCtas; pr++) {
                    const int plo = min(pr * S, n_bins), pcnt = min(n_bins - plo, S);
                    const float * pv = cluster.map_shared_rank(&vals[b][warp][0], pr);
                    for (int j = 0; j < pcnt; j++) { const float a = pv[j]; run = run > a ? run : a; if (run == a) best = plo + j; }
                }
            }
            if (lane == 0) {
                const int T = s_T[warp];
                s_code[warp] = T ? best : 0;
                if (T && rank == 0) codes[(size_t) n_q * s_base[warp] + (size_t) q * T + s_t[warp]] = best;
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < kRvqFrames * Hd; i += blockDim.x) {
            const int f = i / Hd, d = i % Hd;
            res[f][d] = __fsub_rn(res[f][d], __ldg(E + (size_t) s_code[f] * Hd + d));
        }
        __syncthreads();
    }
    cluster.sync();                                      // a CTA's shared memory must outlive its peers' last reads
}

bool rvq_encode(const float * const * embed, const float * const * norms, int n_q, int n_bins, int Hd, const float * latent, const int * T, int n,
                int32_t * codes, cudaStream_t s) {
    if (n_q < 1 || n_q > kMaxCodebooks || n_bins < 1 || n_bins > kRvqMaxBins || Hd < 32 || Hd > kRvqMaxHidden || Hd % 32) return false;
    for (int b = 0; b < n; b++) if (T[b] < 1) return false;
    Codebooks cb{}, nr{};
    for (int q = 0; q < n_q; q++) { cb.e[q] = embed[q]; nr.e[q] = norms[q]; }
    const CodecItems it = codec_items(n, T, T, T, 1);
    const int frames = it.base_in[n];
    g_next_flops = 2.0 * (double) frames * n_q * n_bins * Hd;
    BARK_LAUNCH(rvq_encode_kernel, (frames + kRvqFrames - 1) / kRvqFrames * kRvqCtas, 256, 0, s, latent, cb, nr, n_q, n_bins, Hd, codes, it);
    return true;
}

// chain of one virtual lane out of an LI16 row: up to NG groups of 8 f16 values
template <int NG>
__device__ __forceinline__ void load_chain(const __half * __restrict__ row, int lane, int ngroups, float (&w)[NG * 8]) {
#pragma unroll
    for (int g = 0; g < NG; g++) {
        if (g < ngroups) {
            const uint4 u = __ldg(reinterpret_cast<const uint4 *>(row) + g * 32 + lane);
            const __half2 * h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
            for (int i = 0; i < 4; i++) { const float2 f = __half22float2(h[i]); w[g * 8 + 2 * i] = f.x; w[g * 8 + 2 * i + 1] = f.y; }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// causal conv1d, stride 1 (ops.cpp:59-75): reflect-pad k-1 on the left (ggml.c:15589), im2col rounds the input to
// f16, y[o][t] = b[o] + vec_dot_f16(Cin*k, col[t], w[o]) with col index c*k + j.  Optional ELU on the input
// (decoder.h applies it right before most convs) and residual add on the output (decoder.h:101).
// One block: a tile of TT output positions x a chunk of output channels; the input tile sits in shared memory
// already ELU'd and f16-rounded; a warp keeps one filter's lane chains in registers and walks its positions.
// ------------------------------------------------------------------------------------------------
template <int KW, int NG>
__global__ void __launch_bounds__(256) conv1d_lane_kernel(const float * __restrict__ x, int Cin, const __half * __restrict__ w_li, int Kp,
                                                          const float * __restrict__ bias, int Cout, int o_per_block, int elu_in,
                                                          const float * __restrict__ resid, float * __restrict__ y, const __grid_constant__ CodecItems it) {
    constexpr int TT = 32;
    constexpr int S = ((TT + KW - 1) | 1);               // odd row stride: conflict-free lane -> (c, j) gathers
    extern __shared__ float xs[];                        // [Cin][S]
    const int b = item_at(it.tile0, it.n, blockIdx.x), T = it.L_in[b], t0 = (blockIdx.x - it.tile0[b]) * TT;
    x += (size_t) Cin * it.base_in[b]; y += (size_t) Cout * it.base_in[b];
    if (resid) resid += (size_t) Cout * it.base_in[b];
    for (int i = threadIdx.x; i < Cin * (TT + KW - 1); i += blockDim.x) {
        const int c = i / (TT + KW - 1), j = i % (TT + KW - 1);
        int t = t0 + j - (KW - 1);
        if (t < 0) t = -t;
        float v = 0.f;
        if (t < T) { v = x[(size_t) c * T + t]; if (elu_in) v = elu_exact(v); v = round_f16(v); }
        xs[c * S + j] = v;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int K = Cin * KW, nsteps = K >> 5, ngroups = (nsteps + 7) >> 3;
    int aoff[NG * 8];                                    // smem offset of this lane's chain elements (position-independent part)
#pragma unroll
    for (int c = 0; c < NG * 8; c++) { const int kk = c * 32 + lane; aoff[c] = (kk / KW) * S + (kk % KW); }
    const int o_lo = blockIdx.y * o_per_block, o_hi = min(Cout, o_lo + o_per_block);
    for (int o = o_lo + warp; o < o_hi; o += 8) {
        float wch[NG * 8];
        load_chain<NG>(w_li + (size_t) o * Kp, lane, ngroups, wch);
        const float bo = bias[o];
        for (int tl = 0; tl < TT; tl++) {
            const int t = t0 + tl;
            if (t >= T) break;
            float acc = 0.0f;
#pragma unroll
            for (int c = 0; c < NG * 8; c++) if (c < nsteps) acc = __fmaf_rn(wch[c], xs[aoff[c] + tl], acc);
            float r = lane_tree_reduce(acc);
            if (lane == 0) {
                if ((nsteps << 5) < K) {                                         // K % 32 leftovers: float products summed in double (ggml.c:2281-2283)
                    double sd = (double) r;
                    const __half * wrow = w_li + (size_t) o * Kp;
                    for (int kk = nsteps << 5; kk < K; kk++)
                        sd = __dadd_rn(sd, (double) __fmul_rn(__half2float(wrow[li_offset(kk, 8)]), xs[(kk / KW) * S + (kk % KW) + tl]));
                    r = __double2float_rn(sd);
                }
                r = __fadd_rn(bo, r);                                            // ops.cpp:72 add(repeat(b), dst)
                if (resid) r = __fadd_rn(r, resid[(size_t) o * T + t]);
                y[(size_t) o * T + t] = r;
            }
        }
    }
}

// SMs of the current device: the grid-shaping target of the convolutions below (results do not depend on it)
static int device_sms() {
    int dev = 0, n = 0;
    BARK_CUDA_CHECK(cudaGetDevice(&dev));
    BARK_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    return n;
}

// ------------------------------------------------------------------------------------------------
// conv1d with K = Cin*k < 32 (the encoder's initial conv, K = 7; conv_2 of the first encoder block and of the last decoder block,
// K = 16): ggml_vec_dot_f16 has no full lane step, so the whole dot is its leftover loop, f32 products summed in double from 0
// (ggml.c:2281-2283).  One thread per output position; the block stages a tile of the input (ELU'd, f16-rounded) once.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) conv1d_short_kernel(const float * __restrict__ x, int Cin, int k, const __half * __restrict__ w_li, int Kp,
                                                           const float * __restrict__ bias, int Cout, int o_per_block, int elu_in,
                                                           const float * __restrict__ resid, float * __restrict__ y, const __grid_constant__ CodecItems it) {
    constexpr int TT = 128;
    extern __shared__ float xs[];                        // [Cin][TT + k - 1]
    const int b = item_at(it.tile0, it.n, blockIdx.x), T = it.L_in[b];
    const int W = TT + k - 1, t0 = (blockIdx.x - it.tile0[b]) * TT;
    x += (size_t) Cin * it.base_in[b]; y += (size_t) Cout * it.base_in[b];
    if (resid) resid += (size_t) Cout * it.base_in[b];
    for (int i = threadIdx.x; i < Cin * W; i += blockDim.x) {
        const int c = i / W, j = i % W;
        int t = t0 + j - (k - 1);
        if (t < 0) t = -t;
        float v = 0.f;
        if (t < T) { v = x[(size_t) c * T + t]; if (elu_in) v = elu_exact(v); v = round_f16(v); }
        xs[i] = v;
    }
    __syncthreads();
    const int tl = threadIdx.x, t = t0 + tl;
    if (t >= T) return;
    const int K = Cin * k, o_lo = blockIdx.y * o_per_block, o_hi = min(Cout, o_lo + o_per_block);
    for (int o = o_lo; o < o_hi; o++) {
        const __half * wrow = w_li + (size_t) o * Kp;
        double sd = 0.0;
        for (int kk = 0; kk < K; kk++)
            sd = __dadd_rn(sd, (double) __fmul_rn(__half2float(__ldg(wrow + li_offset(kk, 8))), xs[(kk / k) * W + (kk % k) + tl]));
        float r = __fadd_rn(__ldg(bias + o), __double2float_rn(sd));                 // ops.cpp:72 add(repeat(b), dst)
        if (resid) r = __fadd_rn(r, resid[(size_t) o * T + t]);
        y[(size_t) o * T + t] = r;
    }
}

// ------------------------------------------------------------------------------------------------
// conv1d whose lane chains do not fit in registers (K = Cin*k up to 4096) and/or with a stride: the encoder's down-sampling convs
// (k = 2r, stride r) and its final conv (k 7, K = 3584).  strided_conv_1d (ops.cpp:59-75) reflect-pads k - stride on the left and
// `extra` on the right (ggml.c:15587-15588); output t reads padded positions t*stride .. t*stride + k - 1.
// One block: TT output positions x a chunk of output channels, the padded input span in shared memory (ELU'd, f16-rounded).  A warp
// owns OW output channels at a time and streams their LI16 rows 8 chain steps per 16-byte load; each lane keeps OW x TT accumulators,
// so a weight word is used TT times.  Chain order, tree and bias add are conv1d_lane_kernel's (K % 32 == 0: no leftovers).
// ------------------------------------------------------------------------------------------------
template <int KW, int STRIDE>
__global__ void __launch_bounds__(256) conv1d_stream_kernel(const float * __restrict__ x, int Cin, const __half * __restrict__ w_li,
                                                            int Kp, const float * __restrict__ bias, int Cout, int o_per_block, int elu_in, float * __restrict__ y,
                                                            const __grid_constant__ CodecItems it) {
    constexpr int TT = STRIDE >= 8 ? 8 : 16, OW = 2;
    constexpr int SPAN = (TT - 1) * STRIDE + KW, SR = SPAN | 1, PADL = KW - STRIDE;
    extern __shared__ float xs[];                        // [Cin][SR]
    const int b = item_at(it.tile0, it.n, blockIdx.x), L = it.L_in[b], Lp = it.Lp[b], Tout = it.L_out[b];
    const int t0 = (blockIdx.x - it.tile0[b]) * TT;
    x += (size_t) Cin * it.base_in[b]; y += (size_t) Cout * it.base_out[b];
    for (int i = threadIdx.x; i < Cin * SPAN; i += blockDim.x) {
        const int c = i / SPAN, u = i % SPAN, p = t0 * STRIDE + u;
        float v = 0.f;
        if (p < Lp) {
            int t = p - PADL;
            if (t < 0) t = -t;                           // reflect left (ggml.c:15587)
            if (t >= L) t = 2 * (L - 1) - t;             // reflect right (ggml.c:15588)
            v = x[(size_t) c * L + t];
            if (elu_in) v = elu_exact(v);
            v = round_f16(v);
        }
        xs[c * SR + u] = v;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nsteps = (Cin * KW) >> 5, ngroups = (nsteps + 7) >> 3;
    const int o_lo = blockIdx.y * o_per_block, o_hi = min(Cout, o_lo + o_per_block);
    for (int ob = o_lo + warp * OW; ob < o_hi; ob += 8 * OW) {
        float acc[OW][TT];
#pragma unroll
        for (int q = 0; q < OW; q++)
#pragma unroll
            for (int t = 0; t < TT; t++) acc[q][t] = 0.f;
        for (int g = 0; g < ngroups; g++) {
            float w[OW][8];
#pragma unroll
            for (int q = 0; q < OW; q++) {
                const int o = min(ob + q, o_hi - 1);    // a missing second channel repeats the first; its sums are not stored
                const uint4 u = __ldg(reinterpret_cast<const uint4 *>(w_li + (size_t) o * Kp) + g * 32 + lane);
                const __half2 * h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
                for (int i = 0; i < 4; i++) { const float2 f = __half22float2(h[i]); w[q][2 * i] = f.x; w[q][2 * i + 1] = f.y; }
            }
#pragma unroll
            for (int st = 0; st < 8; st++) {
                const int step = g * 8 + st;
                if (step < nsteps) {
                    const int kk = step * 32 + lane;
                    const float * col = xs + (kk / KW) * SR + (kk % KW);
#pragma unroll
                    for (int t = 0; t < TT; t++) {
                        const float xv = col[t * STRIDE];
#pragma unroll
                        for (int q = 0; q < OW; q++) acc[q][t] = __fmaf_rn(w[q][st], xv, acc[q][t]);
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < OW; q++) {
            float mine = 0.f;
#pragma unroll
            for (int t = 0; t < TT; t++) { const float r = lane_tree_reduce(acc[q][t]); if (lane == t) mine = r; }
            const int o = ob + q, t = t0 + lane;
            if (o < o_hi && lane < TT && t < Tout) y[(size_t) o * Tout + t] = __fadd_rn(__ldg(bias + o), mine);
        }
    }
}

// output length of strided_conv_1d (ops.cpp:8-16, 59-66): extra right padding from get_extra_padding_for_conv_1d, evaluated in
// float like the reference
static void strided_conv_lengths(int L, int k, int stride, int * Lp, int * Tout) {
    const float length = (float) L, ks = (float) k, st = (float) stride, pad_total = (float)(k - stride);
    const float n_frames = (length - ks + pad_total) / st + 1.0f;
    const int ideal_length = (int)((ceilf(n_frames) - 1.0f) * st + (ks - pad_total));
    const int extra = (int)((float) ideal_length - length);
    *Lp = L + (k - stride) + extra;
    *Tout = (*Lp - k) / stride + 1;
}

int conv1d_out_len(int L, int k, int stride) { int Lp, Tout; strided_conv_lengths(L, k, stride, &Lp, &Tout); return Tout; }

// shapes the stream kernel is instantiated for: the encoder's down-sampling convs (k = 2r, stride r) and its final conv
static int conv1d_stream(const float * x, int Cin, const int * L, int n, const ConvW & cv, int stride, bool elu_in, float * y, cudaStream_t s) {
    const int K = Cin * cv.k;
    std::vector<int> Lp((size_t) n), Tout((size_t) n);
    for (int b = 0; b < n; b++) {
        strided_conv_lengths(L[b], cv.k, stride, &Lp[b], &Tout[b]);
        // both reflections must stay inside the input: the left one reads up to k - stride past position 0, the right one `extra`
        if (K % 32 != 0 || cv.k - stride > L[b] - 1 || Lp[b] - L[b] - (cv.k - stride) > L[b] - 1) {
            fprintf(stderr, "bark_b200: unsupported conv shape Cin=%d k=%d stride=%d L=%d\n", Cin, cv.k, stride, L[b]); throw std::runtime_error("unsupported configuration (see the message above)");
        }
    }
    const int TT = stride >= 8 ? 8 : 16, SR = ((TT - 1) * stride + cv.k) | 1;
    CodecItems it = codec_items(n, L, Tout.data(), Tout.data(), TT);
    for (int b = 0; b < n; b++) it.Lp[b] = Lp[b];
    const size_t smem = (size_t) Cin * SR * sizeof(float);
    const int tiles = it.tile0[n];
    int o_per_block = cv.cout;
    const int n_sm = device_sms();
    while (o_per_block > 16 && tiles * ((cv.cout + o_per_block - 1) / o_per_block) < 2 * n_sm) o_per_block = (o_per_block + 1) / 2;
    const dim3 grid(tiles, (cv.cout + o_per_block - 1) / o_per_block);
    g_next_flops = 2.0 * (double) it.base_out[n] * cv.cout * K;
#define STREAM_CASE(KW, ST)                                                                                                  \
    if (cv.k == KW && stride == ST) {                                                                                        \
        BARK_CUDA_CHECK(cudaFuncSetAttribute(conv1d_stream_kernel<KW, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem)); \
        BARK_LAUNCH((conv1d_stream_kernel<KW, ST>), grid, 256, smem, s, x, Cin, cv.w, cv.Kp, cv.b, cv.cout, o_per_block, elu_in ? 1 : 0, y, it); \
        return kConvStream + KW * 100 + ST;                                                                                  \
    }
    STREAM_CASE(4, 2) STREAM_CASE(8, 4) STREAM_CASE(10, 5) STREAM_CASE(16, 8) STREAM_CASE(7, 1)
#undef STREAM_CASE
    fprintf(stderr, "bark_b200: unsupported conv kernel size %d with stride %d\n", cv.k, stride); throw std::runtime_error("unsupported configuration (see the message above)");
}

int conv1d(const float * x, int Cin, const int * L, int n, const ConvW & cv, bool elu_in, const float * resid, float * y, cudaStream_t s, int stride) {
    const int K = Cin * cv.k, nsteps = K / 32, ngroups = (nsteps + 7) / 8;
    if (K < 32 && stride == 1) {
        const int TT = 128;
        const CodecItems it = codec_items(n, L, L, L, TT);
        const int tiles = it.tile0[n];
        int o_per_block = cv.cout;
        const int n_sm = device_sms();
        while (o_per_block > 1 && tiles * ((cv.cout + o_per_block - 1) / o_per_block) < 4 * n_sm) o_per_block = (o_per_block + 1) / 2;
        const size_t smem = (size_t) Cin * (TT + cv.k - 1) * sizeof(float);
        g_next_flops = 2.0 * (double) it.base_in[n] * cv.cout * K;
        BARK_LAUNCH(conv1d_short_kernel, dim3(tiles, (cv.cout + o_per_block - 1) / o_per_block), TT, smem, s, x, Cin, cv.k, cv.w, cv.Kp, cv.b,
                    cv.cout, o_per_block, elu_in ? 1 : 0, resid, y, it);
        return kConvShort;
    }
    const bool lane_fits = stride == 1 && ((cv.k == 1 && ngroups <= 2) || (cv.k == 3 && ngroups <= 3) || (cv.k == 7 && ngroups <= 4));
    if (!lane_fits) {
        if (resid) { fprintf(stderr, "bark_b200: unsupported conv shape Cin=%d k=%d stride=%d with a residual\n", Cin, cv.k, stride); throw std::runtime_error("unsupported configuration (see the message above)"); }
        return conv1d_stream(x, Cin, L, n, cv, stride, elu_in, y, s);
    }
    const int TT = 32;
    const int S = (TT + cv.k - 1) | 1;
    const size_t smem = (size_t) Cin * S * sizeof(float);
    const CodecItems it = codec_items(n, L, L, L, TT);
    const int tiles = it.tile0[n];
    // enough blocks to fill the machine: split the output channels when there are few time tiles
    int o_per_block = cv.cout;
    const int n_sm = device_sms();
    while (o_per_block > 8 && tiles * ((cv.cout + o_per_block - 1) / o_per_block) < 4 * n_sm) o_per_block = (o_per_block + 1) / 2;
    const dim3 grid(tiles, (cv.cout + o_per_block - 1) / o_per_block);
    g_next_flops = 2.0 * (double) it.base_in[n] * cv.cout * K;
#define CONV_CASE(KW, NG)                                                                                                   \
    { BARK_CUDA_CHECK(cudaFuncSetAttribute(conv1d_lane_kernel<KW, NG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024)); \
      BARK_LAUNCH((conv1d_lane_kernel<KW, NG>), grid, 256, smem, s, x, Cin, cv.w, cv.Kp, cv.b, cv.cout, o_per_block, elu_in ? 1 : 0, resid, y, it); \
      return kConvLane + KW * 10 + NG; }
    if (cv.k == 1)      { if (ngroups <= 1) CONV_CASE(1, 1) else CONV_CASE(1, 2) }
    else if (cv.k == 3) { if (ngroups <= 1) CONV_CASE(3, 1) else if (ngroups <= 2) CONV_CASE(3, 2) else CONV_CASE(3, 3) }
    else if (cv.k == 7) { if (ngroups <= 1) CONV_CASE(7, 1) else CONV_CASE(7, 4) }
    else { fprintf(stderr, "bark_b200: unsupported conv kernel size %d\n", cv.k); throw std::runtime_error("unsupported configuration (see the message above)"); }
#undef CONV_CASE
}

// ------------------------------------------------------------------------------------------------
// transposed conv (ops.cpp:77-98, ggml.c:14614-14700): k = 2*stride, output right-trimmed by k - stride -> L = T*stride.
// For output sample p = t*stride + j (0 <= j < stride) the reference accumulates, in this order,
//     v1 = vec_dot_f16(Cin, f16(elu(x[:, t-1])), w[:, o, j + stride])     (skipped for t = 0)
//     v0 = vec_dot_f16(Cin, f16(elu(x[:, t])),   w[:, o, j])
// into a zeroed buffer, then adds the bias.  Weights arrive re-laid-out as rows [o][tap][Cin] in LI16.
// ------------------------------------------------------------------------------------------------
template <int NG>
__global__ void __launch_bounds__(256) convtr1d_lane_kernel(const float * __restrict__ x, int Cin, const __half * __restrict__ w_li, int Kp,
                                                            const float * __restrict__ bias, int Cout, int stride, float * __restrict__ y,
                                                            const __grid_constant__ CodecItems its) {
    constexpr int TF = 16;                               // input frames per block
    constexpr int S = TF + 1 + ((TF + 1) % 2 == 0);      // odd stride
    extern __shared__ float xs[];                        // [Cin][S]: frames t0-1 .. t0+TF-1, ELU'd, f16-rounded
    const int b = item_at(its.tile0, its.n, blockIdx.x), T = its.L_in[b], t0 = (blockIdx.x - its.tile0[b]) * TF;
    x += (size_t) Cin * its.base_in[b]; y += (size_t) Cout * its.base_out[b];
    for (int i = threadIdx.x; i < Cin * (TF + 1); i += blockDim.x) {
        const int c = i / (TF + 1), j = i % (TF + 1);
        const int t = t0 + j - 1;
        xs[c * S + j] = (t >= 0 && t < T) ? round_f16(elu_exact(x[(size_t) c * T + t])) : 0.f;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nsteps = Cin >> 5, ngroups = (nsteps + 7) >> 3;
    const int K2 = 2 * stride, L = T * stride;
    const int items = Cout * stride;                     // work items: (o, j) pairs, spread over blockIdx.y and the warps
    for (int it = blockIdx.y * 8 + warp; it < items; it += gridDim.y * 8) {
        const int o = it / stride, j = it % stride;
        float w0[NG * 8], w1[NG * 8];
        load_chain<NG>(w_li + ((size_t) o * K2 + j) * Kp, lane, ngroups, w0);
        load_chain<NG>(w_li + ((size_t) o * K2 + j + stride) * Kp, lane, ngroups, w1);
        const float bo = bias[o];
        for (int f = 0; f < TF; f++) {
            const int t = t0 + f;
            if (t >= T) break;
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int c = 0; c < NG * 8; c++) if (c < nsteps) {
                const float * col = xs + (c * 32 + lane) * S + f;
                a1 = __fmaf_rn(col[0], w1[c], a1);       // frame t-1, tap j+stride
                a0 = __fmaf_rn(col[1], w0[c], a0);       // frame t,   tap j
            }
            const float r1 = lane_tree_reduce(a1), r0 = lane_tree_reduce(a0);
            if (lane == 0) {
                float acc = 0.0f;
                if (t > 0) acc = __fadd_rn(acc, r1);
                acc = __fadd_rn(acc, r0);
                y[(size_t) o * L + (size_t) t * stride + j] = __fadd_rn(bo, acc);
            }
        }
    }
}

int convtr1d(const float * x, int Cin, const int * T, int n, const ConvW & cv, int stride, float * y, cudaStream_t s) {
    const int nsteps = Cin / 32, ngroups = (nsteps + 7) / 8;
    if (Cin % 32 != 0 || ngroups > 2 || cv.k != 2 * stride) { fprintf(stderr, "bark_b200: unsupported transposed conv Cin=%d k=%d s=%d\n", Cin, cv.k, stride); throw std::runtime_error("unsupported configuration (see the message above)"); }
    const int TF = 16, S = TF + 1 + ((TF + 1) % 2 == 0);
    const size_t smem = (size_t) Cin * S * sizeof(float);
    std::vector<int> L((size_t) n);
    for (int b = 0; b < n; b++) L[(size_t) b] = T[b] * stride;
    const CodecItems it = codec_items(n, T, L.data(), T, TF);
    const int tiles = it.tile0[n];
    int gy = (cv.cout * stride + 7) / 8;
    const int n_sm = device_sms();
    while (gy > 1 && tiles * gy > 8 * n_sm) gy = (gy + 1) / 2;
    g_next_flops = 2.0 * 2.0 * (double) it.base_out[n] * cv.cout * Cin;
    if (ngroups <= 1) BARK_LAUNCH(convtr1d_lane_kernel<1>, dim3(tiles, gy), 256, smem, s, x, Cin, cv.w, cv.Kp, cv.b, cv.cout, stride, y, it);
    else              BARK_LAUNCH(convtr1d_lane_kernel<2>, dim3(tiles, gy), 256, smem, s, x, Cin, cv.w, cv.Kp, cv.b, cv.cout, stride, y, it);
    return ngroups <= 1 ? 1 : 2;
}

// ------------------------------------------------------------------------------------------------
// LSTM (lstm.h:22-78).  Input projections for all steps at once, then the recurrence.
//   gates[t] = (W_ih f16(x_t) + b_ih) + (W_hh f16(h_{t-1}) + b_hh);  i,f,o = sigmoid, g = tanh (order i,f,g,o)
//   c = f*c + i*g;  h = o * tanh(c)
// ------------------------------------------------------------------------------------------------
// gi[t][g] = vec_dot_f16(C, w_ih[g], f16(x[:, t])) + b_ih[g];   one warp per (t, gate row) pair, weights chain reused over 8 steps
__global__ void __launch_bounds__(256) lstm_inproj_lane_kernel(const float * __restrict__ x, int C, const __half * __restrict__ wih_li, int Kp,
                                                               const float * __restrict__ bih, int G4, float * __restrict__ gi, const __grid_constant__ CodecItems it) {
    constexpr int TT = 8;
    extern __shared__ float xs[];                        // [TT][C] f16-rounded
    const int b = item_at(it.tile0, it.n, blockIdx.x), T = it.L_in[b], t0 = (blockIdx.x - it.tile0[b]) * TT;
    x += (size_t) C * it.base_in[b]; gi += (size_t) G4 * it.base_in[b];
    for (int i = threadIdx.x; i < TT * C; i += blockDim.x) {
        const int tl = i / C, c = i % C;
        xs[i] = (t0 + tl < T) ? round_f16(x[(size_t) c * T + t0 + tl]) : 0.f;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nsteps = C >> 5;                           // 16 for C = 512
    for (int g = blockIdx.y * 8 + warp; g < G4; g += gridDim.y * 8) {
        float wch[16];
        load_chain<2>(wih_li + (size_t) g * Kp, lane, (nsteps + 7) >> 3, wch);
        const float bg = bih[g];
        for (int tl = 0; tl < TT && t0 + tl < T; tl++) {
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 16; c++) if (c < nsteps) acc = __fmaf_rn(wch[c], xs[tl * C + c * 32 + lane], acc);
            const float r = lane_tree_reduce(acc);
            if (lane == 0) gi[(size_t)(t0 + tl) * G4 + g] = __fadd_rn(r, bg);
        }
    }
}

// Recurrence: persistent cooperative kernel.  CTA b owns UPB hidden units (4*UPB gate rows of W_hh, held in registers by its
// warps for the whole sequence); every step each CTA reads h_{t-1} (written by all CTAs), computes its gates, updates its
// units and publishes h_t, then all CTAs meet at a grid barrier (monotonic counter in global memory).
__device__ __forceinline__ void grid_barrier(unsigned * counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        while (*((volatile unsigned *) counter) < target) { }
        __threadfence();
    }
    __syncthreads();
}

// One sequence (every single-clip call): CTA b owns UPB hidden units; every step it reads h_{t-1}, computes its 4*UPB gates, updates its
// units and publishes h_t.  Kept beside the batched kernel below because that one, run with one item, is measurably slower per step
// (DESIGN.md §15); lstm_layer picks between them by the number of items.
template <int UPB>
__global__ void __launch_bounds__(UPB * 4 * 32) lstm_recur_one_kernel(const float * __restrict__ gi, int T, int Hn, const __half * __restrict__ whh_li, int Kp,
                                                                      const float * __restrict__ bhh, const float * __restrict__ skip,
                                                                      float * __restrict__ hbuf /*[2][Hn]*/, unsigned * __restrict__ counter, float * __restrict__ out) {
    extern __shared__ float hs[];                        // [Hn] f16-rounded h_{t-1}; then [4*UPB] gate pre-activations
    float * gates = hs + Hn;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;       // warp = local gate row: unit u = warp % UPB, gate q = warp / UPB
    const int u = warp % UPB, q = warp / UPB;
    const int unit = blockIdx.x * UPB + u;
    const int row = q * Hn + unit;
    const int G4 = 4 * Hn, nsteps = Hn >> 5;
    float wch[16];
    load_chain<2>(whh_li + (size_t) row * Kp, lane, (nsteps + 7) >> 3, wch);
    const float bg = bhh[row];
    float c_state = 0.f;                                 // kept by threads 0..UPB-1, one per unit
    for (int t = 0; t < T; t++) {
        const float * hprev = hbuf + (size_t)((t + 1) & 1) * Hn;
        for (int j = threadIdx.x; j < Hn; j += blockDim.x) hs[j] = (t == 0) ? 0.f : round_f16(__ldcg(hprev + j));
        __syncthreads();
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 16; c++) if (c < nsteps) acc = __fmaf_rn(wch[c], hs[c * 32 + lane], acc);
        const float r = lane_tree_reduce(acc);
        if (lane == 0) gates[warp] = __fadd_rn(__ldg(gi + (size_t) t * G4 + row), __fadd_rn(r, bg));     // (ih + b_ih) + (hh + b_hh)
        __syncthreads();
        if ((int) threadIdx.x < UPB) {
            const int uu = threadIdx.x, un = blockIdx.x * UPB + uu;
            const float it = sigmoid_exact(gates[0 * UPB + uu]);
            const float ft = sigmoid_exact(gates[1 * UPB + uu]);
            const float gt = glibc_tanhf_dev(gates[2 * UPB + uu]);
            const float ot = sigmoid_exact(gates[3 * UPB + uu]);
            c_state = __fadd_rn(__fmul_rn(ft, c_state), __fmul_rn(it, gt));
            const float h = __fmul_rn(ot, glibc_tanhf_dev(c_state));
            __stcg(hbuf + (size_t)(t & 1) * Hn + un, h);
            out[(size_t) un * T + t] = skip ? __fadd_rn(skip[(size_t) un * T + t], h) : h;               // decoder.h:72 inpL + out
        }
        grid_barrier(counter, (unsigned)(t + 1) * gridDim.x);
    }
}

// Several items: every step carries all B items of the launch; a warp computes its gate row's dot for each item still inside its own
// sequence (t < T_b), in that item's order and arithmetic (lstm_recur_one_kernel's), so an item's values do not depend on the others.
// The loop runs max T_b steps with one grid barrier per step; an item past its T_b neither updates nor stores.  Thread (u, b) =
// (tid % UPB, tid / UPB) keeps unit u's cell state of item b, so B <= blockDim / UPB.
template <int UPB>
__global__ void __launch_bounds__(UPB * 4 * 32) lstm_recur_kernel(const float * __restrict__ gi, int T_max, int Hn, const __half * __restrict__ whh_li, int Kp,
                                                                  const float * __restrict__ bhh, const float * __restrict__ skip,
                                                                  float * __restrict__ hbuf /*[2][B][Hn]*/, unsigned * __restrict__ counter, float * __restrict__ out,
                                                                  const __grid_constant__ CodecItems its) {
    extern __shared__ float hs[];                        // [B][Hn] f16-rounded h_{t-1} of every item; then [B][4*UPB] gate pre-activations
    __shared__ int s_T[kCodecMaxItems], s_base[kCodecMaxItems];   // the items' lengths and offsets, read every step
    const int B = its.n;
    float * gates = hs + (size_t) B * Hn;
    if ((int) threadIdx.x < B) { s_T[threadIdx.x] = its.L_in[threadIdx.x]; s_base[threadIdx.x] = its.base_in[threadIdx.x]; }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;       // warp = local gate row: unit u = warp % UPB, gate q = warp / UPB
    const int u = warp % UPB, q = warp / UPB;
    const int unit = blockIdx.x * UPB + u;
    const int row = q * Hn + unit;
    const int G4 = 4 * Hn, nsteps = Hn >> 5;
    float wch[16];
    load_chain<2>(whh_li + (size_t) row * Kp, lane, (nsteps + 7) >> 3, wch);
    const float bg = bhh[row];
    float c_state = 0.f;                                 // kept by thread (u, b) for unit u of item b
    const bool owner = (int) threadIdx.x < UPB * B;
    const int my_T = owner ? s_T[threadIdx.x / UPB] : 0, my_base = owner ? s_base[threadIdx.x / UPB] : 0;
    for (int t = 0; t < T_max; t++) {
        const float * hprev = hbuf + (size_t)((t + 1) & 1) * B * Hn;
        for (int b = 0; b < B; b++)
            if (t < s_T[b])
                for (int j = threadIdx.x; j < Hn; j += blockDim.x) hs[b * Hn + j] = (t == 0) ? 0.f : round_f16(__ldcg(hprev + (size_t) b * Hn + j));
        __syncthreads();
        for (int b = 0; b < B; b++) {
            if (t >= s_T[b]) continue;
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 16; c++) if (c < nsteps) acc = __fmaf_rn(wch[c], hs[b * Hn + c * 32 + lane], acc);
            const float r = lane_tree_reduce(acc);
            if (lane == 0)                                                                               // (ih + b_ih) + (hh + b_hh)
                gates[b * 4 * UPB + warp] = __fadd_rn(__ldg(gi + (size_t) G4 * s_base[b] + (size_t) t * G4 + row), __fadd_rn(r, bg));
        }
        __syncthreads();
        if (t < my_T) {                                  // owners only (my_T is 0 for the others)
            const int uu = threadIdx.x % UPB, b = threadIdx.x / UPB, un = blockIdx.x * UPB + uu;
            const float * g = gates + b * 4 * UPB;
            const float it = sigmoid_exact(g[0 * UPB + uu]);
            const float ft = sigmoid_exact(g[1 * UPB + uu]);
            const float gt = glibc_tanhf_dev(g[2 * UPB + uu]);
            const float ot = sigmoid_exact(g[3 * UPB + uu]);
            c_state = __fadd_rn(__fmul_rn(ft, c_state), __fmul_rn(it, gt));
            const float h = __fmul_rn(ot, glibc_tanhf_dev(c_state));
            __stcg(hbuf + (size_t)(t & 1) * B * Hn + (size_t) b * Hn + un, h);
            const size_t o = (size_t) Hn * my_base + (size_t) un * my_T + t;
            out[o] = skip ? __fadd_rn(skip[o], h) : h;                                                     // decoder.h:72 inpL + out
        }
        grid_barrier(counter, (unsigned)(t + 1) * gridDim.x);
    }
}

int lstm_layer(const float * x, int C, const int * T, int n, const __half * wih_li, const __half * whh_li, int Kp, const float * bih, const float * bhh,
               const float * skip, float * gi_scratch, float * hbuf, unsigned * counter, float * out, cudaStream_t s) {
    const int Hn = C, G4 = 4 * Hn;
    if (Hn % 32 != 0 || Hn > 512 || Hn % 4 != 0) { fprintf(stderr, "bark_b200: unsupported LSTM width %d\n", Hn); throw std::runtime_error("unsupported configuration (see the message above)"); }
    const CodecItems it = codec_items(n, T, T, T, 8);
    const int frames = it.base_in[n];
    int T_max = 0;
    for (int b = 0; b < n; b++) T_max = std::max(T_max, T[b]);
    g_next_flops = 2.0 * (double) frames * G4 * C;
    BARK_LAUNCH(lstm_inproj_lane_kernel, dim3(it.tile0[n], 32), 256, (size_t) 8 * C * sizeof(float), s, x, C, wih_li, Kp, bih, G4, gi_scratch, it);
    BARK_CUDA_CHECK(cudaMemsetAsync(counter, 0, sizeof(unsigned), s));
    constexpr int UPB = 4;
    static_assert(UPB * kCodecMaxItems <= UPB * 4 * 32, "one thread per (unit, item) holds the cell state");
    const int blocks = Hn / UPB;                         // 128 CTAs for H = 512: co-resident on the 132 SMs of an H100 (cooperative launch checks it)
    const size_t smem = (size_t) n * (Hn + 4 * UPB) * sizeof(float);
    if (g_prof_on) prof_begin("lstm_recur_kernel", s, 0.0, 2.0 * (double) frames * G4 * Hn);
    if (n == 1) {
        void * args[] = {(void *) &gi_scratch, (void *) &T_max, (void *) &Hn, (void *) &whh_li, (void *) &Kp, (void *) &bhh, (void *) &skip, (void *) &hbuf,
                         (void *) &counter, (void *) &out};
        BARK_CUDA_CHECK(cudaLaunchCooperativeKernel((const void *) lstm_recur_one_kernel<UPB>, dim3(blocks), dim3(UPB * 4 * 32), args, smem, s));
    } else {
        // The attribute belongs to the function on the device, shared by every context and thread: set once, to the largest launch
        // (kCodecMaxItems items of the widest LSTM), never per launch.
        static std::atomic<unsigned long long> configured{0};
        if (first_use_on_this_device(configured))
            BARK_CUDA_CHECK(cudaFuncSetAttribute(lstm_recur_kernel<UPB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 (int)((size_t) kCodecMaxItems * (512 + 4 * UPB) * sizeof(float))));
        void * args[] = {(void *) &gi_scratch, (void *) &T_max, (void *) &Hn, (void *) &whh_li, (void *) &Kp, (void *) &bhh, (void *) &skip, (void *) &hbuf,
                         (void *) &counter, (void *) &out, (void *) &it};
        BARK_CUDA_CHECK(cudaLaunchCooperativeKernel((const void *) lstm_recur_kernel<UPB>, dim3(blocks), dim3(UPB * 4 * 32), args, smem, s));
    }
    if (g_prof_on) prof_end(s);
    ++g_kernel_launches;
    return n == 1 ? kLstmOne : kLstmBatched;
}

// [Cin][Cout][k] (torch ConvTranspose1d layout as stored, ggml [k, Cout, Cin]) -> rows [o][tap][Cin]
__global__ void convtr_rows_kernel(const __half * __restrict__ src, __half * __restrict__ dst, int Cin, int Cout, int k) {
    const size_t total = (size_t) Cin * Cout * k;
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t) gridDim.x * blockDim.x) {
        const int c = (int)(i % Cin), j = (int)((i / Cin) % k), o = (int)(i / ((size_t) Cin * k));
        dst[i] = src[((size_t) c * Cout + o) * k + j];
    }
}
void convtr_rows(const __half * src, __half * dst, int Cin, int Cout, int k, cudaStream_t s) {
    BARK_LAUNCH(convtr_rows_kernel, 592, 256, 0, s, src, dst, Cin, Cout, k);
}

// ------------------------------------------------------------------------------------------------
// Resampling (DESIGN.md §16): torchaudio.functional.resample(u, sr, new_sr) with sinc_interp_hann, width W = 6, rolloff 0.99, on the
// down-mix u[i] = (x[i][0] + ... + x[i][C-1]) / C of upstream EnCodec's convert_audio.  Output k q + j is
//   y = (float) sum_m u[k o + m - w] h[j][m],
// a double accumulator from +0 in increasing m over phase j's nonzero f32 taps (each product is exact in double, so the fma is the
// multiply-then-add), zeros outside [0, n).  The ±0 taps left out cannot change it: the accumulator is never -0.
// ------------------------------------------------------------------------------------------------
constexpr int kResampleW = 6, kResampleTile = 256, kResampleSmemFloats = 12224;     // outputs per CTA at most; input window within 48 KB

long long resample_len(long long n, int sr, int new_sr) {
    const long long g = std::gcd(sr, new_sr), o = sr / g, q = new_sr / g;
    return (q * n + o - 1) / o;
}

std::vector<unsigned char> resample_table(int sr, int new_sr, ResampleTable * t) {
    ResampleTable r;
    r.sr = sr; r.new_sr = new_sr;
    std::vector<unsigned char> bytes;
    if (sr == new_sr) { r.tile = r.smem = kResampleTile; *t = r; return bytes; }
    const int g = std::gcd(sr, new_sr), o = sr / g, q = new_sr / g;
    const double pi = 3.141592653589793, base = std::min(o, q) * 0.99, reach = (double)(kResampleW * o) / base, scale = base / o;
    const int w = (int) std::ceil(reach);
    r.o = o; r.q = q; r.w = w;
    // h[j][m] in torchaudio's expression order (_get_sinc_resample_kernel) with the C library's sin and cos
    auto tap = [&](int j, int m) {
        double x = ((double) -j / q + (double)(m - w) / o) * base;
        x = std::min(std::max(x, (double) -kResampleW), (double) kResampleW);
        const double c = std::cos(x * pi / kResampleW / 2), win = c * c;
        x *= pi;
        const double s = x == 0 ? 1.0 : std::sin(x) / x;
        return (float)(s * (win * scale));
    };
    // Outside |x| < W every tap is the clamped sinc(±6 pi) cos^2(±pi/2), about 1e-49, so ±0 in f32: phase j's nonzero taps lie within
    // reach of its centre w + o j / q, and the candidates are that range plus one index on each side
    std::vector<int4> phase((size_t) q);
    std::vector<float> taps;
    for (int j = 0; j < q; j++) {
        const double centre = w + (double)((long long) o * j) / q;
        int lo = std::max(0, (int) std::floor(centre - reach) - 1), hi = std::min(2 * w + o - 1, (int) std::ceil(centre + reach) + 1);
        while (lo <= hi && tap(j, lo) == 0.0f) lo++;
        while (hi >= lo && tap(j, hi) == 0.0f) hi--;
        phase[(size_t) j] = make_int4(lo, std::max(hi - lo + 1, 0), (int) taps.size(), 0);
        for (int m = lo; m <= hi; m++) taps.push_back(tap(j, m));
    }
    // a CTA's window: its outputs' inputs lie within reach + 2 of o i / q
    for (r.tile = kResampleTile; ; r.tile -= 32) {
        r.smem = (int) std::ceil((r.tile - 1) * (double) o / q + 2 * reach) + 6;
        if (r.smem <= kResampleSmemFloats || r.tile == 32) break;
    }
    bytes.resize(phase.size() * sizeof(int4) + taps.size() * sizeof(float));
    memcpy(bytes.data(), phase.data(), phase.size() * sizeof(int4));
    memcpy(bytes.data() + phase.size() * sizeof(int4), taps.data(), taps.size() * sizeof(float));
    *t = r;
    return bytes;
}

void resample_bind(ResampleTable & t, const void * dev) {
    if (t.sr == t.new_sr) return;
    t.phase = (const int4 *) dev;
    t.taps = (const float *)((const int4 *) dev + t.q);
}

// One CTA per `tile` consecutive outputs.  The CTA finds the span of input its outputs read (the first input and tap count of each
// output's phase), loads it once, down-mixed, into shared memory, and each thread then sums one output over its phase's taps, which
// are read from global memory (the table stays in L2).  phase null: the identity, y = u.
__global__ void __launch_bounds__(kResampleTile) resample_kernel(const float * __restrict__ x, long long n, int C, const int4 * __restrict__ phase,
                                                                 const float * __restrict__ taps, int o, int q, int w, int tile, int L, float * __restrict__ y) {
    extern __shared__ float su[];
    __shared__ int window[2];
    const long long i0 = (long long) blockIdx.x * tile, i = i0 + threadIdx.x, k0 = i0 / q;
    const bool active = (int) threadIdx.x < tile && i < L;
    if (threadIdx.x == 0) { window[0] = INT_MAX; window[1] = INT_MIN; }
    __syncthreads();
    int4 p = make_int4(0, 1, 0, 0);
    int r = (int) threadIdx.x;                                  // output i's first input, relative to k0 o
    if (active && phase) {
        const long long k = i / q;
        p = phase[i - k * q];
        r = (int)((k - k0) * o) + p.x - w;
    }
    if (active && p.y > 0) { atomicMin(&window[0], r); atomicMax(&window[1], r + p.y); }
    __syncthreads();
    const int lo = window[0], span = window[1] - window[0];
    const long long g0 = k0 * o + lo;
    for (int s = threadIdx.x; s < span; s += blockDim.x) {
        const long long g = g0 + s;
        float v = 0.0f;
        if (g >= 0 && g < n) {
            const float * f = x + g * C;
            v = f[0];
            for (int c = 1; c < C; c++) v = __fadd_rn(v, f[c]);
            if (C > 1) v = __fdiv_rn(v, (float) C);
        }
        su[s] = v;
    }
    __syncthreads();
    if (!active) return;
    if (!phase) { y[i] = su[r - lo]; return; }
    const float * u = su + (r - lo), * h = taps + p.z;
    double acc = 0.0;
    for (int c = 0; c < p.y; c++) acc = __fma_rn((double) u[c], (double) h[c], acc);
    y[i] = __double2float_rn(acc);
}

void resample(const float * x, long long n, int C, const ResampleTable & t, float * y, int L, cudaStream_t s) {
    if (L < 1) return;
    const long long grid = ((long long) L + t.tile - 1) / t.tile;
    BARK_LAUNCH(resample_kernel, (unsigned) grid, kResampleTile, (size_t) t.smem * sizeof(float), s, x, n, C, t.phase, t.taps, t.o, t.q, t.w, t.tile, L, y);
}

}  // namespace bark
