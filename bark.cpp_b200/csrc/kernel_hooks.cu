// Kernel paths on host buffers (include/bark_b200.h), for the tests and the tools/ benchmarks: each entry point checks its arguments,
// uploads them, runs one kernel path on the default stream, waits for it and copies the result back.  None touches a bark_context.
#include "../../include/bark_b200.h"
#include "context.h"
#include "codec_kernels.h"
#include "gpt_kernels.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <optional>
#include <string>
#include <vector>

using namespace bark;

namespace {

// Every device allocation of one call, freed on every exit, including a CUDA failure thrown mid-way
struct DeviceBuffers {
    std::vector<void *> p;
    ~DeviceBuffers() { for (void * q : p) cudaFree(q); }
    template <typename T = void> T * alloc(size_t bytes) {
        p.push_back(nullptr);
        BARK_CUDA_CHECK(cudaMalloc(&p.back(), bytes));
        return (T *) p.back();
    }
    template <typename T> T * upload(const T * host, size_t bytes) {
        T * d = alloc<T>(bytes);
        BARK_CUDA_CHECK(cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice));
        return d;
    }
    template <typename T> T * poisoned(size_t bytes) {                 // 0xff bytes (-1 / NaN): a missing store shows up
        T * d = alloc<T>(bytes);
        BARK_CUDA_CHECK(cudaMemset(d, 0xff, bytes));
        return d;
    }
};

void download(void * host, const void * dev, size_t bytes) { BARK_CUDA_CHECK(cudaMemcpy(host, dev, bytes, cudaMemcpyDeviceToHost)); }

constexpr size_t kGuard = 4096;                 // bytes of kPattern on each side of a guarded output
constexpr unsigned char kPattern = 0x5a;

// `bytes` of device output between two guard bands that are checked after the kernel, so a stray store shows up.  The output starts
// as NaN, or for the RESID epilogues as the residual at `resid` (host), which the kernel adds to.
struct GuardedOutput {
    unsigned char * base; size_t bytes;
    GuardedOutput(DeviceBuffers & mem, size_t bytes, const void * resid) : base(mem.alloc<unsigned char>(bytes + 2 * kGuard)), bytes(bytes) {
        BARK_CUDA_CHECK(cudaMemset(base, kPattern, bytes + 2 * kGuard));
        if (resid) BARK_CUDA_CHECK(cudaMemcpy(base + kGuard, resid, bytes, cudaMemcpyHostToDevice));
        else       BARK_CUDA_CHECK(cudaMemset(base + kGuard, 0xff, bytes));
    }
    template <typename T> T * out() const { return (T *)(base + kGuard); }
    // copies the output to `dst` (host); false, with a message naming `fn`, when a store landed in either band
    bool read(const char * fn, void * dst) const {
        std::vector<unsigned char> h(bytes + 2 * kGuard);
        download(h.data(), base, h.size());
        memcpy(dst, h.data() + kGuard, bytes);
        for (size_t i = 0; i < kGuard; i++)
            if (h[i] != kPattern || h[kGuard + bytes + i] != kPattern) {
                fprintf(stderr, "%s: a store landed outside the output (guard band overwritten)\n", fn);
                return false;
            }
        return true;
    }
};

// After the launches: a launch the configuration rejects is thrown (the entry point's failure value); a fault while the kernels ran
// is reported under `fn`.  True when the call's work completed.
bool finish(const char * fn) {
    BARK_CUDA_CHECK(cudaGetLastError());
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) fprintf(stderr, "%s: %s\n", fn, cudaGetErrorString(e));
    return e == cudaSuccess;
}

// Every padding element of a permuted mat-mul operand -> NaN (all bits set: NaN in f16 and in f32), so a kernel that folds one into a
// stored sum returns NaN.  gm: the group-major layout of group stride gs (row capacity * 128), padding = rows >= rows or columns >= K;
// else the row-major LI layout of rows of gs = Kp elements, padding = columns >= K.
template <typename U>               // U: the element's bits, uint16_t (f16) or uint32_t (f32)
__global__ void poison_padding_kernel(U * p, size_t total, size_t gs, int rows, int K, bool gm) {
    constexpr int G = 16 / sizeof(U);
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t) gridDim.x * blockDim.x) {
        int r = 0, k;
        if (gm) { const int w = (int)(i % kGmGroup); r = (int)(i % gs / kGmGroup); k = (int)(i / gs) * kGmGroup + (w & 3) * 32 + (w >> 2); }
        else    { const int j = (int)(i % gs), e = j % G, gv = j / G; k = ((gv / 32) * G + e) * 32 + gv % 32; }     // as permute_to_li_kernel
        if (r >= rows || k >= K) p[i] = (U) ~0u;
    }
}

void poison_padding(void * p, size_t es, size_t total, size_t gs, int rows, int K, bool gm) {
    if (es == 2) BARK_LAUNCH(poison_padding_kernel<uint16_t>, 1184, 256, 0, 0, (uint16_t *) p, total, gs, rows, K, gm);
    else         BARK_LAUNCH(poison_padding_kernel<uint32_t>, 1184, 256, 0, 0, (uint32_t *) p, total, gs, rows, K, gm);
}

// One device function of common.cuh on the floats of bit patterns lo + i * stride (mod 2^32), i < count, generated here: the device
// libm against the host's (tests/test_codec_kernels_gpu.py).  fn: the DeviceMathFn order of bark_b200_device_math.
__global__ void device_math_kernel(int fn, uint32_t lo, uint32_t stride, uint32_t count, float * out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const float x = __uint_as_float(lo + i * stride);
        float r;
        switch (fn) {
        case 0:  r = glibc_expm1f_dev(x); break;
        case 1:  r = glibc_tanhf_dev(x); break;
        case 2:  r = glibc_expf_dev(x); break;
        case 3:  r = ggml_v_expf_dev(x); break;
        case 4:  r = elu_exact(x); break;
        case 5:  r = sigmoid_exact(x); break;
        default: r = round_f16(x); break;
        }
        out[i] = r;
    }
}

// the loader's re-layout of an f16 weight of `rows` rows of K (loader.cu): LI rows of li_padded_k(K, 2), every padding element NaN
__half * li_weight(DeviceBuffers & mem, const __half * d_rows, int rows, int K, int * Kp) {
    *Kp = li_padded_k(K, 2);
    __half * li = mem.alloc<__half>((size_t) rows * *Kp * 2);
    permute_to_li(d_rows, li, rows, K, W_F16, 0);
    poison_padding(li, 2, (size_t) rows * *Kp, *Kp, rows, K, false);
    return li;
}

// n item lengths of a codec hook: 1 to kCodecMaxItems items, each at least `min_len`; their sum through `total`
bool codec_lengths(const char * fn, const int * L, int n, int min_len, size_t * total) {
    if (!L || n < 1 || n > kCodecMaxItems) { fprintf(stderr, "%s: %d items (1 to %d)\n", fn, n, kCodecMaxItems); return false; }
    *total = 0;
    for (int b = 0; b < n; b++) {
        if (L[b] < min_len) { fprintf(stderr, "%s: item %d has length %d (at least %d)\n", fn, b, L[b], min_len); return false; }
        *total += (size_t) L[b];
    }
    return true;
}

// a group-major operand of group stride gs (host) -> row-major [M][N] elements of es bytes
void gm_to_rows(const unsigned char * gm, void * dst, int M, int N, size_t gs, size_t es) {
    for (int m = 0; m < M; m++)
        for (int k = 0; k < N; k++) memcpy((unsigned char *) dst + ((size_t) m * N + k) * es, gm + gm_offset(m, k, gs) * es, es);
}

int sm_count() {
    int dev = 0, n_sm = 0;
    BARK_CUDA_CHECK(cudaGetDevice(&dev)); BARK_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    return n_sm;
}

// The epilogue of a parity-path or quantised mat-mul into `out`: rows [M][N] (STORE / RESID), Q, K and V blocks of [M][N/3] (QKV), or
// GELU through gelu_tab (host, 65536 f16) into the next mat-mul's operand of type act_wt and group stride act_Kp (GELU_ACT).
MatmulEpilogue matmul_epilogue(DeviceBuffers & mem, int mode, float * out, int M, int N, const uint16_t * gelu_tab, int act_wt, int act_Kp) {
    MatmulEpilogue ep; ep.mode = mode;
    if (mode == EPI_STORE || mode == EPI_RESID) { ep.out = out; ep.ldo = N; }
    else if (mode == EPI_QKV) { const int E = N / 3; ep.out = out; ep.k_out = out + (size_t) M * E; ep.v_out = out + 2 * (size_t) M * E; ep.ldo = E; }
    else { ep.act_out = out; ep.act_wt = act_wt; ep.act_Kp = act_Kp; ep.gelu_tab = mem.upload((const __half *) gelu_tab, 65536 * 2); }
    return ep;
}

// The device filter and sampler on host rows with the uniforms given: filter_rows_kernel when the filter is on, then
// sample_rows_kernel at the instantiation asked for, then every row either kernel flags replayed on the host from the raw logits
// (filter_row_host, sample_token_given_u), as sample_and_replay does it.  device_tokens keeps the sampler's tokens before the replay;
// flags has bit 0 for the sampler and bit 1 for the filter; kept (may be null) gets the logits the filter kept, n without a filter.
int sample_given_u(const char * fn, const float * logits, int n, int rows, float temp, const bark_b200_sampling * s, const double * u, int threads,
                   int32_t * tokens, int32_t * device_tokens, int32_t * flags, float * eos_p, int32_t * kept) {
    if (!logits || !tokens || !device_tokens || !flags || !eos_p || (temp != 0.0f && !u)) return -1;
    if (n < 2 || n > kSampleMaxLogits || rows < 1 || rows > 1024 || !std::isfinite(temp) || temp < 0.0f) return -1;
    if (threads != 0 && threads != 256 && threads != 1024) return -1;
    if (temp != 0.0f) for (int r = 0; r < rows; r++) if (!(u[r] >= 0.0 && u[r] < 1.0)) return -1;
    const bark_b200_sampling f = s ? *s : bark_b200_sampling{0, 0, 1.0f};
    if (!sampling_valid(fn, f)) return -1;
    const bool filtered = filter_on(f);
    DeviceBuffers mem;
    const size_t bytes = (size_t) rows * n * 4, rb = (size_t) rows * 4;
    const float * dl = mem.upload(logits, bytes);
    const double * du = temp != 0.0f ? mem.upload(u, (size_t) rows * sizeof(double)) : nullptr;
    int32_t * dtok = mem.poisoned<int32_t>(rb), * dsflags = mem.poisoned<int32_t>(rb);
    float * deos = mem.poisoned<float>(rb);
    float * dfilt = nullptr; int32_t * dkept = nullptr, * dfflags = nullptr;
    if (filtered) {
        dfilt = mem.alloc<float>(bytes); dkept = mem.poisoned<int32_t>(rb); dfflags = mem.poisoned<int32_t>(rb);
        filter_rows(dl, n, n, rows, f, dfilt, dkept, dfflags, threads, 0);
    }
    sample_rows(filtered ? dfilt : dl, n, n, rows, temp, du, dtok, 0, nullptr, deos, dsflags, 0, threads, 0);
    if (!finish(fn)) return -1;
    std::vector<int32_t> ff((size_t) rows, 0);
    download(device_tokens, dtok, rb); download(flags, dsflags, rb); download(eos_p, deos, rb);
    if (filtered) download(ff.data(), dfflags, rb);
    if (kept && filtered) download(kept, dkept, rb);
    else if (kept) std::fill(kept, kept + rows, n);
    int replays = 0;
    std::vector<float> row;
    for (int r = 0; r < rows; r++) {
        tokens[r] = device_tokens[r];
        flags[r] = (flags[r] ? 1 : 0) | (ff[(size_t) r] ? 2 : 0);
        if (!flags[r]) continue;
        row.assign(logits + (size_t) r * n, logits + (size_t) (r + 1) * n);
        if (filtered) filter_row_host(row.data(), n, f);
        tokens[r] = sample_token_given_u(row.data(), n, temp, temp != 0.0f ? u[r] : 0.0, &eos_p[r]);
        replays++;
    }
    return replays;
}

}  // namespace

// the RVQ encode kernel: norms from rvq_norms_kernel, codes [n_q][T] from rvq_encode_kernel
extern "C" int bark_b200_rvq_encode(const float * latent, int T, const float * codebooks, int hidden, int n_bins, int n_q, int32_t * codes) {
    return guarded(0, [&] {
        if (!latent || !codebooks || !codes || T < 1 || hidden < 32 || hidden > 128 || hidden % 32 || n_bins < 1 || n_bins > 1024 || n_q < 1 || n_q > kMaxCodebooks) return 0;
        DeviceBuffers mem;
        const size_t n_cw = (size_t) n_q * n_bins;
        const float * dl = mem.upload(latent, (size_t) hidden * T * 4), * dcb = mem.upload(codebooks, n_cw * hidden * 4);
        float * dn = mem.alloc<float>(n_cw * 4);
        int32_t * dc = mem.poisoned<int32_t>((size_t) n_q * T * 4);
        const float * emb[kMaxCodebooks], * nrm[kMaxCodebooks];
        for (int q = 0; q < n_q; q++) {
            emb[q] = dcb + (size_t) q * n_bins * hidden; nrm[q] = dn + (size_t) q * n_bins;
            rvq_norms(emb[q], n_bins, hidden, dn + (size_t) q * n_bins, 0);
        }
        if (!rvq_encode(emb, nrm, n_q, n_bins, hidden, dl, &T, 1, dc, 0) || !finish("bark_b200_rvq_encode")) return 0;
        download(codes, dc, (size_t) n_q * T * 4);
        return 1;
    });
}

// resample_kernel on interleaved host frames, its taps table built as the codec scratch builds it; L samples to out
extern "C" int bark_b200_resample(const float * in, int n_frames, int channels, int in_rate, int out_rate, float * out, int cap) {
    return guarded(-1, [&] {
        const char * fn = "bark_b200_resample";
        if (!in) { fprintf(stderr, "%s: null input\n", fn); return -1; }
        if (!resample_input_ok(fn, "", in, n_frames, channels, in_rate)) return -1;
        if (out_rate < kResampleMinRate || out_rate > kResampleMaxRate) { fprintf(stderr, "%s: output rate %d Hz (%d to %d)\n", fn, out_rate, kResampleMinRate, kResampleMaxRate); return -1; }
        const long long L = resample_len(n_frames, in_rate, out_rate);
        if (L > INT_MAX) { fprintf(stderr, "%s: %lld output samples (at most 2^31 - 1)\n", fn, L); return -1; }
        if (!out) return (int) L;
        if (cap < L) { fprintf(stderr, "%s: output capacity %d for %lld samples\n", fn, cap, L); return -1; }
        ResampleTable t;
        const std::vector<unsigned char> bytes = resample_table(in_rate, out_rate, &t);
        DeviceBuffers mem;
        if (!bytes.empty()) resample_bind(t, mem.upload(bytes.data(), bytes.size()));
        const float * d_in = mem.upload(in, (size_t) n_frames * channels * sizeof(float));
        const GuardedOutput y(mem, (size_t) L * sizeof(float), nullptr);
        resample(d_in, n_frames, channels, t, y.out<float>(), (int) L, 0);
        if (!finish(fn) || !y.read(fn, out)) return -1;
        return (int) L;
    });
}

// fast mode: C = A[M][K] W[N][K]^T through one of the fine pass's GEMM epilogues, and attention over [n][E] f16 q / k / v
extern "C" int bark_b200_fast_gemm(const uint16_t * A, const uint16_t * W, void * C, int M, int N, int K, int epilogue, int bn) {
    return guarded(0, [&] {
        if (!A || !W || !C || M < 1 || N < 1 || K < 64 || K % 64) return 0;
        if (epilogue != FEPI_F32 && epilogue != FEPI_RESID && epilogue != FEPI_GELU16 && epilogue != FEPI_QKV16) return 0;
        if (epilogue == FEPI_QKV16 && N % 6) return 0;
        DeviceBuffers mem;
        const __half * dA = mem.upload((const __half *) A, (size_t) M * K * 2), * dW = mem.upload((const __half *) W, (size_t) N * K * 2);
        const bool qkv = epilogue == FEPI_QKV16;
        // output regions in the order they are laid out in C: [M][N] f32 or f16; QKV16: Q|K [M][2N/3] f16, then V^T [N/3][M] f16
        const GuardedOutput c(mem, qkv ? (size_t) M * (2 * N / 3) * 2 : (size_t) M * N * (epilogue == FEPI_GELU16 ? 2 : 4), epilogue == FEPI_RESID ? C : nullptr);
        std::optional<GuardedOutput> vt;
        FastEpi ep; ep.mode = epilogue; ep.ldo = N;
        if (epilogue == FEPI_F32 || epilogue == FEPI_RESID) ep.out32 = c.out<float>();
        else                                                ep.out16 = c.out<__half>();
        if (qkv) {                                                     // the fine pass's arguments
            vt.emplace(mem, (size_t) M * (N / 3) * 2, nullptr);
            ep.ldo = 2 * N / 3; ep.vt = vt->out<__half>(); ep.vt_ld = M; ep.v_col0 = 2 * N / 3;
        }
        const int ran = fast_gemm(dA, K, dW, K, M, N, K, ep, sm_count(), bn, 0);
        if (!finish("bark_b200_fast_gemm") || !ran) return 0;
        if (!c.read("bark_b200_fast_gemm", C) || (vt && !vt->read("bark_b200_fast_gemm", (unsigned char *) C + c.bytes))) return -1;
        return ran;
    });
}

// fast mode's weight conversion: W [n_out][K] in the file's type (f32, or the blocks of a quantised type) -> f16 [n_out][K]
extern "C" int bark_b200_fast_convert(int wtype, const void * src, int n_out, int K, uint16_t * dst, int * non_finite) {
    return guarded(0, [&] {
        const WType t = (WType) wtype;
        if (!src || !dst || !non_finite || n_out < 1 || K < 32 || K % 32 || (t != W_F32 && t != W_Q4_0 && !qx_supported(t))) return 0;
        const size_t n = (size_t) n_out * K;
        DeviceBuffers mem;
        const void * d_src = mem.upload((const unsigned char *) src, t == W_F32 ? n * 4 : n / 32 * (t == W_Q4_0 ? 18 : qx_block_bytes(t)));
        int * d_count = mem.alloc<int>(sizeof(int));
        BARK_CUDA_CHECK(cudaMemset(d_count, 0, sizeof(int)));
        const GuardedOutput c(mem, n * 2, nullptr);
        fast_convert(d_src, t, n_out, K, c.out<__half>(), d_count, 0);
        if (!finish("bark_b200_fast_convert")) return 0;
        if (!c.read("bark_b200_fast_convert", dst)) return -1;
        download(non_finite, d_count, sizeof(int));
        return 1;
    });
}

extern "C" int bark_b200_fast_attention(const uint16_t * q, const uint16_t * k, const uint16_t * v, uint16_t * out, int n, int E, int H) {
    return guarded(0, [&] {
        if (!q || !k || !v || !out || n < 128 || n % 128 || E != H * 64) return 0;
        std::vector<uint16_t> qk((size_t) n * 2 * E), vt((size_t) E * n);
        for (int r = 0; r < n; r++) {
            memcpy(&qk[(size_t) r * 2 * E], q + (size_t) r * E, (size_t) E * 2); memcpy(&qk[(size_t) r * 2 * E + E], k + (size_t) r * E, (size_t) E * 2);
            for (int c = 0; c < E; c++) vt[(size_t) c * n + r] = v[(size_t) r * E + c];
        }
        DeviceBuffers mem;
        const __half * dqk = mem.upload((const __half *) qk.data(), qk.size() * 2), * dvt = mem.upload((const __half *) vt.data(), vt.size() * 2);
        __half * dout = mem.alloc<__half>((size_t) n * E * 2);
        const bool ok = fast_attention(dqk, 2 * E, E, dvt, n, E, H, dout, 0);
        if (!finish("bark_b200_fast_attention") || !ok) return 0;
        download(out, dout, (size_t) n * E * 2);
        return 1;
    });
}

// parity-path attention on f32 rows (tools/attn_bench.py too): the result is written as f32 rows [N][E], the operand form store_act
// produces for quantised weights.  path: 0 = as attention() chooses for this shape, 1 = attn_fused_kernel, 2 = three kernels.
extern "C" int bark_b200_parity_attention(const float * q, const float * k, const float * v, float * out, int N, int n_kv, int n_past, int E, int H, int causal,
                                          int path) {
    return guarded(0, [&] {
        if (!q || !k || !v || !out || N < 1 || n_kv < 1 || n_kv > 1024 || n_past < 0 || H < 1 || E % H || path < 0 || path > 2) return 0;
        const int D = E / H;
        if (D % 32 || D > 128) return 0;
        // the three kernels' row limit is the score buffer's, which this call sizes itself
        if (path == ATTN_TILED && N > attn_tiled_max_rows(H, sm_count())) return 0;
        DeviceBuffers mem;
        const size_t q_bytes = (size_t) N * E * 4, kv_bytes = (size_t) n_kv * E * 4;
        const float * dq = mem.upload(q, q_bytes), * dk = mem.upload(k, kv_bytes), * dv = mem.upload(v, kv_bytes);
        float * dout = mem.poisoned<float>(q_bytes), * dsc = mem.alloc<float>((size_t) H * N * n_kv * 4);
        attention(dq, dk, dv, N, n_kv, n_past, E, H, causal != 0, dsc, dout, W_Q4_0, E, 0, (AttnPath) path);
        if (!finish("bark_b200_parity_attention")) return 0;
        download(out, dout, q_bytes);
        return 1;
    });
}

// the batched decode step's attention, called as SlotKV::attend calls it (max_kv = the largest pos + 1): row b's query, new K and V rows
// are q / k_new / v_new [b] (ws.q, ws.kbuf, ws.vbuf), its cache [cap][E] at k_cache / v_cache + b * cap * E.  Each cache is its own
// guarded allocation whose rows from pos[b] on are NaN before the launch, so a key or value read before the append or from a wrong row
// shows up, and so does a missing append; the scores start as NaN too.  act: the operand format of the result, 0 f32 rows (quantised
// c_proj), 1 f16 / 2 f32 group-major at row capacity B; it comes back row-major [B][E].
extern "C" int bark_b200_batch_attention(const float * q, const float * k_new, const float * v_new, float * k_cache, float * v_cache, const int32_t * pos,
                                         int B, int cap, int E, int H, int act, void * out) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_batch_attention";
        if (!q || !k_new || !v_new || !k_cache || !v_cache || !pos || !out || B < 1 || B > 8 || cap < 1 || cap > 1024 || H < 1 || E % H) return 0;
        const int D = E / H;
        if ((D != 32 && D != 64 && D != 96 && D != 128) || act < 0 || act > 2) return 0;
        int max_kv = 0;
        for (int b = 0; b < B; b++) {
            if (pos[b] < 0 || pos[b] >= cap) return 0;
            max_kv = std::max(max_kv, pos[b] + 1);
        }
        DeviceBuffers mem;
        const size_t row = (size_t) E * 4, slab = (size_t) cap * E;
        const float * dq = mem.upload(q, B * row), * dk = mem.upload(k_new, B * row), * dv = mem.upload(v_new, B * row);
        const int32_t * d_pos = mem.upload(pos, (size_t) B * sizeof(int32_t));
        std::vector<GuardedOutput> kc, vc;
        BatchKV kv{};
        for (int b = 0; b < B; b++) {
            kc.emplace_back(mem, slab * 4, k_cache + b * slab); vc.emplace_back(mem, slab * 4, v_cache + b * slab);
            kv.k[b] = kc[b].out<float>(); kv.v[b] = vc[b].out<float>();
            BARK_CUDA_CHECK(cudaMemset(kv.k[b] + (size_t) pos[b] * E, 0xff, (cap - pos[b]) * row));
            BARK_CUDA_CHECK(cudaMemset(kv.v[b] + (size_t) pos[b] * E, 0xff, (cap - pos[b]) * row));
        }
        float * scores = mem.poisoned<float>((size_t) B * H * max_kv * 4);
        const WType wt = act == 0 ? W_Q4_0 : act == 1 ? W_F16 : W_F32;
        const size_t es = act == 1 ? 2 : 4, gs = act == 0 ? (size_t) E : (size_t) B * kGmGroup;
        const GuardedOutput o(mem, act == 0 ? B * row : gm_groups(E) * gs * es, nullptr);
        attention_batch(dq, dk, dv, kv, d_pos, B, max_kv, E, H, scores, o.out<void>(), wt, (int) gs, 0);
        if (!finish(fn)) return 0;
        bool clean = true;
        for (int b = 0; b < B; b++) clean = kc[b].read(fn, k_cache + b * slab) && vc[b].read(fn, v_cache + b * slab) && clean;
        std::vector<unsigned char> h(act == 0 ? 0 : o.bytes);
        clean = o.read(fn, act == 0 ? out : h.data()) && clean;
        if (act != 0) gm_to_rows(h.data(), out, B, E, gs, es);
        return clean ? 1 : -1;
    });
}

// the parity path's row reductions: op 0 LayerNorm, op 1 soft_max; impl 0 the multi-row kernels (layernorm_act_kernel writing plain
// f32 rows, softmax_row), impl 1 the decode kernels' block_layernorm / softmax_exp_rcp
extern "C" int bark_b200_parity_rows(int op, int impl, const float * x, int rows, int n, const float * g, const float * b, float * out, unsigned * replays) {
    return guarded(0, [&] {
        if (!x || !out || !replays || op < 0 || op > 1 || impl < 0 || impl > 1 || rows < 1 || n < 1 || n > 1024 || (op == 0 && !g)) return 0;
        DeviceBuffers mem;
        const size_t bytes = (size_t) rows * n * 4;
        const float * dx = mem.upload(x, bytes);
        const float * dg = op == 0 ? mem.upload(g, (size_t) n * 4) : nullptr, * db = op == 0 && b ? mem.upload(b, (size_t) n * 4) : nullptr;
        float * dout = mem.poisoned<float>(bytes);
        unsigned * dcnt = mem.alloc<unsigned>(2 * sizeof(unsigned));
        BARK_CUDA_CHECK(cudaMemset(dcnt, 0, 2 * sizeof(unsigned)));
        if (impl == 1)    decode_rows(op, dx, rows, n, dg, db, dout, dcnt, 0);
        else if (op == 0) layernorm_act(dx, rows, n, dg, db, dout, W_Q4_0, n, dcnt, 0);
        else {            BARK_CUDA_CHECK(cudaMemcpy(dout, dx, bytes, cudaMemcpyDeviceToDevice)); softmax_rows(dout, rows, n, dcnt, 0); }
        if (!finish("bark_b200_parity_rows")) return 0;
        unsigned cnt[2];
        download(cnt, dcnt, sizeof(cnt));
        download(out, dout, bytes);
        *replays = cnt[0] + cnt[1];
        return 1;
    });
}

// the device sampler, without and with the top-k / top-p filter (sample_given_u above)
extern "C" int bark_b200_sample_given_u(const float * logits, int n, int rows, float temp, const double * u, int threads, int32_t * tokens,
                                        int32_t * device_tokens, int32_t * flags, float * eos_p) {
    return guarded(-1, [&] {
        return sample_given_u("bark_b200_sample_given_u", logits, n, rows, temp, nullptr, u, threads, tokens, device_tokens, flags, eos_p, nullptr);
    });
}
extern "C" int bark_b200_sample_filtered_given_u(const float * logits, int n, int rows, float temp, const struct bark_b200_sampling * s, const double * u,
                                                 int threads, int32_t * tokens, int32_t * device_tokens, int32_t * flags, float * eos_p, int32_t * kept) {
    return guarded(-1, [&] {
        return sample_given_u("bark_b200_sample_filtered_given_u", logits, n, rows, temp, s, u, threads, tokens, device_tokens, flags, eos_p, kept);
    });
}

// parity-path dense mat-muls (tools/gemm_bench.py too): A [M][K] and W [N][K] go through permute_to_gm, as the loader and the activation
// writers lay them out (row capacity and o_pad rounded up to the tallest / widest tile), and for the few-row kernel W also through
// permute_to_li, as the loader lays out its row-major copy; every padding element of both is NaN.  The result comes back row-major.
extern "C" int bark_b200_parity_gemm(const void * A, const void * W, void * C, int M, int N, int K, int wtype, int epilogue, int variant,
                                     const uint16_t * gelu_tab) {
    return guarded(0, [&] {
        if (!A || !W || !C || M < 1 || N < 1 || K < 32 || K % 32 || (wtype != W_F32 && wtype != W_F16) || variant < 0) return 0;
        if (epilogue < EPI_STORE || epilogue > EPI_QKV || (epilogue == EPI_QKV && N % 3) || (epilogue == EPI_GELU_ACT && !gelu_tab)) return 0;
        const size_t es = wtype == W_F16 ? 2 : 4;
        const int rows_cap = (M + 31) / 32 * 32, o_pad = (N + kGemmOPad - 1) / kGemmOPad * kGemmOPad;
        const size_t gs = (size_t) rows_cap * kGmGroup, w_gs = (size_t) o_pad * kGmGroup;
        DeviceBuffers mem;
        void * d_a = mem.alloc(gm_groups(K) * gs * es), * d_w = mem.alloc(gm_groups(K) * w_gs * es);
        const void * d_w_rows = mem.upload(W, (size_t) N * K * es);
        permute_to_gm(mem.upload(A, (size_t) M * K * es), d_a, M, rows_cap, K, (WType) wtype, 0);
        permute_to_gm(d_w_rows, d_w, N, o_pad, K, (WType) wtype, 0);
        poison_padding(d_a, es, gm_groups(K) * gs, gs, M, K, true);
        poison_padding(d_w, es, gm_groups(K) * w_gs, w_gs, N, K, true);
        DMat dm; dm.n_out = N; dm.K = K; dm.type = (WType) wtype; dm.p_gm = d_w; dm.o_pad = o_pad;
        if (variant == 0 || variant == kLaneRowsVariant) {
            dm.Kp = li_padded_k(K, (int) es); dm.p = mem.alloc((size_t) N * dm.Kp * es);
            permute_to_li(d_w_rows, dm.p, N, K, (WType) wtype, 0);
            poison_padding(dm.p, es, (size_t) N * dm.Kp, dm.Kp, N, K, false);
        }
        // output: STORE / RESID / QKV f32 [M][N] (QKV: Q, K, V blocks of [M][N/3] each); GELU_ACT: the group-major operand of the next mul_mat
        const bool gm = epilogue == EPI_GELU_ACT;
        const GuardedOutput c(mem, gm ? gm_groups(N) * gs * es : (size_t) M * N * 4, epilogue == EPI_RESID ? C : nullptr);
        const MatmulEpilogue ep = matmul_epilogue(mem, epilogue, c.out<float>(), M, N, gelu_tab, wtype, (int) gs);
        int ran;
        if (variant == 0)                     ran = lane_matmul(dm, d_a, (int) gs, M, ep, nullptr, 0);
        else if (variant == kLaneRowsVariant) { lane_matmul_rows(dm, d_a, (int) gs, M, ep, 0); ran = kLaneRowsVariant; }
        else                                  ran = lane_gemm_tiled(dm, d_a, (int) gs, M, ep, 0, variant);
        if (!finish("bark_b200_parity_gemm") || !ran) return 0;
        std::vector<unsigned char> h(gm ? c.bytes : 0);
        if (!c.read("bark_b200_parity_gemm", gm ? h.data() : C)) return -1;
        if (gm) gm_to_rows(h.data(), C, M, N, gs, es);
        return ran;
    });
}

// quantised mat-muls: the weight rows arrive as the file's blocks and go through the loader's split (q4_split / qx_split); the
// activation rows are f32, as store_act leaves them for a quantised model.  The q8 operand lives in this call's own scratch.
extern "C" int bark_b200_quant_matmul(int wtype, const void * W, const float * A, float * C, int M, int N, int K, int epilogue, int path,
                                      const uint16_t * gelu_tab, int8_t * q_out, float * d_out, float * s_out) {
    return guarded(0, [&] {
        const WType t = (WType) wtype;
        if (!W || !A || !C || M < 1 || N < 1 || K < 32 || K % 32 || (t != W_Q4_0 && !qx_supported(t)) || path < 0 || path > 2) return 0;
        if (epilogue < EPI_STORE || epilogue > EPI_QKV || (epilogue == EPI_QKV && N % 3) || (epilogue == EPI_GELU_ACT && !gelu_tab)) return 0;
        const bool q81 = t == W_Q4_1 || t == W_Q5_1;
        if ((path != 0 && (t != W_Q4_0 || M != 1 || K > 4096)) || (s_out && !q81)) return 0;
        const int nb = K / 32;
        const size_t n_blocks = (size_t) N * nb;
        DeviceBuffers mem;
        const void * d_raw = mem.upload(W, n_blocks * (t == W_Q4_0 ? 18 : qx_block_bytes(t)));
        DMat dm; dm.n_out = N; dm.K = K; dm.Kp = K; dm.type = t; dm.p = mem.alloc(n_blocks * (t == W_Q8_0 ? 32 : 16)); dm.scales = mem.alloc(n_blocks * 2);
        if (t == W_Q4_0) q4_split(d_raw, n_blocks, dm.p, dm.scales, 0);
        else {
            dm.mins = mem.alloc(n_blocks * 2); dm.qh = mem.alloc(n_blocks * 4);
            qx_split(d_raw, n_blocks, t, dm.p, dm.qh, dm.scales, dm.mins, 0);
        }
        const float * d_a = mem.upload(A, (size_t) M * K * 4);
        Q8Scratch q8;
        q8.q = mem.alloc<int8_t>((size_t) M * K); q8.d = mem.alloc<float>((size_t) M * nb * 4); q8.s = mem.alloc<float>((size_t) M * nb * 4);
        const GuardedOutput c(mem, (size_t) M * N * 4, epilogue == EPI_RESID ? C : nullptr);
        // GELU_ACT: f32 rows, as a quantised model's fc pass leaves its operand
        const MatmulEpilogue ep = matmul_epilogue(mem, epilogue, c.out<float>(), M, N, gelu_tab, W_Q4_0, N);
        if (path == 0) lane_matmul(dm, d_a, K, M, ep, &q8, 0);
        else           decode_q4_rows(path == 1, d_a, K, dm.p, dm.scales, N, ep, q8.q, q8.d, 0);
        if (!finish("bark_b200_quant_matmul")) return 0;
        if (!c.read("bark_b200_quant_matmul", C)) return -1;
        if (q_out) download(q_out, q8.q, (size_t) M * K);
        if (d_out) download(d_out, q8.d, (size_t) M * nb * 4);
        if (s_out) download(s_out, q8.s, (size_t) M * nb * 4);
        return 1;
    });
}

// the EnCodec convolution launcher conv1d on n items of x [Cin][L_b], its weight laid out as loader.cu lays it out
extern "C" int bark_b200_codec_conv1d(const float * x, int Cin, const int * L, int n, const uint16_t * w, const float * bias, int Cout, int k, int stride,
                                      int elu_in, const float * resid, float * y) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_conv1d";
        size_t total = 0;
        if (!x || !w || !bias || !y || Cin < 1 || Cout < 1 || k < 1 || stride < 1 || stride > k) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        // stride 1: the k - 1 reflected on the left must lie inside the item (ggml_pad_reflect_1d; the short and lane kernels would read
        // zeros there).  Strided: conv1d's own check refuses an item too short for either reflection.
        if (!codec_lengths(fn, L, n, stride == 1 ? k : 1, &total)) return 0;
        size_t out_total = 0;
        for (int b = 0; b < n; b++) out_total += (size_t) conv1d_out_len(L[b], k, stride);
        DeviceBuffers mem;
        ConvW cv; cv.k = k; cv.cin = Cin; cv.cout = Cout;
        cv.w = li_weight(mem, mem.upload((const __half *) w, (size_t) Cout * Cin * k * 2), Cout, Cin * k, &cv.Kp);
        cv.b = mem.upload(bias, (size_t) Cout * 4);
        const float * dx = mem.upload(x, total * Cin * 4), * dr = resid ? mem.upload(resid, out_total * Cout * 4) : nullptr;
        const GuardedOutput o(mem, out_total * Cout * 4, nullptr);
        const int ran = conv1d(dx, Cin, L, n, cv, elu_in != 0, dr, o.out<float>(), 0, stride);
        if (!finish(fn)) return 0;
        return o.read(fn, y) ? ran : -1;
    });
}

// convtr1d (ELU on the input, k = 2 stride, right trim, bias) on n items of x [Cin][T_b]; w [Cin][Cout][k] as stored, through the
// loader's convtr_rows and permute_to_li
extern "C" int bark_b200_codec_convtr1d(const float * x, int Cin, const int * T, int n, const uint16_t * w, const float * bias, int Cout, int stride,
                                        float * y) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_convtr1d";
        size_t total = 0;
        if (!x || !w || !bias || !y || Cin < 1 || Cout < 1 || stride < 1) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        if (!codec_lengths(fn, T, n, 1, &total)) return 0;
        const int k = 2 * stride;
        DeviceBuffers mem;
        ConvW cv; cv.k = k; cv.cin = Cin; cv.cout = Cout;
        __half * rows = mem.alloc<__half>((size_t) Cin * Cout * k * 2);
        convtr_rows(mem.upload((const __half *) w, (size_t) Cin * Cout * k * 2), rows, Cin, Cout, k, 0);
        cv.w = li_weight(mem, rows, Cout * k, Cin, &cv.Kp);
        cv.b = mem.upload(bias, (size_t) Cout * 4);
        const float * dx = mem.upload(x, total * Cin * 4);
        const GuardedOutput o(mem, total * stride * Cout * 4, nullptr);
        const int ran = convtr1d(dx, Cin, T, n, cv, stride, o.out<float>(), 0);
        if (!finish(fn)) return 0;
        return o.read(fn, y) ? ran : -1;
    });
}

// lstm_layer on n items of x [C][T_b] (wih, whh [4C][C] f16 as stored; bih, bhh [4C]); skip (may be null) added to the output
extern "C" int bark_b200_codec_lstm(const float * x, int C, const int * T, int n, const uint16_t * wih, const uint16_t * whh, const float * bih,
                                    const float * bhh, const float * skip, float * out) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_lstm";
        size_t total = 0;
        if (!x || !wih || !whh || !bih || !bhh || !out || C < 1) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        if (!codec_lengths(fn, T, n, 1, &total)) return 0;
        const size_t G4 = (size_t) 4 * C;
        DeviceBuffers mem;
        int Kp = 0;
        const __half * dih = li_weight(mem, mem.upload((const __half *) wih, G4 * C * 2), (int) G4, C, &Kp);
        const __half * dhh = li_weight(mem, mem.upload((const __half *) whh, G4 * C * 2), (int) G4, C, &Kp);
        const float * dbi = mem.upload(bih, G4 * 4), * dbh = mem.upload(bhh, G4 * 4);
        const float * dx = mem.upload(x, total * C * 4), * ds = skip ? mem.upload(skip, total * C * 4) : nullptr;
        float * gi = mem.poisoned<float>(total * G4 * 4), * hbuf = mem.poisoned<float>((size_t) 2 * kCodecMaxItems * C * 4);
        unsigned * counter = mem.alloc<unsigned>(sizeof(unsigned));
        const GuardedOutput o(mem, total * C * 4, nullptr);
        const int ran = lstm_layer(dx, C, T, n, dih, dhh, Kp, dbi, dbh, ds, gi, hbuf, counter, o.out<float>(), 0);
        if (!finish(fn)) return 0;
        return o.read(fn, out) ? ran : -1;
    });
}

// A CodecWindow from the hook's arrays; false (message naming fn) for a null array or an item without outputs
static bool hook_window(const char * fn, int n, const long long * org, const long long * first, const int * n_out, CodecWindow * w, size_t * out_total) {
    if (!org || !first || !n_out) { fprintf(stderr, "%s: null window array\n", fn); return false; }
    *out_total = 0;
    for (int b = 0; b < n; b++) {
        if (n_out[b] < 1) { fprintf(stderr, "%s: item %d has %d outputs (at least 1)\n", fn, b, n_out[b]); return false; }
        w->org[b] = org[b]; w->first[b] = first[b]; w->n_out[b] = n_out[b]; *out_total += (size_t) n_out[b];
    }
    return true;
}

// conv1d over windows (the launcher refuses a window whose outputs read outside it)
extern "C" int bark_b200_codec_conv1d_window(const float * x, int Cin, const int * L, int n, const long long * org, const long long * first, const int * n_out,
                                             const uint16_t * w, const float * bias, int Cout, int k, int stride, int elu_in, const float * resid, float * y) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_conv1d_window";
        size_t total = 0, out_total = 0;
        if (!x || !w || !bias || !y || Cin < 1 || Cout < 1 || k < 1 || stride < 1 || stride > k || (resid && stride > 1)) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        CodecWindow win;
        if (!codec_lengths(fn, L, n, 1, &total) || !hook_window(fn, n, org, first, n_out, &win, &out_total)) return 0;
        DeviceBuffers mem;
        ConvW cv; cv.k = k; cv.cin = Cin; cv.cout = Cout;
        cv.w = li_weight(mem, mem.upload((const __half *) w, (size_t) Cout * Cin * k * 2), Cout, Cin * k, &cv.Kp);
        cv.b = mem.upload(bias, (size_t) Cout * 4);
        const float * dx = mem.upload(x, total * Cin * 4), * dr = resid ? mem.upload(resid, out_total * Cout * 4) : nullptr;
        const GuardedOutput o(mem, out_total * Cout * 4, nullptr);
        const int ran = conv1d(dx, Cin, L, n, cv, elu_in != 0, dr, o.out<float>(), 0, stride, &win);
        if (!finish(fn)) return 0;
        return o.read(fn, y) ? ran : -1;
    });
}

// convtr1d over windows
extern "C" int bark_b200_codec_convtr1d_window(const float * x, int Cin, const int * L, int n, const long long * org, const long long * first, const int * n_out,
                                               const uint16_t * w, const float * bias, int Cout, int stride, float * y) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_convtr1d_window";
        size_t total = 0, out_total = 0;
        if (!x || !w || !bias || !y || Cin < 1 || Cout < 1 || stride < 1) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        CodecWindow win;
        if (!codec_lengths(fn, L, n, 1, &total) || !hook_window(fn, n, org, first, n_out, &win, &out_total)) return 0;
        const int k = 2 * stride;
        DeviceBuffers mem;
        ConvW cv; cv.k = k; cv.cin = Cin; cv.cout = Cout;
        __half * rows = mem.alloc<__half>((size_t) Cin * Cout * k * 2);
        convtr_rows(mem.upload((const __half *) w, (size_t) Cin * Cout * k * 2), rows, Cin, Cout, k, 0);
        cv.w = li_weight(mem, rows, Cout * k, Cin, &cv.Kp);
        cv.b = mem.upload(bias, (size_t) Cout * 4);
        const float * dx = mem.upload(x, total * Cin * 4);
        const GuardedOutput o(mem, out_total * stride * Cout * 4, nullptr);
        const int ran = convtr1d(dx, Cin, L, n, cv, stride, o.out<float>(), 0, &win);
        if (!finish(fn)) return 0;
        return o.read(fn, y) ? ran : -1;
    });
}

// lstm_layer from a state [n][2][C] (null: zeros), written back
extern "C" int bark_b200_codec_lstm_state(const float * x, int C, const int * T, int n, const uint16_t * wih, const uint16_t * whh, const float * bih,
                                          const float * bhh, const float * skip, float * state, float * out) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_lstm_state";
        size_t total = 0;
        if (!x || !wih || !whh || !bih || !bhh || !out || C < 1) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        if (!codec_lengths(fn, T, n, 1, &total)) return 0;
        const size_t G4 = (size_t) 4 * C, sb = (size_t) n * 2 * C * 4;
        DeviceBuffers mem;
        int Kp = 0;
        const __half * dih = li_weight(mem, mem.upload((const __half *) wih, G4 * C * 2), (int) G4, C, &Kp);
        const __half * dhh = li_weight(mem, mem.upload((const __half *) whh, G4 * C * 2), (int) G4, C, &Kp);
        const float * dbi = mem.upload(bih, G4 * 4), * dbh = mem.upload(bhh, G4 * 4);
        const float * dx = mem.upload(x, total * C * 4), * ds = skip ? mem.upload(skip, total * C * 4) : nullptr;
        float * gi = mem.poisoned<float>(total * G4 * 4), * hbuf = mem.poisoned<float>((size_t) 2 * kCodecMaxItems * C * 4);
        unsigned * counter = mem.alloc<unsigned>(sizeof(unsigned));
        std::vector<float> zeros;
        if (!state) zeros.assign((size_t) n * 2 * C, 0.f);
        float * dst = mem.upload(state ? state : zeros.data(), sb);
        std::vector<float *> per((size_t) n);
        for (int b = 0; b < n; b++) per[(size_t) b] = dst + (size_t) b * 2 * C;
        const GuardedOutput o(mem, total * C * 4, nullptr);
        const int ran = lstm_layer(dx, C, T, n, dih, dhh, Kp, dbi, dbh, ds, gi, hbuf, counter, o.out<float>(), 0, per.data());
        if (!finish(fn)) return 0;
        if (state) download(state, dst, sb);
        return o.read(fn, out) ? ran : -1;
    });
}

// rvq_decode on n items of codes [n_q][T_b] through codebooks [n_q][n_bins][hidden] -> x [hidden][T_b]
extern "C" int bark_b200_codec_rvq_decode(const int32_t * codes, int n_q, const int * T, int n, const float * codebooks, int hidden, int n_bins, float * x) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_codec_rvq_decode";
        size_t total = 0;
        if (!codes || !codebooks || !x || n_q < 1 || n_q > kMaxCodebooks || hidden < 1 || n_bins < 1) { fprintf(stderr, "%s: invalid arguments\n", fn); return 0; }
        if (!codec_lengths(fn, T, n, 1, &total)) return 0;
        for (size_t i = 0; i < total * n_q; i++)
            if (codes[i] < 0 || codes[i] >= n_bins) { fprintf(stderr, "%s: code %d outside [0, %d)\n", fn, codes[i], n_bins); return 0; }
        DeviceBuffers mem;
        CodecModel cm;
        cm.hidden_dim = hidden;
        const float * dcb = mem.upload(codebooks, (size_t) n_q * n_bins * hidden * 4);
        for (int q = 0; q < n_q; q++) cm.embed[q] = (float *) dcb + (size_t) q * n_bins * hidden;
        const int32_t * dc = mem.upload(codes, total * n_q * 4);
        const GuardedOutput o(mem, total * hidden * 4, nullptr);
        rvq_decode(cm, dc, n_q, T, n, o.out<float>(), 0);
        if (!finish(fn)) return 0;
        return o.read(fn, x) ? 1 : -1;
    });
}

// device_math_kernel: count <= 2^24 results, one 64 MB output at most
extern "C" int bark_b200_device_math(int fn, uint32_t lo_bits, uint32_t stride, uint32_t count, float * out) {
    return guarded(0, [&] {
        if (!out || fn < 0 || fn > 6 || stride < 1 || count < 1 || count > (1u << 24)) { fprintf(stderr, "bark_b200_device_math: invalid arguments\n"); return 0; }
        DeviceBuffers mem;
        const GuardedOutput o(mem, (size_t) count * 4, nullptr);
        BARK_LAUNCH(device_math_kernel, std::min<uint32_t>((count + 255) / 256, 4096), 256, 0, 0, fn, lo_bits, stride, count, o.out<float>());
        if (!finish("bark_b200_device_math")) return 0;
        return o.read("bark_b200_device_math", out) ? 1 : -1;
    });
}

// resample_kernel over windows of n items, each with its own table (built as a stream builds it) and format, in one launch
extern "C" int bark_b200_resample_window(const float * in, const int * n_frames, const int * channels, const int * in_rates, const int * out_rates,
                                         const long long * org, const long long * first, const int * n_out, const long long * end, int n, float * out) {
    return guarded(0, [&] {
        const char * fn = "bark_b200_resample_window";
        if (!in || !n_frames || !channels || !in_rates || !out_rates || !out) { fprintf(stderr, "%s: null argument\n", fn); return 0; }
        if (n < 1 || n > kCodecMaxItems) { fprintf(stderr, "%s: %d items (1 to %d)\n", fn, n, kCodecMaxItems); return 0; }
        CodecWindow cw;
        size_t out_total = 0, in_total = 0;
        if (!hook_window(fn, n, org, first, n_out, &cw, &out_total)) return 0;
        std::vector<ResampleWindow> w((size_t) n);
        std::vector<std::vector<unsigned char>> bytes((size_t) n);
        for (int b = 0; b < n; b++) {
            const std::string item = "item " + std::to_string(b) + ": ";
            if (n_frames[b] < 0) { fprintf(stderr, "%s: %s%d frames\n", fn, item.c_str(), n_frames[b]); return 0; }
            if (n_frames[b] > 0 && !resample_input_ok(fn, item, in + in_total, n_frames[b], channels[b], in_rates[b])) return 0;
            if (channels[b] < 1 || channels[b] > kResampleMaxChannels || std::min(in_rates[b], out_rates[b]) < kResampleMinRate ||
                std::max(in_rates[b], out_rates[b]) > kResampleMaxRate) { fprintf(stderr, "%s: %sformat outside the resampler's limits\n", fn, item.c_str()); return 0; }
            bytes[(size_t) b] = resample_table(in_rates[b], out_rates[b], &w[(size_t) b].t);
            w[(size_t) b].org = org[b]; w[(size_t) b].first = first[b]; w[(size_t) b].n_out = n_out[b]; w[(size_t) b].len = n_frames[b];
            w[(size_t) b].C = channels[b]; w[(size_t) b].end = end && end[b] >= 0 ? end[b] : LLONG_MAX;
            in_total += (size_t) n_frames[b] * channels[b];
        }
        DeviceBuffers mem;
        const float * d_in = mem.upload(in, std::max(in_total, (size_t) 1) * sizeof(float));
        const GuardedOutput y(mem, out_total * sizeof(float), nullptr);
        size_t xo = 0, yo = 0;
        for (int b = 0; b < n; b++) {
            if (!bytes[(size_t) b].empty()) resample_bind(w[(size_t) b].t, mem.upload(bytes[(size_t) b].data(), bytes[(size_t) b].size()));
            w[(size_t) b].x = d_in + xo; w[(size_t) b].y = y.out<float>() + yo;
            xo += (size_t) n_frames[b] * channels[b]; yo += (size_t) n_out[b];
        }
        resample_windows(w.data(), n, 0);
        if (!finish(fn)) return 0;
        return y.read(fn, out) ? 1 : -1;
    });
}
