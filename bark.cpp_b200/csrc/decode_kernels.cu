// Persistent decode step: ONE cooperative launch evaluates a whole causal-GPT token (N = 1, n_past > 0), i.e. everything
// bark_build_gpt_graph (bark.cpp:1186-1414) emits for a single position — ~35 ggml nodes and ~400 thread barriers per
// layer on the CPU, ~10 kernel launches per layer in the multi-kernel path (gpt_forward.cu) — with the same bit-exact
// arithmetic (common.cuh "Lane order").
//
// One CTA per SM, 512 threads.
//  * Weights are a pure stream: each CTA owns a contiguous row range of every matrix (lane-interleaved rows), each warp a
//    contiguous slice of that range.  As soon as a warp finishes a phase, its lane 0 issues ONE TMA bulk copy
//    (cp.async.bulk + a per-warp mbarrier) of its rows of the phase after next into a private shared-memory staging area, so
//    HBM latency hides behind two phases and no block-wide barrier surrounds the weight stream (a CTA-wide TMA ring fed by one
//    elected thread puts that thread on the critical path of every phase).  The copies carry an L2 evict-first policy: the
//    weights streamed per token (188 MB for bark-small, ≈ 625 MB for bark-large) would otherwise flush the KV cache, the exchange words, local memory and
//    the kernel's own code out of the 50 MB L2 on every token, and every other CTA waits for the one that missed.
//  * Activations cross CTAs as TAGGED words: every exchanged float travels in one 8-byte {value, epoch} store; consumers
//    spin on the words they need until the epoch matches.  Data and "ready" flag arrive in the same L2 transaction, so a
//    grid-wide dependency costs one store->load latency instead of store + fence + atomic + poll + load (a classic
//    barrier would be needed 6 times per layer).  Epochs are unique per use and never reset.
//    The vectors EVERY CTA gathers (q, attention output, residual stream, MLP activations) are published into kReplicas copies
//    (lanes 0..7 of the producing warp store the same word into 8 buffers) and CTA c polls copy c % 8 with 16-byte loads: an L2
//    line then has 1/8 of the CTAs as readers and half as many requests (tools/microbench/exchange_rounds.cu times one grid-wide
//    dependency both ways) — hot lines, not the latency of one L2 round trip, are what makes an exchange expensive.
//  * KV rows of older positions are staged in shared memory with cp.async BEFORE waiting for q / the probabilities.
//  * Nothing the phases need lives in local memory: block-wide state is in static shared memory (BlockCtx).
//
// Phases of a layer (each ends by publishing tagged outputs, the next begins by consuming them):
//   P1  LN1 -> QKV rows          -> q, k_new, v_new (+ K/V appended to the f32 KV cache for later tokens)
//   P2  scores[h][k] = <K[k][h], q[h]> * scale, (h,k) pairs spread over all warps     -> scores
//   P3  per (head, 16 columns of the head): soft_max + P.V                             -> att
//   P4  c_proj rows + residual                                                         -> x
//   P5  LN2 -> c_fc rows -> GELU table                                                 -> ff
//   P6  mlp/c_proj rows + residual                                                     -> x
// then LN_f -> lm_head rows [lm_lo, lm_hi) -> logits (plain stores; the kernel ends).
#include "epilogue.cuh"
#include "gpt_kernels.h"

namespace bark {

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
static_assert(kWarps == 16, "the soft_max tile is 16 columns wide: one warp finishes one column");
constexpr int kWarpSlotBytes = 12 * 1024;       // per-warp staging area: two halves, phases alternate (rows are fetched two phases ahead)
constexpr int kHalfSlotBytes = kWarpSlotBytes / 2;
constexpr int kReplicas = kDecodeReplicas;      // copies of every all-to-all exchange vector (gpt_kernels.h)

struct SmemLayout {
    static constexpr int wslot = 0;                                 // kWarps x 12 KB: each warp's weight rows of its next two phases (TMA bulk copies)
    static constexpr int act = wslot + kWarps * kWarpSlotBytes;     // two-plane LI activation operand, up to 4096 floats
    static constexpr int x = act + 4096 * 4;                        // residual stream, up to 1024 floats
    static constexpr int q = x + 1024 * 4;                          // q vector / probabilities row, up to 1024 floats
    static constexpr int part = q + 1024 * 4;                       // P.V lane partials [32][16] + chunk sums [128]
    static constexpr int red = part + (32 * 16 + 128) * 4;          // reduction scratch: 16 doubles + 16 floats + 16 doubles + 4 broadcast slots
    static constexpr int sched = red + (kWarps + kWarps / 2 + kWarps + 4) * 8;   // per-CTA row ranges: kMaxPhases x PhaseSched
    static constexpr int total = sched + 128 * 32;
};

// ---- PTX helpers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
    const long long t0 = clock64();                          // slow path only: a protocol bug must trap, not hang the GPU
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (!done && clock64() - t0 > 4000000000ll) __trap();
    }
}
// one bulk copy global -> shared, completion counted on `bar`, L2 evict-first (the weight stream is read once per token)
__device__ __forceinline__ void tma_bulk_g2s_stream(uint32_t dst, const void * src, uint32_t bytes, uint32_t bar, unsigned long long policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(policy) : "memory");
}
__device__ __forceinline__ unsigned long long l2_evict_first_policy() {
    unsigned long long pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// ---- tagged exchange -------------------------------------------------------------------------------------------------
typedef unsigned long long tagged_t;                                // low 32 bits: float payload, high 32 bits: epoch
__device__ __forceinline__ void publish(tagged_t * p, float v, uint32_t tag) {
    const tagged_t w = ((tagged_t) tag << 32) | (tagged_t) __float_as_uint(v);
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ tagged_t peek(const tagged_t * p) {
    tagged_t w;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    return w;
}
// two adjacent tagged words in one 16-byte request (each word is still its own {value, epoch} unit)
__device__ __forceinline__ void peek2(const tagged_t * p, tagged_t & a, tagged_t & b) {
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
// lanes 0 .. kReplicas-1 of a warp store the same word into the kReplicas copies of an all-to-all vector (copy stride `n` words)
__device__ __forceinline__ void publish_all(tagged_t * base, int n, int i, float v, uint32_t tag, int lane) {
    if (lane < kReplicas) publish(base + (size_t) lane * n + i, v, tag);
}
__shared__ unsigned s_poll_ns;                                      // back-off between polls (DecodeArgs::poll_ns, default 40)
// Head start per exchange type (DecodeArgs::headstart): how long a CTA sleeps before its FIRST poll of that exchange.  Polling is not
// free: one CTA per SM x 512 threads re-reading tagged words every ~100 ns approach the L2's request rate and slow the very producers
// they wait for, while sleeping past the arrival sits on the critical path.  Timing only, never results.
enum { XT_Q = 0, XT_ATT = 1, XT_X1 = 2, XT_FF = 3, XT_X2 = 4, XT_SC = 5, XT_COUNT = 6 };
__shared__ unsigned s_headstart[XT_COUNT];
__device__ __forceinline__ float consume1(const tagged_t * p, uint32_t tag) {
    tagged_t w = peek(p);
    while ((uint32_t)(w >> 32) != tag) { __nanosleep(s_poll_ns); w = peek(p); }       // back off: thousands of pollers share a few L2 lines
    return __uint_as_float((uint32_t) w);
}
// two-plane LI index of column k in the shared activation operand: LDS.128 of one plane is contiguous across lanes
__device__ __forceinline__ int act_index(int k) {
    const int v = k & 31, c = k >> 5, g = c >> 3, e = c & 7;
    return (((g << 1) + (e >> 2)) * 32 + v) * 4 + (e & 3);
}

// debug stamps (BARK_B200_DECODE_TIMING=1): thread 0 of CTA 0 stamps every layer (rows 0..L-1 of the buffer), thread 0 of
// every CTA stamps layer 5 (rows 64 + cta); 32 slots per row, %globaltimer nanoseconds.  s_tim is null in normal runs.
__shared__ unsigned long long * s_tim;
__shared__ int s_tim_layer, s_tim_tid;                               // s_tim_tid: the stamping thread (0, or lane 0 of another warp: BARK_B200_DECODE_TIMING_TID)
// TM = false (every normal run) compiles the stamps away: even a not-taken stamp is two shared-memory loads and a branch on
// the critical path of a single warp, ~30 times per layer.
template <bool TM>
__device__ __forceinline__ void tstamp(int i) {
    if (TM && s_tim && (int) threadIdx.x == s_tim_tid) {
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        const int layer = s_tim_layer;
        if (blockIdx.x == 0) s_tim[layer * 32 + i] = t;
        if (layer == 5) s_tim[(64 + blockIdx.x) * 32 + i] = t;
    }
}

// finer stamps of CTA 0 for one code region (rows `row0 + layer` of the buffer: 32.. = row phases, 48.. = LayerNorm)
template <bool TM>
__device__ __forceinline__ void tstamp2(int row0, int i) {
    if (TM && s_tim && (int) threadIdx.x == s_tim_tid && blockIdx.x == 0 && s_tim_layer < 16) {
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        s_tim[(row0 + s_tim_layer) * 32 + i] = t;
    }
}

// Fetch a published vector into shared memory.  Every thread takes entries tid, tid + 512, ... (n <= MAXJ * 512): all loads
// go out together, stragglers are re-polled.  Deliberately NOT inlined: the kernel lives or dies by its instruction-cache
// footprint (a 100 KB body re-fetched from L2 every layer cost 5-10x, see DESIGN.md), so shared pieces are real calls.
enum { SINK_PLAIN = 0, SINK_ACT = 1, SINK_ACT_R16 = 2 };
template <int MAXJ>
__device__ __forceinline__ void consume_to_smem_inl(const tagged_t * g, int n, uint32_t tag, float * dst, int mode, int xt) {
    constexpr int PJ = MAXJ / 2;                             // pairs of words per thread (n is even: E % 32 == 0)
    tagged_t w[PJ][2];
    g += (size_t)(blockIdx.x % kReplicas) * n;               // this CTA's copy of the vector
    const unsigned hs = s_headstart[xt];
    if (hs) __nanosleep(hs);                                 // the producers need about this long: do not hammer their lines meanwhile
#pragma unroll
    for (int j = 0; j < PJ; j++) { const int i = 2 * (threadIdx.x + j * kThreads); if (i < n) peek2(g + i, w[j][0], w[j][1]); }
#pragma unroll
    for (int j = 0; j < PJ; j++) {
        const int i = 2 * (threadIdx.x + j * kThreads);
        if (i < n) {
            while ((uint32_t)(w[j][0] >> 32) != tag || (uint32_t)(w[j][1] >> 32) != tag) { __nanosleep(s_poll_ns); peek2(g + i, w[j][0], w[j][1]); }
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const float v = __uint_as_float((uint32_t) w[j][e]);
                if (mode == SINK_PLAIN) dst[i + e] = v; else dst[act_index(i + e)] = mode == SINK_ACT_R16 ? round_f16(v) : v;
            }
        }
    }
    __syncthreads();
}
// one private (not replicated) vector of any length, one word per load: the score row of a head (a few consumer CTAs per head)
__device__ __forceinline__ void consume_row_to_smem(const tagged_t * g, int n, uint32_t tag, float * dst) {      // (inline: a call here would force the caller's prefetched V registers onto the stack)
    tagged_t w[2];
    const unsigned hs = s_headstart[XT_SC];
    if (hs) __nanosleep(hs);
#pragma unroll
    for (int j = 0; j < 2; j++) { const int i = threadIdx.x + j * kThreads; if (i < n) w[j] = peek(g + i); }
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const int i = threadIdx.x + j * kThreads;
        if (i < n) {
            while ((uint32_t)(w[j] >> 32) != tag) { __nanosleep(s_poll_ns); w[j] = peek(g + i); }
            dst[i] = __uint_as_float((uint32_t) w[j]);
        }
    }
    __syncthreads();
}
// out-of-line copy: the kernel lives or dies by its instruction-cache footprint, so shared pieces are real calls
template <int MAXJ>
__device__ __noinline__ void consume_to_smem(const tagged_t * g, int n, uint32_t tag, float * dst, int mode, int xt) {
    consume_to_smem_inl<MAXJ>(g, n, tag, dst, mode, xt);
}

// A double division is a long dependent-latency sequence (on the LayerNorm critical path it would dominate), so the kernel never divides in double on the common path.  It only has to decide which FLOAT the
// reference's (float)(sum / n) is: with c = sum * (1/n) and a rigorous half-width w covering both the summation-order
// uncertainty and the error of the multiply-by-reciprocal, both ends of [c - w, c + w] rounding to the same float
// settles it; the exact (slow) path runs otherwise.

// reciprocal of a positive double to ~2^-50 relative error: float seed + 2 Newton steps (4 DFMA)
__device__ __forceinline__ double approx_rcp(double x) {
    double y = (double) __frcp_rn((float) x);
    double e = __fma_rn(-x, y, 1.0); y = __fma_rn(y, e, y);
    e = __fma_rn(-x, y, 1.0);        y = __fma_rn(y, e, y);
    return y;
}

// LayerNorm of xs[0..E) (ggml.c:11964-12013; order-independence argument in layernorm_act_kernel, gpt_kernels.cu) ->
// activation operand (optionally f16-rounded) in two-plane LI order.  Block-wide: each thread owns <= 2 elements.
// One block barrier per statistic: warps leave their partial sums in shared memory and EVERY thread adds the 16 partials and
// takes the rounding decision itself (identical inputs, identical arithmetic -> identical result), instead of funnelling
// through warp 0 and a second barrier.  red: [0,16) double mean partials, [16,24) 16 float |x| partials, [24,40) double
// variance partials.
// COPY: 1 in decode_rows_kernel (the row tests) — the same source as a separate function, so that a second caller cannot change the
// register allocation ptxas picks for the one the decode step calls.
template <bool ROUND16, bool TM, bool NATURAL = false, int COPY = 0>
__device__ __noinline__ void block_layernorm(const float * xs, int E, double inv_E, const float * __restrict__ g, const float * __restrict__ b, float * act,
                                             double * red, unsigned * fallback_counter, int sb) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tb = sb == 1 ? 0 : 16;
    tstamp2<TM>(48, tb + 0);
    double * sA = red, * sB = red + kWarps + kWarps / 2;
    float * fA = reinterpret_cast<float *>(red + kWarps);
    const int i0 = tid, i1 = tid + kThreads;
    const bool h0 = i0 < E, h1 = i1 < E;
    // gains / biases are different vectors every layer (L2 or HBM latency): fetch them now, use them at the end
    const float g0 = h0 ? __ldg(g + i0) : 0.f, g1 = h1 ? __ldg(g + i1) : 0.f;
    const float b0 = (b && h0) ? __ldg(b + i0) : 0.f, b1 = (b && h1) ? __ldg(b + i1) : 0.f;
    const float x0 = h0 ? xs[i0] : 0.f, x1 = h1 ? xs[i1] : 0.f;
    const double slack = 2.0 * (double) E * 0x1p-53 * (1.0 + 1e-6);

    // ---- mean ----
    double s = (double) x0 + (double) x1;
    float a = fabsf(x0) + fabsf(x1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); a += __shfl_xor_sync(0xffffffffu, a, o); }
    tstamp2<TM>(48, tb + 1);
    if (lane == 0) { sA[warp] = s; fA[warp] = a; }
    __syncthreads();
    tstamp2<TM>(48, tb + 2);
    float mean;
    {
        // the 16 warp partials are combined by a 4-level xor butterfly inside every warp (lane l starts from partial l & 15): every lane of
        // every warp ends with the same bits (each level adds the same two values on both sides, addition is commutative), any order is
        // covered by the bracket below.  The alternative — every thread loads all 16 partials and adds them itself — is 32 LDS + 30 FP64
        // adds per thread and issue-bound.
        double qd[1]; float qf[1];
        qd[0] = sA[lane & (kWarps - 1)]; qf[0] = fA[lane & (kWarps - 1)];
#pragma unroll
        for (int o = kWarps / 2; o > 0; o >>= 1) { qd[0] += __shfl_xor_sync(0xffffffffu, qd[0], o); qf[0] += __shfl_xor_sync(0xffffffffu, qf[0], o); }
        const double S = qd[0]; const float A = qf[0];
        if (S == 1.25) tstamp2<TM>(48, tb + 15);               // (forces the tree to be complete before the next stamp)
        tstamp2<TM>(48, tb + 3);
        const double c = S * inv_E;
        const double hw = (slack * (double) A * 1.001) * inv_E + fabs(c) * 0x1p-50;     // 1.001: the float abs-sum may be low by n*2^-24
        mean = __double2float_rn(c - hw);
        if (mean != __double2float_rn(c + hw)) {                                        // rare: replay the reference's sequential sum (every thread, same result)
            double ss = 0.0;
            for (int i = 0; i < E; i++) ss = __dadd_rn(ss, (double) xs[i]);
            mean = __double2float_rn(__ddiv_rn(ss, (double) E));
            if (fallback_counter && tid == 0) atomicAdd(fallback_counter, 1u);
        }
    }
    tstamp<TM>(sb);
    // ---- variance ----
    const float v0 = __fsub_rn(x0, mean), v1 = __fsub_rn(x1, mean);
    double s2 = (h0 ? (double) __fmul_rn(v0, v0) : 0.0) + (h1 ? (double) __fmul_rn(v1, v1) : 0.0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    if (s2 == 1.25) tstamp2<TM>(48, tb + 15);
    tstamp2<TM>(48, tb + 5);
    if (lane == 0) sB[warp] = s2;
    __syncthreads();
    tstamp2<TM>(48, tb + 6);
    float scale;
    {
        double qd[1];
        qd[0] = sB[lane & (kWarps - 1)];
#pragma unroll
        for (int o = kWarps / 2; o > 0; o >>= 1) qd[0] += __shfl_xor_sync(0xffffffffu, qd[0], o);
        const double S2 = qd[0];
        const double c = S2 * inv_E;
        const double hw = (slack * S2) * inv_E + c * 0x1p-50;
        float variance = __double2float_rn(c - hw);
        if (variance != __double2float_rn(c + hw)) {
            double ss = 0.0;
            for (int i = 0; i < E; i++) { const float v = __fsub_rn(xs[i], mean); ss = __dadd_rn(ss, (double) __fmul_rn(v, v)); }
            variance = __double2float_rn(__ddiv_rn(ss, (double) E));
            if (fallback_counter && tid == 0) atomicAdd(fallback_counter, 1u);
        }
        scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(variance, 1e-5f)));
    }
    if (scale == 1.25f) tstamp2<TM>(48, tb + 15);
    tstamp2<TM>(48, tb + 7);
    if (h0) { float y = __fmul_rn(__fmul_rn(v0, scale), g0); if (b) y = __fadd_rn(y, b0); act[NATURAL ? i0 : act_index(i0)] = ROUND16 ? round_f16(y) : y; }
    if (h1) { float y = __fmul_rn(__fmul_rn(v1, scale), g1); if (b) y = __fadd_rn(y, b1); act[NATURAL ? i1 : act_index(i1)] = ROUND16 ? round_f16(y) : y; }
    tstamp2<TM>(48, tb + 8);
    __syncthreads();
    tstamp2<TM>(48, tb + 9);
}

// Per-CTA row ranges of every phase, built once per launch in shared memory (the divisions and table look-ups they replace
// cost ~2 us of single-thread time per phase when done on the fly).
struct PhaseSched { int r0, r1, K, row_bytes; const unsigned char * w; const unsigned char * ws; };   // rows [r0, r1) of this phase belong to this CTA

enum { EP_QKV = 0, EP_RESID = 1, EP_GELU = 2, EP_LOGITS = 3 };

// GELU of v given its table entry t = gelu_tab[f16(v)], already loaded (ggml_vec_gelu_f32, ggml.c:2557-2571)
__device__ __forceinline__ float gelu_sel(float v, __half t) { return v <= -10.0f ? 0.0f : v >= 10.0f ? v : __half2float(t); }

template <typename WT> struct Unpack;
template <> struct Unpack<__half> {
    static constexpr int G = 8;
    __device__ static void w(const uint4 & u, float (&f)[8]) {
        const __half2 * h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
        for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
    }
};
template <> struct Unpack<float> {
    static constexpr int G = 4;
    __device__ static void w(const uint4 & u, float (&f)[4]) { f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w); }
};

// NR adjacent weight rows against the shared activation operand, lane order.  SH: the rows sit in this warp's staging area and
// are read with ld.shared (a generic-pointer load of shared memory is tracked like a global load and costs several times the
// latency: ncu showed the unpack instructions behind it waiting on the long scoreboard); otherwise they stream from global
// memory.  The NR chains are independent, so two rows cost barely more than one.
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v; asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));   // volatile: stays behind the (volatile) mbarrier wait
    return v;
}
template <typename WT, bool SH, int NR>
__device__ __forceinline__ void row_dot(const unsigned char * row, int row_bytes, const float * act, int K, int lane, float (&out)[NR]) {
    constexpr int G = Unpack<WT>::G;
    const int nsteps = K >> 5;
    const uint4 * wv = reinterpret_cast<const uint4 *>(row) + lane;
    const uint32_t sw = SH ? smem_u32(row) + lane * 16 : 0u;
    const int rstride = row_bytes >> 4;                        // uint4 words between adjacent rows
    auto fetch = [&](int n, int i) -> uint4 { return SH ? lds128(sw + n * row_bytes + i * 512) : wv[n * rstride + i * 32]; };
    float acc[NR];
#pragma unroll
    for (int n = 0; n < NR; n++) acc[n] = 0.0f;
    if constexpr (G == 8) {
        const int ng = nsteps >> 3, tail = nsteps & 7;
#pragma unroll 3
        for (int g = 0; g < ng; g++) {
            const float4 a0 = *reinterpret_cast<const float4 *>(act + ((g * 2) * 32 + lane) * 4);
            const float4 a1 = *reinterpret_cast<const float4 *>(act + ((g * 2 + 1) * 32 + lane) * 4);
#pragma unroll
            for (int n = 0; n < NR; n++) {
                float w[8]; Unpack<WT>::w(fetch(n, g), w);
                float c = acc[n];
                c = __fmaf_rn(w[0], a0.x, c); c = __fmaf_rn(w[1], a0.y, c); c = __fmaf_rn(w[2], a0.z, c); c = __fmaf_rn(w[3], a0.w, c);
                c = __fmaf_rn(w[4], a1.x, c); c = __fmaf_rn(w[5], a1.y, c); c = __fmaf_rn(w[6], a1.z, c); c = __fmaf_rn(w[7], a1.w, c);
                acc[n] = c;
            }
        }
        if (tail) {
            const float * a0 = act + ((ng * 2) * 32 + lane) * 4, * a1 = act + ((ng * 2 + 1) * 32 + lane) * 4;
#pragma unroll
            for (int n = 0; n < NR; n++) {
                float w[8]; Unpack<WT>::w(fetch(n, ng), w);
#pragma unroll
                for (int e = 0; e < 8; e++) if (e < tail) acc[n] = __fmaf_rn(w[e], e < 4 ? a0[e] : a1[e - 4], acc[n]);
            }
        }
    } else {
        // f32 rows: 4 chain steps per 16 bytes = one quad of the two-plane operand (quad index = chain step / 4)
        const int nq = nsteps >> 2, tail = nsteps & 3;
        for (int qd = 0; qd < nq; qd++) {
            const float4 a = *reinterpret_cast<const float4 *>(act + (qd * 32 + lane) * 4);
#pragma unroll
            for (int n = 0; n < NR; n++) {
                float w[4]; Unpack<WT>::w(fetch(n, qd), w);
                float c = acc[n];
                c = __fmaf_rn(w[0], a.x, c); c = __fmaf_rn(w[1], a.y, c); c = __fmaf_rn(w[2], a.z, c); c = __fmaf_rn(w[3], a.w, c);
                acc[n] = c;
            }
        }
        if (tail) {
            const float * a = act + (nq * 32 + lane) * 4;
#pragma unroll
            for (int n = 0; n < NR; n++) {
                float w[4]; Unpack<WT>::w(fetch(n, nq), w);
#pragma unroll
                for (int e = 0; e < 4; e++) if (e < tail) acc[n] = __fmaf_rn(w[e], a[e], acc[n]);
            }
        }
    }
#pragma unroll
    for (int n = 0; n < NR; n++) out[n] = lane_tree_reduce(acc[n]);
}

// ---- q4_0 weights (BASELINE configs[3]) ---------------------------------------------------------------------------------------------
// WT = Q4: the phase streams 16-byte nibble words [rows][K/32] plus f16 block scales [rows][K/32]; the activation operand is the
// q8_0 quantisation of the f32 vector (quantize_row_q8_0, ggml-quants.c:944-1000); a dot product is ggml_vec_dot_q4_0_q8_0's AVX2
// flavour (ggml-quants.c:4191-4214): eight float accumulators per output, one fused multiply-add per block, hsum_float_8.  Same
// arithmetic as q4_kernels.cu (the per-op path), here inside the persistent step: eight lanes own one output, a warp four rows.
struct Q4 {};
template <typename WT> struct IsQ4 { static constexpr bool v = false; };
template <> struct IsQ4<Q4> { static constexpr bool v = true; };

// act (f32, natural order) -> int8 q[K] + f32 d[K/32] (the f16-rounded scale, widened back); block-wide, one warp per 32-element block.
// A non-finite product gives -128 (cvtps_epi32 -> INT_MIN, then the saturating packs), as in quantize_q8x_kernel.
__device__ __forceinline__ void quantize_act_q8(const float * act, int K, int8_t * q, float * d) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int b = warp; b < (K >> 5); b += kWarps) {
        const float v = act[b * 32 + lane];
        float amax = fabsf(v);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float id = amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f;
        const float p = __fmul_rn(v, id);
        q[b * 32 + lane] = (int8_t)(isfinite(p) ? __float2int_rn(p) : -128);
        if (lane == 0) d[b] = __half2float(__float2half_rn(__fdiv_rn(amax, 127.0f)));
    }
    __syncthreads();
}

// up to 4 adjacent q4_0 rows against the q8 operand; every lane of group g = lane / 8 returns the result of row g
template <bool SH>
__device__ __forceinline__ float row_dot_q4(const unsigned char * qrows, const unsigned char * srows, int nrows, int nb, const int8_t * aq, const float * ad, int lane) {
    const int l = lane & 7, row = min(lane >> 3, nrows - 1);
    const bool high = l >= 4;
    const unsigned char * wq = qrows + (size_t) row * nb * 16 + (l & 3) * 4;
    const unsigned char * ws = srows + (size_t) row * nb * 2;
    // every operand through ld.shared (a generic-pointer load of shared memory is tracked like a global load: long scoreboard)
    const uint32_t s_wq = SH ? smem_u32(wq) : 0u, s_ws = SH ? smem_u32(ws) : 0u, s_aq = smem_u32(aq) + l * 4, s_ad = smem_u32(ad);
    float acc = 0.0f;
    constexpr int UB = 8;
    for (int b0 = 0; b0 < nb; b0 += UB) {
        uint32_t wr[UB]; float dr[UB]; int yr[UB];
#pragma unroll
        for (int u = 0; u < UB; u++) if (b0 + u < nb) {
            unsigned short hs; float da;
            if (SH) { asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wr[u]) : "r"(s_wq + (b0 + u) * 16) : "memory"); asm volatile("ld.shared.u16 %0, [%1];" : "=h"(hs) : "r"(s_ws + (b0 + u) * 2) : "memory"); }
            else    { wr[u] = __ldg(reinterpret_cast<const uint32_t *>(wq + (size_t)(b0 + u) * 16)); hs = __ldg(reinterpret_cast<const unsigned short *>(ws + (size_t)(b0 + u) * 2)); }
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(da) : "r"(s_ad + (b0 + u) * 4) : "memory");
            asm volatile("ld.shared.s32 %0, [%1];" : "=r"(yr[u]) : "r"(s_aq + (b0 + u) * 32) : "memory");
            dr[u] = __fmul_rn(__half2float(__ushort_as_half(hs)), da);
        }
#pragma unroll
        for (int u = 0; u < UB; u++) {
            if (b0 + u < nb) {
                const uint32_t w = (high ? (wr[u] >> 4) : wr[u]) & 0x0f0f0f0fu;
                const int wi = (int) __vsub4(w, 0x08080808u);
                acc = __fmaf_rn(dr[u], (float) __dp4a(wi, yr[u], 0), acc);
            }
        }
    }
    acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, 4));      // hsum_float_8 (ggml-quants.c:48-54)
    acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, 2));
    acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, 1));
    return acc;
}
// dequantize_row_q4_0 (ggml-quants.c:1515-1533) of one element of a wte row kept in the file's 18-byte blocks
__device__ __forceinline__ float wte_q4_value(const void * wte, int E, int row, int i) {
    const unsigned char * blk = (const unsigned char *) wte + ((size_t) row * (E >> 5) + (i >> 5)) * 18;
    const float d = __half2float(__ushort_as_half((unsigned short)(blk[0] | (blk[1] << 8))));
    const int j = i & 31, q = j < 16 ? (blk[2 + j] & 0x0f) : (blk[2 + j - 16] >> 4);
    return __fmul_rn((float)(q - 8), d);
}

// embedding of the one new token (bark.cpp:1226-1228, 1259): every CTA keeps its own copy of the residual stream.  token_ptr != null:
// the token is read from device memory (the previous step's sample) and clamped to the vocabulary
template <typename WT>
__device__ __forceinline__ void embed_token(const void * wte, const float * wpe, const int32_t * token_ptr, int token, int n_vocab_in, int E, int n_past, float * xs) {
    if (token_ptr) token = min(max(__ldcg(token_ptr), 0), n_vocab_in - 1);
    for (int i = threadIdx.x; i < E; i += kThreads) {
        float t;
        if constexpr (IsQ4<WT>::v) t = wte_q4_value(wte, E, token, i);
        else t = (float) ((const WT *) wte)[(size_t) token * E + i];
        xs[i] = __fadd_rn(t, wpe[(size_t) n_past * E + i]);
    }
}

constexpr int kMaxTasks = 8;        // (h, k) score tasks per warp per batch of the transposed butterfly; a warp's key tail holds up to 2 * kMaxTasks (key_tail).
                                    // 128 CTAs: bark-small has 80 score CTAs, H * block_size / (80 * kWarps) = 12 * 1024 / 1280 < 10 tasks per warp; bark-large f16
                                    // has 64 score CTAs whose tails hold 8 tasks, so past n_kv = 513 (16 * n_past > 8 * 1024) the rest run without the prefetch

// Block-wide state of the phases, in static shared memory (a by-reference struct in local memory cost L1/L2 round trips on
// the critical path: the 72 KB of per-thread stack frames do not fit the L1 left over next to 220 KB of shared memory).
struct BlockCtx {
    tagged_t * gq, * gk, * gv, * gx, * gff, * gatt, * gscores;
    float * mem_k, * mem_v, * logits;
    const __half * gelu_tab;
    unsigned long long policy;       // L2 evict-first descriptor of the weight stream
    int E, ctx, n_past, n_phases;
    float scale;                     // score scale 1 / sqrt(head size): the kernel body has no register to spare for it across the layer loop
};
__shared__ BlockCtx s_bc;
__shared__ __align__(8) unsigned long long s_bar[kWarps][2];       // per warp, per staging half: "rows have landed"
extern __shared__ __align__(128) unsigned char dsm[];

__device__ __forceinline__ const PhaseSched * sched_tab() { return reinterpret_cast<const PhaseSched *>(dsm + SmemLayout::sched); }
// rows [a, b) of this warp: the CTA's range cut into 16 contiguous slices (contiguous rows = one bulk copy)
__device__ __forceinline__ void warp_rows(const PhaseSched & p, int warp, int & a, int & b) {
    const int n = p.r1 - p.r0;
    a = p.r0 + ((warp * n) >> 4); b = p.r0 + (((warp + 1) * n) >> 4);
}

// q4_0 rows are staged when both pieces fit a half and satisfy the bulk copy's 16-byte size / address granularity (tiny test models
// with K < 256 have 8-byte scale rows: those phases read from global memory instead)
__device__ __forceinline__ bool q4_staged(uint32_t qbytes, uint32_t sbytes, const unsigned char * ssrc) {
    return qbytes != 0 && qbytes + sbytes <= (uint32_t) kHalfSlotBytes && (sbytes & 15u) == 0 && (reinterpret_cast<uintptr_t>(ssrc) & 15u) == 0;
}

// Lane 0: start the bulk copy of this warp's rows of `phase` into half (phase & 1) of its staging area and arm that half's
// mbarrier.  The barrier is armed exactly once per phase (with or without bytes), so use k of a half completes barrier
// phase k and run_phase waits on parity (phase >> 1) & 1.  Rows that do not fit (lm_head over the whole vocabulary, K = 4096
// rows of bark-large) are read from global memory by run_phase instead.
__device__ __forceinline__ void stage_rows(int phase) {
    if (phase >= s_bc.n_phases || (threadIdx.x & 31) != 0) return;
    const int warp = threadIdx.x >> 5, half = phase & 1;
    const PhaseSched p = sched_tab()[phase];
    int a, b; warp_rows(p, warp, a, b);
    const uint32_t bytes = (uint32_t)((b - a) * p.row_bytes);
    const uint32_t bar = smem_u32(&s_bar[warp][half]);
    const uint32_t dst = smem_u32(dsm + SmemLayout::wslot) + warp * kWarpSlotBytes + half * kHalfSlotBytes;
    if (p.ws) {                                              // q4_0: nibble words, then the f16 block scales behind them (two bulk copies, one barrier)
        const uint32_t sbytes = (uint32_t)((b - a) * (p.K >> 5) * 2);
        const unsigned char * ssrc = p.ws + (size_t) a * (p.K >> 5) * 2;
        if (q4_staged(bytes, sbytes, ssrc)) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(bar, bytes + sbytes);
            tma_bulk_g2s_stream(dst, p.w + (size_t) a * p.row_bytes, bytes, bar, s_bc.policy);
            tma_bulk_g2s_stream(dst + bytes, ssrc, sbytes, bar, s_bc.policy);
        } else {
            mbar_arrive(bar);
        }
        return;
    }
    if (bytes != 0 && bytes <= (uint32_t) kHalfSlotBytes) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // this half was just read through the generic proxy
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s_stream(dst, p.w + (size_t) a * p.row_bytes, bytes, bar, s_bc.policy);
    } else {
        mbar_arrive(bar);
    }
}

// bytes of this warp's half of the staging slot that `phase` occupies (what stage_rows copies there)
__device__ __forceinline__ uint32_t staged_bytes_of(int phase, int warp) {
    const PhaseSched p = sched_tab()[phase];
    int a, b; warp_rows(p, warp, a, b);
    const uint32_t bytes = (uint32_t)((b - a) * p.row_bytes);
    if (p.ws) {
        const uint32_t sbytes = (uint32_t)((b - a) * (p.K >> 5) * 2);
        return q4_staged(bytes, sbytes, p.ws + (size_t) a * (p.K >> 5) * 2) ? bytes + sbytes : 0u;
    }
    return bytes <= (uint32_t) kHalfSlotBytes ? bytes : 0u;
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const float * src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// This warp's rows of `phase`: lane-order dot against the shared activation operand; outputs are published with epoch
// `otag` (or stored, for the logits).  Then the rows of the phase after next start streaming in.  No block-wide synchronisation.
template <typename WT, bool TM>
__device__ __noinline__ void run_phase(int phase, int ep, int layer, uint32_t otag, int sb) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tb = sb == 3 ? 0 : sb == 18 ? 8 : sb == 24 ? 16 : 24;
    tstamp2<TM>(32, tb + 0);
    const PhaseSched p = sched_tab()[phase];
    const float * act = reinterpret_cast<const float *>(dsm + SmemLayout::act);
    const float * xs = reinterpret_cast<const float *>(dsm + SmemLayout::x);
    const int half = phase & 1;
    int a, b; warp_rows(p, warp, a, b);
    const uint32_t bytes = (uint32_t)((b - a) * p.row_bytes);
    const bool staged = bytes != 0 && bytes <= (uint32_t) kHalfSlotBytes;
    const unsigned char * slot = dsm + SmemLayout::wslot + (size_t) warp * kWarpSlotBytes + (size_t) half * kHalfSlotBytes;
    mbar_wait(smem_u32(&s_bar[warp][half]), (uint32_t)(phase >> 1) & 1u);
    tstamp<TM>(sb);
    const int E = s_bc.E;
    // one output row: lane 0 publishes / stores it in the form the consumer of this phase expects
    // every lane holds the row's result (lane_tree_reduce): lanes 0..7 write the copies of an all-to-all vector, lane 0 everything else
    auto emit = [&](int r, float v) {
        if (ep == EP_QKV) {
            const size_t slot_off = ((size_t) layer * s_bc.ctx + s_bc.n_past) * E;
            if (r < E) publish_all(s_bc.gq, E, r, v, otag, lane);
            else if (lane == 0) {
                if (r < 2 * E) { publish(s_bc.gk + (r - E), v, otag); s_bc.mem_k[slot_off + (r - E)] = v; }
                else           { publish(s_bc.gv + (r - 2 * E), v, otag); s_bc.mem_v[slot_off + (r - 2 * E)] = v; }
            }
        } else if (ep == EP_RESID) {
            publish_all(s_bc.gx, E, r, __fadd_rn(v, xs[r]), otag, lane);
        } else if (lane == 0) {
            s_bc.logits[r] = v;
        }
    };
    if constexpr (IsQ4<WT>::v) {
        // four adjacent rows per pass (eight lanes per row); operand = the q8 blocks quantize_act_q8 left in shared memory
        const int nb = p.K >> 5;
        const int8_t * aq = reinterpret_cast<const int8_t *>(dsm + SmemLayout::q);
        const float * ad = reinterpret_cast<const float *>(dsm + SmemLayout::part) + 512;
        const uint32_t sbytes = (uint32_t)((b - a) * nb * 2);
        const unsigned char * ssrc = p.ws + (size_t) a * nb * 2;
        const bool st4 = q4_staged(bytes, sbytes, ssrc);
        for (int r = a; r < b; r += 4) {
            const int n = min(4, b - r);
            const float t = st4 ? row_dot_q4<true>(slot + (size_t)(r - a) * p.row_bytes, slot + bytes + (size_t)(r - a) * nb * 2, n, nb, aq, ad, lane)
                                : row_dot_q4<false>(p.w + (size_t) r * p.row_bytes, p.ws + (size_t) r * nb * 2, n, nb, aq, ad, lane);
#pragma unroll
            for (int g = 0; g < 4; g++) {
                const float v = __shfl_sync(0xffffffffu, t, g * 8);
                if (g < n && lane < kReplicas) {
                    if (ep == EP_GELU) publish_all(s_bc.gff, 4 * E, r + g, gelu_sel(v, s_bc.gelu_tab[__half_as_ushort(__float2half_rn(v))]), otag, lane);
                    else emit(r + g, v);
                }
            }
        }
        __syncwarp();
        tstamp<TM>(sb + 1);
        stage_rows(phase + 2);
        tstamp<TM>(sb + 2);
        return;
    } else {
    int j = 0;
    tstamp2<TM>(32, tb + 1);
    for (int r = a; r < b;) {
        const unsigned char * row = staged ? slot + (size_t) j * p.row_bytes : p.w + (size_t) r * p.row_bytes;
        if (r + 1 < b) {                                      // two adjacent rows at once: independent chains, and both table look-ups in flight together
            float v[2];
            if (staged) row_dot<WT, true, 2>(row, p.row_bytes, act, p.K, lane, v);
            else { float u[1]; row_dot<WT, false, 1>(row, p.row_bytes, act, p.K, lane, u); v[0] = u[0]; row_dot<WT, false, 1>(row + p.row_bytes, p.row_bytes, act, p.K, lane, u); v[1] = u[0]; }
            if (v[0] == 1.2345e30f) tstamp2<TM>(32, tb + 7);
            tstamp2<TM>(32, tb + 2);
            if (lane < kReplicas) {
                if (ep == EP_GELU) {
                    const __half t0 = s_bc.gelu_tab[__half_as_ushort(__float2half_rn(v[0]))], t1 = s_bc.gelu_tab[__half_as_ushort(__float2half_rn(v[1]))];
                    publish_all(s_bc.gff, 4 * E, r, gelu_sel(v[0], t0), otag, lane); publish_all(s_bc.gff, 4 * E, r + 1, gelu_sel(v[1], t1), otag, lane);
                } else { emit(r, v[0]); emit(r + 1, v[1]); }
            }
            tstamp2<TM>(32, tb + 3);
            r += 2; j += 2;
        } else {
            float v[1];
            if (staged) row_dot<WT, true, 1>(row, p.row_bytes, act, p.K, lane, v); else row_dot<WT, false, 1>(row, p.row_bytes, act, p.K, lane, v);
            if (v[0] == 1.2345e30f) tstamp2<TM>(32, tb + 7);
            tstamp2<TM>(32, tb + 4);
            if (lane < kReplicas) {
                if (ep == EP_GELU) publish_all(s_bc.gff, 4 * E, r, gelu_sel(v[0], s_bc.gelu_tab[__half_as_ushort(__float2half_rn(v[0]))]), otag, lane);
                else emit(r, v[0]);
            }
            tstamp2<TM>(32, tb + 5);
            r += 1; j += 1;
        }
    }
    __syncwarp();                                             // all lanes are done reading this half
    tstamp<TM>(sb + 1);
    stage_rows(phase + 2);
    tstamp<TM>(sb + 2);
    }
}

}  // namespace

// P2 of a layer (scores) for the CTAs that take score tasks, and P3 (soft_max + P.V) for the CTAs that own a soft_max tile, are real
// calls with their own register allocation.  Inlined into the 128-register kernel body the "prefetched" V values were spilled right after
// each load (LDG -> STL in the SASS: every load waited for its data, on the soft_max CTAs that are the critical path); here they stay
// in registers.
// Where this warp keeps the K rows of its score tasks: the tail of half 0 of its staging slot, behind the rows of the two phases that
// use that half (c_attn and c_fc of every layer: the split of rows over CTAs and warps is the same in every layer).  cap = tasks that fit.
template <int DSTEPS>
__device__ __forceinline__ void key_tail(int warp, uint32_t & off, int & cap) {
    constexpr int D = DSTEPS * 32;
    off = (max(staged_bytes_of(0, warp), staged_bytes_of(2, warp)) + 127u) & ~127u;
    cap = min(2 * kMaxTasks, (int)(((uint32_t) kHalfSlotBytes - min(off, (uint32_t) kHalfSlotBytes)) / (uint32_t)(D * 4)));
}

// Score CTAs, split mode: copy the K rows (older positions) of this warp's score tasks of `layer` into the key tail, asynchronously
// (cp.async, 16 bytes per lane).  Called a whole layer ahead — right after the warp's scores of the previous layer are out, when these
// CTAs have nothing to do but wait for the attention output — so the rows are in shared memory long before q arrives.  (Prefetched into
// registers when q was about to arrive, they came back 1-3 us after q: the scores were the critical path of the layer.)
template <int DSTEPS>
__device__ __noinline__ void p2_stage_keys(int layer, int H, int n_kv, unsigned score_cta0) {
    constexpr int D = DSTEPS * 32, GPT = D / 4;              // 16-byte pieces per task
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = s_bc.E, ctx = s_bc.ctx, n_past = s_bc.n_past;
    uint32_t off; int cap; key_tail<DSTEPS>(warp, off, cap);
    const float * Kc = s_bc.mem_k + (size_t) layer * ctx * E;
    const int total = H * n_past, gw = (int)(blockIdx.x - score_cta0) * kWarps + warp, nw = (int)(gridDim.x - score_cta0) * kWarps;   // tasks = (head, OLDER position)
    const uint32_t dst = smem_u32(dsm + SmemLayout::wslot + (size_t) warp * kWarpSlotBytes + off);
#pragma unroll 2
    for (int q = lane; q < cap * GPT; q += 32) {
        const int i = q / GPT, g = q - i * GPT, t = gw + i * nw;
        if (t < total) {
            const int h = t / n_past, k = t - h * n_past;
            cp_async_16(dst + (uint32_t) q * 16u, Kc + (size_t) k * E + h * D + g * 4);
        }
    }
    cp_async_commit();
}

// P2 of a layer (scores) for the CTAs that take score tasks, and P3 (soft_max + P.V) for the CTAs that own a soft_max tile, are real
// calls with their own register allocation.  Inlined into the 128-register kernel body the "prefetched" K / V values were spilled right
// after each load (LDG -> STL in the SASS: every load waited for its data, on the soft_max CTAs that are the critical path); now neither
// lives in registers at all.
// Task i of this warp is t = gw + i * nw = (h, k); (h, k) advance incrementally (one division for the stride instead of two per task; a
// float-reciprocal divmod per task spills in this kernel).  Eight dot products at a time are reduced
// TOGETHER by a transposed butterfly: stage xor 16 swaps half of the eight partials, xor 8 a quarter, xor 4 one, then xor 1 / xor 2 on
// the single survivor — per task exactly the additions of lane_tree_reduce (each add sees the same two values, addition is commutative),
// 11 shuffles instead of 40, and eight lanes publish the eight scores at once.
template <int DSTEPS, bool TM>
__device__ __noinline__ void p2_scores(int il, int H, int n_kv, uint32_t t_qkv, uint32_t t_sc, unsigned score_cta0) {
    constexpr int D = DSTEPS * 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = s_bc.E, ctx = s_bc.ctx, n_past = s_bc.n_past;
    const float scale = s_bc.scale;
    float * qs = reinterpret_cast<float *>(dsm + SmemLayout::q);
    const float * Kc = s_bc.mem_k + (size_t) il * ctx * E;
    // tasks t = gw + i * nw over (head, OLDER position) = (t / n_past, t % n_past); the H scores of the NEW position (its key arrives through
    // the exchange) are one extra task each for the first H warps — kept out of the loop below: with the poll of the exchange word inlined
    // sixteen times the loop was ~400 instructions per batch and sixteen warps per SM issue every one of them
    const int total = H * n_past, gw = (int)(blockIdx.x - score_cta0) * kWarps + warp, nw = (int)(gridDim.x - score_cta0) * kWarps;
    const int sq = nw / n_past, sr = nw - sq * n_past;
    uint32_t off; int cap; key_tail<DSTEPS>(warp, off, cap);
    if (score_cta0 == 0) cap = 0;                            // unsplit mode: the K rows were not staged
    const float * ks = reinterpret_cast<const float *>(dsm + SmemLayout::wslot + (size_t) warp * kWarpSlotBytes + off) + lane;   // task i, chain step c: ks[i * D + c * 32]
    tstamp<TM>(6);
    consume_to_smem<2>(s_bc.gq, E, t_qkv, qs, SINK_PLAIN, XT_Q);
    tstamp<TM>(7);
    if (cap > 0) { cp_async_wait_all(); __syncwarp(); }      // the warp reads back only what its own lanes copied
    int h = gw / n_past, k = gw - h * n_past;                // task 0
    int done = 0;                                            // tasks handled through the staged rows
#pragma unroll 1
    for (int b0 = 0; b0 < cap && gw + b0 * nw < total; b0 += kMaxTasks) {
        float r[kMaxTasks];
#pragma unroll
        for (int i = 0; i < kMaxTasks; i++) {
            float acc = 0.0f;
            if (b0 + i < cap && h < H) {
#pragma unroll
                for (int c = 0; c < DSTEPS; c++) acc = __fmaf_rn(ks[(b0 + i) * D + c * 32], qs[h * D + c * 32 + lane], acc);
            }
            r[i] = acc;
            k += sr; h += sq; if (k >= n_past) { k -= n_past; h++; }
        }
        static_assert(kMaxTasks == 8, "the transposed butterfly below is written for eight tasks");
        const bool u16 = (lane & 16) != 0, u8 = (lane & 8) != 0, u4 = (lane & 4) != 0;
#pragma unroll
        for (int i = 0; i < 4; i++) { const float keep = u16 ? r[i + 4] : r[i], send = u16 ? r[i] : r[i + 4]; r[i] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, 16)); }
#pragma unroll
        for (int i = 0; i < 2; i++) { const float keep = u8 ? r[i + 2] : r[i], send = u8 ? r[i] : r[i + 2]; r[i] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, 8)); }
        { const float keep = u4 ? r[1] : r[0], send = u4 ? r[0] : r[1]; r[0] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, 4)); }
        r[0] = __fadd_rn(r[0], __shfl_xor_sync(0xffffffffu, r[0], 1));
        r[0] = __fadd_rn(r[0], __shfl_xor_sync(0xffffffffu, r[0], 2));
        const int mine = b0 + (u16 ? 4 : 0) + (u8 ? 2 : 0) + (u4 ? 1 : 0);     // the task whose complete sum this lane holds
        const int t = gw + mine * nw;
        if ((lane & 3) == 0 && mine < cap && t < total) {
            const int hh = t / n_past, kk = t - hh * n_past;
            publish(s_bc.gscores + (size_t) hh * ctx + kk, __fmul_rn(r[0], scale), t_sc);
        }
        done = min(b0 + kMaxTasks, cap);
    }
#pragma unroll 1
    for (int t = gw + done * nw; t < total; t += nw) {       // tasks beyond the staged ones (none for bark-small; small grids, unsplit mode): straight from global memory
        const int hh = t / n_past, kk = t - hh * n_past;
        float acc = 0.0f;
#pragma unroll
        for (int c = 0; c < DSTEPS; c++) acc = __fmaf_rn(__ldcg(Kc + (size_t) kk * E + hh * D + c * 32 + lane), qs[hh * D + c * 32 + lane], acc);
        const float rr = lane_tree_reduce(acc);
        if (lane == 0) publish(s_bc.gscores + (size_t) hh * ctx + kk, __fmul_rn(rr, scale), t_sc);
    }
#pragma unroll 1
    for (int hh = gw; hh < H; hh += nw) {                    // the new position against itself, head hh
        float acc = 0.0f;
#pragma unroll
        for (int c = 0; c < DSTEPS; c++) acc = __fmaf_rn(consume1(s_bc.gk + hh * D + c * 32 + lane, t_qkv), qs[hh * D + c * 32 + lane], acc);
        const float rr = lane_tree_reduce(acc);
        if (lane == 0) publish(s_bc.gscores + (size_t) hh * ctx + n_past, __fmul_rn(rr, scale), t_sc);
    }
}

// soft_max of one score row (ggml.c:13953-14042), block-wide, shared by the decode step and decode_rows_kernel: leaves
// exp(p[k] - max) in p[0, n_kv) and returns 1/sum, the factor ggml_vec_scale_f32 applies (the probabilities are formed where they
// are used).  red: the reduction scratch (its broadcast slots included); fallbacks[1] counts rows whose 1/sum needed the sequential
// replay (fallbacks may be null).
template <bool TM>
__device__ __forceinline__ float softmax_exp_rcp(float * p, int n_kv, double * red, unsigned * fallbacks) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float * bc = reinterpret_cast<float *>(red + kWarps + kWarps / 2 + kWarps);
    float mx = __int_as_float(0xff800000);
#pragma unroll 1
    for (int i = tid; i < n_kv; i += kThreads) mx = fmaxf(mx, p[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float * fred = reinterpret_cast<float *>(red);
    if (lane == 0) fred[warp] = mx;
    __syncthreads();
    mx = fred[0];
#pragma unroll
    for (int w = 1; w < kWarps; w++) mx = fmaxf(mx, fred[w]);
    tstamp<TM>(11);
    // exp: whole chunks of 8 through the vector polynomial (ggml.c:2706-2746), the n_kv % 8 tail through libm expf
    // (ggml.c:2880-2884) — one element per thread, every element independent of the others
    const int nchunks = n_kv >> 3, n8 = nchunks << 3;
#pragma unroll 1
    for (int i = tid; i < n_kv; i += kThreads) {
        const float d = __fsub_rn(p[i], mx);
        p[i] = i < n8 ? ggml_v_expf_dev(d) : glibc_expf_dev(d);
    }
    __syncthreads();
    tstamp<TM>(12);
    // sum = sequential double accumulation of the chunk sums (in-chunk float tree of the 8-wide vector code), then the
    // tail (ggml.c:2845-2888).  All terms are positive, so a tree sum S brackets the sequential one within
    // +-2n*2^-53*S; if 1/sum rounds to the same float at both ends of the bracket the order cannot matter, else replay
    // sequentially.  Done by warp 0, broadcast through bc[2].
    if (warp == 0) {
        auto chunk_sum = [&](int c) {
            const float4 lo4 = *reinterpret_cast<const float4 *>(p + c * 8), hi4 = *reinterpret_cast<const float4 *>(p + c * 8 + 4);
            const float t0 = __fadd_rn(hi4.x, lo4.x), t1 = __fadd_rn(hi4.y, lo4.y), t2 = __fadd_rn(hi4.z, lo4.z), t3 = __fadd_rn(hi4.w, lo4.w);
            return __fadd_rn(__fadd_rn(t0, t2), __fadd_rn(t1, t3));
        };
        double s = 0.0;
#pragma unroll 1
        for (int c = lane; c < nchunks; c += 32) s += (double) chunk_sum(c);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) {
            const double dl = 2.0 * (double)(nchunks + 8) * 0x1p-53 * s * (1.0 + 1e-6);
            double lo = s - dl, hi = s + dl;
#pragma unroll 1
            for (int i = n8; i < n_kv; i++) { const double tl = (double) p[i]; lo = __dadd_rn(lo, tl); hi = __dadd_rn(hi, tl); }
            // 1/sum without a double division: y ~ 1/mid to 2^-50, the bracket [lo, hi] and that error go into the half-width
            const double mid = 0.5 * (lo + hi), y = approx_rcp(mid);
            const double rw = (hi - lo) * y * 0.5 + 0x1p-48;                       // relative half-width
            float f_lo = __double2float_rn(y * (1.0 - rw));
            const float f_hi = __double2float_rn(y * (1.0 + rw));
            if (f_lo != f_hi) {
                double q2 = 0.0;
#pragma unroll 1
                for (int c = 0; c < nchunks; c++) q2 = __dadd_rn(q2, (double) chunk_sum(c));
#pragma unroll 1
                for (int i = n8; i < n_kv; i++) q2 = __dadd_rn(q2, (double) p[i]);
                f_lo = __double2float_rn(__ddiv_rn(1.0, q2));
                if (fallbacks) atomicAdd(fallbacks + 1, 1u);
            }
            bc[2] = f_lo;
        }
    }
    __syncthreads();
    tstamp<TM>(13);
    return bc[2];
}

template <int DSTEPS, bool TM>
__device__ __noinline__ void p3_attention(int il, int n_kv, uint32_t t_qkv, uint32_t t_sc, uint32_t t_att, unsigned * ln_fallbacks) {
    constexpr int D = DSTEPS * 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = s_bc.E, ctx = s_bc.ctx, n_past = s_bc.n_past;
    float * act = reinterpret_cast<float *>(dsm + SmemLayout::act);
    float * qs = reinterpret_cast<float *>(dsm + SmemLayout::q);
    float * part = reinterpret_cast<float *>(dsm + SmemLayout::part);
    double * red = reinterpret_cast<double *>(dsm + SmemLayout::red);
    struct { float * mem_v; unsigned * ln_fallbacks; } A{s_bc.mem_v, ln_fallbacks};
    // V of older positions.  Thread (v, dd) owns virtual lane v of output column dd: chain steps k = v + 32 c.  A warp holds two values of
    // v and all 16 columns, i.e. per chain step two 64-byte pieces of V rows — and copies exactly those, ASYNCHRONOUSLY (cp.async, 16 bytes per
    // lane: one instruction moves four chain steps of the warp), into the unused tail of its own staging half: half 1 holds the warp's
    // c_proj rows right now, at most a third of it.  The copies drain while the scores are computed elsewhere and cost neither registers
    // nor waiting.  (Held in registers, the 33 values were spilled right after each load — LDG -> STL in the SASS, every load waiting for
    // its data, on exactly the CTAs that are the critical path.)
    // When the tail is too small (f32 weights and a long context) the P.V loop loads from global memory itself.
    constexpr int parts = D >> 4;                            // CTAs per head: CTA c owns columns [16 (c % parts), +16) of head c / parts
    const int pv_h = blockIdx.x / parts, pv_c = blockIdx.x % parts, np = n_kv & ~31;
    const int v = tid >> 4, dd = tid & 15, h = pv_h;
    const int col0 = pv_h * D + pv_c * 16;
    const int nstep = np >> 5, r = n_kv - np;
    const int nstep_all = nstep + (r > 0 ? 1 : 0);           // the leftover rows k = np + v are chain step `nstep` of the same layout
    const float * Vt = A.mem_v + (size_t) il * ctx * E + col0;       // row k of the tile: Vt + k * E, 16 floats
    const uint32_t voff = (staged_bytes_of(4 * il + 1, warp) + 127u) & ~127u;
    const bool vs_ok = voff + (uint32_t) nstep_all * 128u <= (uint32_t) kHalfSlotBytes;
    const float * vs = reinterpret_cast<const float *>(dsm + SmemLayout::wslot + (size_t) warp * kWarpSlotBytes + kHalfSlotBytes + voff);   // [step][2 x 16] floats
    if (vs_ok) {
        const uint32_t dst = smem_u32(vs);
        const int sub = lane >> 3, vl2 = (lane >> 2) & 1, g = lane & 3;        // lane: chain step within a group of four, which of the warp's two rows, 16-byte piece of the row
#pragma unroll 2
        for (int c0 = 0; c0 < nstep_all; c0 += 4) {
            const int c = c0 + sub, k = 2 * warp + vl2 + 32 * c;
            if (c < nstep_all && k < n_past) cp_async_16(dst + (uint32_t)(((c * 2 + vl2) * 16 + g * 4) * 4), Vt + (size_t) k * E + g * 4);
        }
        cp_async_commit();
    }
    const float v_new = consume1(s_bc.gv + col0 + dd, t_qkv);     // value row of the new position
    __syncthreads();                                         // slower warps may still be reading q (in `qs`) for their score tasks
    tstamp<TM>(9);
    float * p = qs;                                          // scores row -> exp(score - max); the 1/sum factor is applied on use
    consume_row_to_smem(s_bc.gscores + (size_t) h * ctx, n_kv, t_sc, p);
    tstamp<TM>(10);
    const float sc_f = softmax_exp_rcp<TM>(p, n_kv, red, A.ln_fallbacks);    // probabilities = p[k] * sc_f, formed where they are used
    float acc = 0.0f;
    if (vs_ok) {
        cp_async_wait_all(); __syncwarp();                   // the warp reads back only what its own lanes copied
#pragma unroll 8
        for (int c = 0; c < nstep; c++) {
            const int k = v + 32 * c;
            const float vv = k < n_past ? vs[c * 32 + lane] : v_new;       // (a slot that was not copied holds stale bytes: read, not used)
            acc = __fmaf_rn(vv, __fmul_rn(p[k], sc_f), acc);
        }
    } else {
#pragma unroll 8
        for (int c = 0; c < nstep; c++) {
            const int k = v + 32 * c;
            const float vv = k < n_past ? __ldcg(Vt + (size_t) k * E + dd) : v_new;
            acc = __fmaf_rn(vv, __fmul_rn(p[k], sc_f), acc);
        }
    }
    part[v * 17 + dd] = acc;                                 // (row stride 17: conflict-free for this store and for the column reads below)
    // leftovers k = np .. n_kv-1 as the pinned build compiles them (oracle orc_vec_dot_f32): 8-groups and a 4-group of
    // rounded multiply + add, then <= 3 fused multiply-adds.  Thread (v, dd) prepares term v: the rounded product where
    // the chain adds one, the bare value where it fuses.
    const int r8 = r & ~7, n4 = r8 + ((r - r8) >= 4 ? 4 : 0);
    if (v < r) {
        const float vv = (np + v < n_past) ? (vs_ok ? vs[nstep * 32 + lane] : __ldcg(Vt + (size_t)(np + v) * E + dd)) : v_new;
        act[v * 16 + dd] = v < n4 ? __fmul_rn(vv, __fmul_rn(p[np + v], sc_f)) : vv;
    }
    __syncthreads();
    tstamp<TM>(15);
    {
        // warp w finishes output column w: lane l holds virtual lane l's partial, the shuffle tree is lane_tree_reduce (the reference's
        // order); every lane then runs the short leftover chain on the same values, and lanes 0..7 store the eight copies of the result
        float sum = lane_tree_reduce(part[lane * 17 + warp]);
#pragma unroll 8
        for (int j = 0; j < n4; j++) sum = __fadd_rn(sum, act[j * 16 + warp]);            // (16 warps run this at once: keep it to a load and an add per step)
#pragma unroll 1
        for (int j = n4; j < r; j++) sum = __fmaf_rn(act[j * 16 + warp], __fmul_rn(p[np + j], sc_f), sum);
        publish_all(s_bc.gatt, E, col0 + warp, sum, t_att, lane);
    }
    __syncthreads();                                     // `act` / `qs` are reused by the next phase
}

template <typename WT, int DSTEPS, bool TM>
__global__ void __launch_bounds__(kThreads, 1) gpt_decode_step_kernel(DecodeArgs A) {
    float * act = reinterpret_cast<float *>(dsm + SmemLayout::act);
    float * xs = reinterpret_cast<float *>(dsm + SmemLayout::x);
    float * qs = reinterpret_cast<float *>(dsm + SmemLayout::q);
    float * part = reinterpret_cast<float *>(dsm + SmemLayout::part);
    double * red = reinterpret_cast<double *>(dsm + SmemLayout::red);
    float * bc = reinterpret_cast<float *>(red + kWarps + kWarps / 2 + kWarps);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int D = DSTEPS * 32;
    const int E = A.E, H = A.H, L = A.L, ctx = A.block_size, n_past = A.n_past, n_kv = n_past + 1;
    constexpr bool kQ4 = IsQ4<WT>::v;
    constexpr bool kRound = !kQ4 && sizeof(WT) == 2;
    constexpr int kSinkAct = kQ4 ? SINK_PLAIN : kRound ? SINK_ACT_R16 : SINK_ACT;     // q4_0: the f32 vector in natural order, quantised to q8 blocks below
    int8_t * act_q = reinterpret_cast<int8_t *>(dsm + SmemLayout::q);                  // q4_0 operand: aliases the q / probabilities row (free during the row phases)
    float * act_d = reinterpret_cast<float *>(dsm + SmemLayout::part) + 512;

    // ---- per-CTA row ranges, block context and the staging barriers in shared memory ----
    PhaseSched * sched = reinterpret_cast<PhaseSched *>(dsm + SmemLayout::sched);
    const int n_phases = 4 * L + 1;
    if (tid < n_phases) {
        const DecodePhase ph = A.phases[tid];
        int lo = 0, hi = ph.n_out;
        if (tid == n_phases - 1) { lo = A.lm_lo; hi = A.lm_hi; }
        const int n = hi - lo, G = gridDim.x, base = n / G, rem = n % G, cta = blockIdx.x;
        PhaseSched e;
        e.r0 = lo + cta * base + min(cta, rem); e.r1 = e.r0 + base + (cta < rem ? 1 : 0);      // balanced split: floor or ceil of n / G rows
        e.K = ph.K; e.row_bytes = ph.row_bytes; e.w = (const unsigned char *) ph.w; e.ws = (const unsigned char *) ph.ws;
        sched[tid] = e;
    }
    if (tid == kThreads - 1) {
        s_bc.gq = (tagged_t *) A.gq; s_bc.gk = (tagged_t *) A.gk; s_bc.gv = (tagged_t *) A.gv; s_bc.gx = (tagged_t *) A.gx; s_bc.gff = (tagged_t *) A.gff;
        s_bc.gatt = (tagged_t *) A.gatt; s_bc.gscores = (tagged_t *) A.gscores;
        s_bc.mem_k = A.mem_k; s_bc.mem_v = A.mem_v; s_bc.logits = A.logits; s_bc.gelu_tab = A.gelu_tab;
        s_bc.policy = l2_evict_first_policy();
        s_bc.E = E; s_bc.ctx = ctx; s_bc.n_past = n_past; s_bc.n_phases = n_phases; s_bc.scale = 1.0f / sqrtf((float) E / (float) H);
        s_tim = A.timing; s_tim_layer = 0; s_tim_tid = A.timing_tid; s_poll_ns = A.poll_ns;
    }
    if (tid < XT_COUNT) {                                    // head starts (CTAs with a soft_max tile reach the att exchange right behind their own tile)
        const bool pv = (int) blockIdx.x < A.H * ((A.E / A.H) >> 4);
        s_headstart[tid] = (tid == XT_ATT && pv) ? 0u : A.headstart[tid];
    }
    if (lane == 0) {
        mbar_init(smem_u32(&s_bar[warp][0]), 1); mbar_init(smem_u32(&s_bar[warp][1]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    stage_rows(0);
    stage_rows(1);

    embed_token<WT>(A.wte, A.wpe, A.token_ptr, A.token, A.n_vocab_in, E, n_past, xs);
    __syncthreads();

    uint32_t tag = A.tag_base;                               // unique epoch per exchange; the host advances the base by 6 * L per launch
    const double inv_E = A.inv_E;

    const int parts = D >> 4;                                // P3: CTAs per head
    const bool pv_cta = (int) blockIdx.x < H * parts;
    const unsigned score_cta0 = (gridDim.x >= (unsigned)(H * parts + 64)) ? (unsigned)(H * parts) : 0u;      // first CTA that takes score tasks
    const bool score_cta = blockIdx.x >= score_cta0;

    // split mode (score_cta0 != 0): the score CTAs' staging tails are free for K rows (the soft_max CTAs keep V tiles in theirs)
    if (score_cta0 != 0 && score_cta) p2_stage_keys<DSTEPS>(0, H, n_kv, score_cta0);
#pragma unroll 1
    for (int il = 0; il < L; il++) {
        const DecodeLayerVec lv = A.layer_vecs[il];
        const uint32_t t_qkv = tag + 1, t_sc = tag + 2, t_att = tag + 3, t_x1 = tag + 4, t_ff = tag + 5, t_x2 = tag + 6;
        tag += 6;
        if (tid == A.timing_tid) s_tim_layer = il;           // (the stamping thread is the only reader)
        tstamp<TM>(0);
        // ---- P1: LN1 -> QKV ----
        block_layernorm<kRound, TM, kQ4>(xs, E, inv_E, lv.ln_1_g, lv.ln_1_b, act, red, A.ln_fallbacks, 1);
        if constexpr (kQ4) quantize_act_q8(act, E, act_q, act_d);
        tstamp<TM>(2);
        run_phase<WT, TM>(4 * il + 0, EP_QKV, il, t_qkv, 3);

        // ---- P2 (scores) and P3 (soft_max + P.V), out of line (see p2_scores).  The CTAs that own a soft_max tile take no score tasks when
        // enough other CTAs exist: they are the critical path of the layer (they still have the whole of P3 to do once the scores exist) ----
        if constexpr (kQ4) __syncthreads();                    // the q8 operand aliases `qs`: every warp must be done with its QKV rows before q lands there
        if (score_cta) {
            p2_scores<DSTEPS, TM>(il, H, n_kv, t_qkv, t_sc, score_cta0);
            tstamp<TM>(8);
            if (score_cta0 != 0 && il + 1 < L) p2_stage_keys<DSTEPS>(il + 1, H, n_kv, score_cta0);      // next layer's K rows: these CTAs only wait for the attention output now
        } else {
            tstamp<TM>(8);
        }
        if (pv_cta) p3_attention<DSTEPS, TM>(il, n_kv, t_qkv, t_sc, t_att, A.ln_fallbacks);
        tstamp<TM>(16);

        // ---- P4: c_proj + residual ----
        consume_to_smem<2>(s_bc.gatt, E, t_att, act, kSinkAct, XT_ATT);    // (CTAs without a soft_max tile would otherwise poll for the whole of P3)
        if constexpr (kQ4) quantize_act_q8(act, E, act_q, act_d);
        tstamp<TM>(17);
        run_phase<WT, TM>(4 * il + 1, EP_RESID, il, t_x1, 18);

        // ---- P5: LN2 -> c_fc -> GELU ----
        consume_to_smem<2>(s_bc.gx, E, t_x1, xs, SINK_PLAIN, XT_X1);
        tstamp<TM>(21);
        block_layernorm<kRound, TM, kQ4>(xs, E, inv_E, lv.ln_2_g, lv.ln_2_b, act, red, A.ln_fallbacks, 22);
        if constexpr (kQ4) quantize_act_q8(act, E, act_q, act_d);
        tstamp<TM>(23);
        run_phase<WT, TM>(4 * il + 2, EP_GELU, il, t_ff, 24);
        __syncthreads();                                         // the ff vector lands in `act`, which slower warps may still be reading
        tstamp<TM>(27);

        // ---- P6: mlp/c_proj + residual ----
        consume_to_smem<8>(s_bc.gff, 4 * E, t_ff, act, kSinkAct, XT_FF);
        if constexpr (kQ4) quantize_act_q8(act, 4 * E, act_q, act_d);
        tstamp<TM>(28);
        run_phase<WT, TM>(4 * il + 3, EP_RESID, il, t_x2, 29);

        consume_to_smem<2>(s_bc.gx, E, t_x2, xs, SINK_PLAIN, XT_X2);
    }
    if (tid == A.timing_tid) s_tim_layer = L;                 // row L: start of the final norm
    // ---- final norm + lm_head window ----
    tstamp<TM>(0);
    block_layernorm<kRound, TM, kQ4>(xs, E, inv_E, A.ln_f_g, A.ln_f_b, act, red, A.ln_fallbacks, 1);
    if constexpr (kQ4) quantize_act_q8(act, E, act_q, act_d);
    tstamp<TM>(2);
    run_phase<WT, TM>(4 * L, EP_LOGITS, 0, 0, 3);
}

// The decode kernels' two row reductions on their own, one CTA of kThreads per row (bark_b200_parity_rows): op 0 = block_layernorm
// (natural column order, no f16 rounding), op 1 = softmax_exp_rcp with the probabilities formed as P.V forms them.  counters[0] counts
// LayerNorm replays, counters[1] soft_max replays.
__global__ void __launch_bounds__(kThreads) decode_rows_kernel(int op, const float * __restrict__ x, int n, double inv_n, const float * __restrict__ g,
                                                               const float * __restrict__ b, float * __restrict__ out, unsigned * counters) {
    __shared__ double red[kWarps + kWarps / 2 + kWarps + 4];
    __shared__ __align__(16) float p[1024];
    const float * xr = x + (size_t) blockIdx.x * n;
    float * orow = out + (size_t) blockIdx.x * n;
    if (op == 0) { block_layernorm<false, false, true, 1>(xr, n, inv_n, g, b, orow, red, counters, 1); return; }
    for (int i = threadIdx.x; i < n; i += kThreads) p[i] = xr[i];
    __syncthreads();
    const float sc_f = softmax_exp_rcp<false>(p, n, red, counters);
    for (int i = threadIdx.x; i < n; i += kThreads) orow[i] = __fmul_rn(p[i], sc_f);
}

void decode_rows(int op, const float * x, int rows, int n, const float * g, const float * b, float * out, unsigned * counters, cudaStream_t s) {
    BARK_LAUNCH(decode_rows_kernel, rows, kThreads, 0, s, op, x, n, 1.0 / n, g, b, out, counters);
}

// The decode step's q4_0 pieces on their own (bark_b200_quant_matmul paths 1 and 2), one CTA: quantize_act_q8 of one row into shared
// memory, then every warp takes four rows at a time through row_dot_q4.  SH: the warp first copies them into its own slot in the layout
// stage_rows leaves (the rows' nibble words, then their f16 scales); otherwise they are read from global memory.
template <bool SH>
__global__ void __launch_bounds__(kThreads) decode_q4_rows_kernel(const float * __restrict__ x, int K, const unsigned char * __restrict__ wq,
                                                                  const unsigned char * __restrict__ ws, int n_out, MatmulEpilogue ep,
                                                                  int8_t * __restrict__ q_out, float * __restrict__ d_out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nb = K >> 5;
    int8_t * aq = reinterpret_cast<int8_t *>(dsm);
    float * ad = reinterpret_cast<float *>(dsm + K);
    unsigned char * slot = dsm + K + nb * 4 + (size_t) warp * 4 * nb * 18;
    quantize_act_q8(x, K, aq, ad);
    for (int i = threadIdx.x; i < K; i += kThreads) q_out[i] = aq[i];
    for (int i = threadIdx.x; i < nb; i += kThreads) d_out[i] = ad[i];
    for (int r = warp * 4; r < n_out; r += kWarps * 4) {
        const int n = min(4, n_out - r);
        float t;
        if constexpr (SH) {
            const uint32_t * src = reinterpret_cast<const uint32_t *>(wq + (size_t) r * nb * 16);
            const unsigned short * ssrc = reinterpret_cast<const unsigned short *>(ws + (size_t) r * nb * 2);
            for (int i = lane; i < n * nb * 4; i += 32) reinterpret_cast<uint32_t *>(slot)[i] = src[i];
            for (int i = lane; i < n * nb; i += 32) reinterpret_cast<unsigned short *>(slot + n * nb * 16)[i] = ssrc[i];
            __syncwarp();
            t = row_dot_q4<true>(slot, slot + n * nb * 16, n, nb, aq, ad, lane);
            __syncwarp();
        } else {
            t = row_dot_q4<false>(wq + (size_t) r * nb * 16, ws + (size_t) r * nb * 2, n, nb, aq, ad, lane);
        }
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const float v = __shfl_sync(0xffffffffu, t, g * 8);
            if (lane == 0 && g < n) matmul_epilogue(ep, 0, r + g, v);
        }
    }
}

void decode_q4_rows(bool staged, const float * x, int K, const void * qs, const void * scales, int n_out, const MatmulEpilogue & ep, int8_t * q_out,
                    float * d_out, cudaStream_t s) {
    const size_t smem = (size_t) K + (K >> 5) * 4 + (staged ? (size_t) kWarps * 4 * (K >> 5) * 18 : 0);
    const unsigned char * wq = (const unsigned char *) qs, * ws = (const unsigned char *) scales;
    if (staged) {
        BARK_CUDA_CHECK(cudaFuncSetAttribute(decode_q4_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
        BARK_LAUNCH(decode_q4_rows_kernel<true>, 1, kThreads, smem, s, x, K, wq, ws, n_out, ep, q_out, d_out);
    } else {
        BARK_LAUNCH(decode_q4_rows_kernel<false>, 1, kThreads, smem, s, x, K, wq, ws, n_out, ep, q_out, d_out);
    }
}

static size_t decode_smem_bytes() { return (size_t) SmemLayout::total + 128; }

int decode_tags_per_step(int n_layer) { return 6 * n_layer; }

template <typename WT, int DSTEPS, bool TM>
static void launch_variant(DecodeArgs a, int n_sm, cudaStream_t s) {
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured))
        BARK_CUDA_CHECK(cudaFuncSetAttribute(gpt_decode_step_kernel<WT, DSTEPS, TM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) decode_smem_bytes()));
    void * kargs[] = {(void *) &a};
    BARK_CUDA_CHECK(cudaLaunchCooperativeKernel((const void *) gpt_decode_step_kernel<WT, DSTEPS, TM>, dim3(n_sm), dim3(kThreads), kargs, decode_smem_bytes(), s));
}
template <typename WT, int DSTEPS>
static void launch_one(DecodeArgs a, int n_sm, cudaStream_t s) {
    if (a.timing) launch_variant<WT, DSTEPS, true>(a, n_sm, s); else launch_variant<WT, DSTEPS, false>(a, n_sm, s);   // stamps exist only in the BARK_B200_DECODE_TIMING build of the kernel
}

void launch_decode_step(const DecodeArgs & args, WType wt, int n_sm, cudaStream_t s) {
    const int dsteps = args.E / args.H / 32;
    if (g_prof_on) prof_begin("gpt_decode_step_kernel", s, g_next_bytes, g_next_flops);
    if (wt == W_Q4_0) {
        switch (dsteps) { case 1: launch_one<Q4, 1>(args, n_sm, s); break; case 2: launch_one<Q4, 2>(args, n_sm, s); break;
                          case 3: launch_one<Q4, 3>(args, n_sm, s); break; default: launch_one<Q4, 4>(args, n_sm, s); }
    } else if (wt == W_F16) {
        switch (dsteps) { case 1: launch_one<__half, 1>(args, n_sm, s); break; case 2: launch_one<__half, 2>(args, n_sm, s); break;
                          case 3: launch_one<__half, 3>(args, n_sm, s); break; default: launch_one<__half, 4>(args, n_sm, s); }
    } else {
        switch (dsteps) { case 1: launch_one<float, 1>(args, n_sm, s); break; case 2: launch_one<float, 2>(args, n_sm, s); break;
                          case 3: launch_one<float, 3>(args, n_sm, s); break; default: launch_one<float, 4>(args, n_sm, s); }
    }
    if (g_prof_on) prof_end(s);
    g_next_bytes = g_next_flops = 0.0;
    ++g_kernel_launches;
}

}  // namespace bark
