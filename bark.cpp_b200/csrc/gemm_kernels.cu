// Register-tiled lane-order kernels for the multi-row passes: prefill of the causal models (257 / <=887 rows) and the
// fine model's 1024-row passes (bark.cpp:1416-1584) — the dense contractions of the hot path.
//
// Bit-exactness fixes the shape of the tiling: every output element is 32 lane partials (common.cuh "Lane order"),
// each a serial FMA chain over k = v, v+32, ..., so a warp's 32 lanes all work on the SAME outputs — lane v owns
// virtual lane v of an 8 x 8 output tile (64 accumulators per lane, 2048 per warp).  Operand reuse therefore comes
// from registers (each converted operand feeds 8 FMAs) and shared memory (a 32 x 32 or 32 x 16 block tile), not from giving
// different lanes different outputs.  The 32 partials of all 64 outputs are then combined through shared memory and
// lane_tree_reduce_local, or with a transposed butterfly (62 shuffles instead of 64 x 5); both perform exactly the additions
// of GGML_F32x8_REDUCE.
//
// Both operands are in the group-major layout (common.cuh), so a pipeline stage of the block tile is a handful of
// contiguous spans: 2-4 TMA bulk copies into a 4-stage shared-memory ring (mbarrier complete_tx).
#include "epilogue.cuh"
#include "gpt_kernels.h"

#include <algorithm>
#include <string.h>

namespace bark {

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
// atomicAdd with acquire-release semantics at CTA scope: one instruction instead of fence.sc + atomic + fence.sc
__device__ __forceinline__ int atom_add_acq_rel_cta(int * p, int v) {
    int old;
    asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(smem_u32(p)), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void * src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// Combine the 32 lane partials of 64 outputs.  In: r[i] = this lane's partial of output i.  Out: r[0], r[1] = the complete
// sums of outputs base, base+1 with base = (b4<<5)|(b3<<4)|(b2<<3)|(b0<<2)|(b1<<1), b = bits of the lane id.
// Stage order xor 16, 8, 4, 1, 2 = the tree of GGML_F32x8_REDUCE (ggml.c:1405-1422); each add is commutative.
template <int N, int MASK>
__device__ __forceinline__ void butterfly_stage(float (&r)[64], bool upper) {
#pragma unroll
    for (int i = 0; i < N / 2; i++) {
        const float keep = upper ? r[i + N / 2] : r[i];
        const float send = upper ? r[i] : r[i + N / 2];
        r[i] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, MASK));
    }
}
__device__ __forceinline__ int butterfly_reduce64(float (&r)[64], int lane) {
    butterfly_stage<64, 16>(r, (lane & 16) != 0);
    butterfly_stage<32, 8>(r, (lane & 8) != 0);
    butterfly_stage<16, 4>(r, (lane & 4) != 0);
    butterfly_stage<8, 1>(r, (lane & 1) != 0);
    butterfly_stage<4, 2>(r, (lane & 2) != 0);
    return ((lane & 16) << 1) | ((lane & 8) << 1) | ((lane & 4) << 1) | ((lane & 1) << 2) | (lane & 2);
}

constexpr int kStages = 4;
constexpr int kRedLd = 36;       // row stride (floats) of the tile-end reduction scratch: 16-byte reads of 8 consecutive rows hit 8 bank quads

// Block-tile configurations (the `variant` of lane_gemm_tiled): WM x WO warps, each with an 8 x OT output tile, MINB CTAs per SM.
// A stage holds (BM + BO) rows x 512 bytes: 256 columns of f16 (two groups) or 128 columns of f32 (one group).
// PIPE (f16): the operand words of a stage are loaded as 32-bit halves (chain steps 0-1, 2-3), each half one group ahead of the
// FMAs that use it, so the next half's loads are in flight under the current half's FMAs in the same registers.
template <int WM_, int WO_, int OT_, int MINB_, bool PIPE_ = false> struct TileCfg {
    static constexpr int WM = WM_, WO = WO_, OT = OT_, MINB = MINB_;
    static constexpr bool PIPE = PIPE_;
    static constexpr int kWarps = WM * WO, kThreads = 32 * kWarps, kBM = 8 * WM, kBO = OT * WO, kNAcc = 8 * OT;
    static constexpr int kStageBytes = (kBM + kBO) * 512;
    // one CTA per SM leaves room to combine the lane partials through shared memory; two per SM keep the transposed butterfly
    static constexpr bool kSmemReduce = MINB == 1;
    static constexpr size_t kRedOff = ((size_t) kStages * kStageBytes + kStages * 12 + 15) & ~(size_t) 15;
    static constexpr size_t kSmem = kRedOff + (kSmemReduce ? (size_t) kWarps * 32 * kRedLd * 4 : 0);
};
typedef TileCfg<4, 2, 8, 2>  Tile32x16;      // variant 1: 32 x 16, 8 warps of 8 x 8, 2 CTAs per SM (few rows: twice the tiles)
typedef TileCfg<4, 4, 8, 1, true> Tile32x32;  // variant 2: 32 x 32, 16 warps of 8 x 8, 1 CTA per SM, operand loads pipelined (f16)

// lane v's four elements of one row of one 128-column group (group-major layout, common.cuh)
template <typename T> struct QuadOp;
template <> struct QuadOp<__half> {
    typedef uint2 V;
    static constexpr int kGroupsPerStage = 2;
    __device__ __forceinline__ static float elem(const uint2 & u, int c) {       // c is a compile-time constant after unrolling
        const uint32_t w = c < 2 ? u.x : u.y;
        const __half2 h = *reinterpret_cast<const __half2 *>(&w);
        return (c & 1) ? __high2float(h) : __low2float(h);
    }
};
template <> struct QuadOp<float> {
    typedef uint4 V;
    static constexpr int kGroupsPerStage = 1;
    __device__ __forceinline__ static float elem(const uint4 & u, int c) { return __uint_as_float(c == 0 ? u.x : c == 1 ? u.y : c == 2 ? u.z : u.w); }
};

// One 128-column group of a warp's 8 x OT tile: acc[mi * OT + oi] += its 4 chain steps (FULL) or the first `steps` of them (the last
// group of a K that is not a multiple of 128).  ga / gw: lane v's word of the tile's first activation / weight row.
template <typename T, int OT, bool FULL>
__device__ __forceinline__ void fma_group(const unsigned char * ga, const unsigned char * gw, float (&acc)[8 * OT], int steps) {
    typedef typename QuadOp<T>::V QV;
    constexpr int kRowB = kGmGroup * sizeof(T);
    QV pa[8], pw[OT];
#pragma unroll
    for (int mi = 0; mi < 8; mi++) pa[mi] = *reinterpret_cast<const QV *>(ga + mi * kRowB);
#pragma unroll
    for (int oi = 0; oi < OT; oi++) pw[oi] = *reinterpret_cast<const QV *>(gw + oi * kRowB);
#pragma unroll
    for (int c = 0; c < 4; c++) {
        if (FULL || c < steps) {
            float af[8], wf[OT];
#pragma unroll
            for (int mi = 0; mi < 8; mi++) af[mi] = QuadOp<T>::elem(pa[mi], c);
#pragma unroll
            for (int oi = 0; oi < OT; oi++) wf[oi] = QuadOp<T>::elem(pw[oi], c);
#pragma unroll
            for (int mi = 0; mi < 8; mi++)
#pragma unroll
                for (int oi = 0; oi < OT; oi++) acc[mi * OT + oi] = __fmaf_rn(wf[oi], af[mi], acc[mi * OT + oi]);
        }
    }
}

// f16, chain steps 2h and 2h+1 of a group from the h-th 32-bit halves of the operand words (a: 8 activation rows, w: OT weight rows)
template <int OT>
__device__ __forceinline__ void fma_half(const uint32_t (&a)[8], const uint32_t (&w)[OT], float (&acc)[8 * OT]) {
#pragma unroll
    for (int c = 0; c < 2; c++) {
        float af[8], wf[OT];
#pragma unroll
        for (int mi = 0; mi < 8; mi++) { const __half2 h = *reinterpret_cast<const __half2 *>(&a[mi]); af[mi] = c ? __high2float(h) : __low2float(h); }
#pragma unroll
        for (int oi = 0; oi < OT; oi++) { const __half2 h = *reinterpret_cast<const __half2 *>(&w[oi]); wf[oi] = c ? __high2float(h) : __low2float(h); }
#pragma unroll
        for (int mi = 0; mi < 8; mi++)
#pragma unroll
            for (int oi = 0; oi < OT; oi++) acc[mi * OT + oi] = __fmaf_rn(wf[oi], af[mi], acc[mi * OT + oi]);
    }
}
template <int OT>
__device__ __forceinline__ void load_half(const unsigned char * ga, const unsigned char * gw, int h, uint32_t (&a)[8], uint32_t (&w)[OT]) {
#pragma unroll
    for (int mi = 0; mi < 8; mi++) a[mi] = *reinterpret_cast<const uint32_t *>(ga + mi * 256 + h * 4);
#pragma unroll
    for (int oi = 0; oi < OT; oi++) w[oi] = *reinterpret_cast<const uint32_t *>(gw + oi * 256 + h * 4);
}

}  // namespace

// C[m][o] = lane-order dot(act[m], W[o]).  Persistent CTAs walk BM x BO block tiles (o fastest, so CTAs running at the same time
// share activation rows in L2); WM x WO warps, 8 x OT outputs per warp (TileCfg).
//
// Both operands are group-major: for one 128-column group the BM activation rows of a tile are one contiguous span, the BO weight
// rows another, so a pipeline stage is 2 (f32) or 4 (f16) bulk copies issued by ONE thread.  (Row-major operands would need a copy
// per row; the copy instruction takes uniform operands, so the compiler serialises the lanes and the issuing warp - also a
// consumer - falls behind, with the other warps waiting on the `full` barrier.)
//
// The k-steps of ALL of a CTA's tiles form one stream through the 4-stage ring.  Nobody waits to refill a slot: every warp
// bumps the slot's counter when it is done reading (an acquire-release atomic: its reads happen before the refill), and the warp
// whose bump completes a multiple of the warp count issues the copies for stage s + 4.  The counters only grow, so no reset store
// has to be ordered before the next round's bumps.
//
// Tile end: with one CTA per SM each warp writes its partials to its own shared-memory scratch 32 outputs at a time and lane u
// then adds the 32 partials of output u with lane_tree_reduce_local (32 stores + 8 16-byte loads + 31 adds per lane and slice);
// with two CTAs per SM there is no room for the scratch and the transposed butterfly does it in registers.
template <typename T, typename Cfg>
__global__ void __launch_bounds__(Cfg::kThreads, Cfg::MINB) lane_gemm_tiled_kernel(const T * __restrict__ Wg, int K, int w_gs, int O, const T * __restrict__ act, int act_gs, int M, MatmulEpilogue ep) {
    constexpr int GPS = QuadOp<T>::kGroupsPerStage, OT = Cfg::OT, kBM = Cfg::kBM, kBO = Cfg::kBO, kStageBytes = Cfg::kStageBytes;
    constexpr int kRowB = kGmGroup * sizeof(T);              // bytes of one row of one group: 256 (f16) / 512 (f32)
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t full = smem_u32(smem + kStages * kStageBytes);
    int * const cnt = reinterpret_cast<int *>(smem + kStages * kStageBytes + kStages * 8);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / Cfg::WO, wo = warp % Cfg::WO;
    const int nsteps = K >> 5;                                // chain steps per lane
    const int ngroups = (nsteps + 3) >> 2;                    // 128-column groups; the last may be partial
    const int nstages = (ngroups + GPS - 1) / GPS;            // pipeline stages per tile
    const int tiles_o = (O + kBO - 1) / kBO, tiles_m = (M + kBM - 1) / kBM, n_tiles = tiles_o * tiles_m;
    const int my_tiles = ((int) blockIdx.x < n_tiles) ? (n_tiles - 1 - (int) blockIdx.x) / (int) gridDim.x + 1 : 0;
    const int total_steps = my_tiles * nstages;

    if (tid == 0) {
        for (int s = 0; s < kStages; s++) { mbar_init(full + s * 8, 1); cnt[s] = 0; }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int step) {                              // ONE thread: stage `step` of this CTA's stream
        const int ti = step / nstages, sg = step - ti * nstages;
        const int tile = blockIdx.x + ti * gridDim.x;
        const int m0 = (tile / tiles_o) * kBM, o0 = (tile % tiles_o) * kBO;
        const int slot = step % kStages;
        const uint32_t bar = full + slot * 8;
        const int g0 = sg * GPS, ng = min(GPS, ngroups - g0);
        mbar_expect_tx(bar, (uint32_t)(ng * (kBM + kBO) * kRowB));
        const uint32_t dst = smem_u32(smem + (size_t) slot * kStageBytes);
        for (int j = 0; j < ng; j++) {
            tma_bulk_g2s(dst + j * (kBM + kBO) * kRowB, act + (size_t)(g0 + j) * act_gs + (size_t) m0 * kGmGroup, kBM * kRowB, bar);
            tma_bulk_g2s(dst + j * (kBM + kBO) * kRowB + kBM * kRowB, Wg + (size_t)(g0 + j) * w_gs + (size_t) o0 * kGmGroup, kBO * kRowB, bar);
        }
    };
    if (tid == 0) for (int s0 = 0; s0 < kStages && s0 < total_steps; s0++) issue(s0);

    int step = 0;
    for (int ti = 0; ti < my_tiles; ti++) {
        const int tile = blockIdx.x + ti * gridDim.x;
        const int m0 = (tile / tiles_o) * kBM, o0 = (tile % tiles_o) * kBO;
        float acc[Cfg::kNAcc];
#pragma unroll
        for (int i = 0; i < Cfg::kNAcc; i++) acc[i] = 0.0f;
        for (int sg = 0; sg < nstages; sg++, step++) {
            const int slot = step % kStages;
            mbar_wait(full + slot * 8, (uint32_t)(step / kStages) & 1);
            const unsigned char * st = smem + (size_t) slot * kStageBytes;
            const unsigned char * const ga0 = st + lane * sizeof(typename QuadOp<T>::V) + wm * 8 * kRowB;
            const unsigned char * const gw0 = st + kBM * kRowB + lane * sizeof(typename QuadOp<T>::V) + wo * OT * kRowB;
            if constexpr (Cfg::PIPE) {
                if (nsteps - sg * GPS * 4 >= GPS * 4) {       // every group of the stage full (uniform across the block)
                    uint32_t a0[8], w0[OT], a1[8], w1[OT];
                    load_half<OT>(ga0, gw0, 0, a0, w0);
#pragma unroll
                    for (int j = 0; j < GPS; j++) {
                        const int off = j * (kBM + kBO) * kRowB;
                        load_half<OT>(ga0 + off, gw0 + off, 1, a1, w1);
                        fma_half<OT>(a0, w0, acc);
                        if (j + 1 < GPS) load_half<OT>(ga0 + off + (kBM + kBO) * kRowB, gw0 + off + (kBM + kBO) * kRowB, 0, a0, w0);
                        fma_half<OT>(a1, w1, acc);
                    }
                    goto released;
                }
            }
#pragma unroll
            for (int j = 0; j < GPS; j++) {
                const int g = sg * GPS + j;
                if (g < ngroups) {                            // uniform across the block
                    const unsigned char * ga = ga0 + j * (kBM + kBO) * kRowB, * gw = gw0 + j * (kBM + kBO) * kRowB;
                    const int steps = nsteps - g * 4;         // chain steps from this group on
                    if (steps >= 4) fma_group<T, OT, true>(ga, gw, acc, 4);
                    else            fma_group<T, OT, false>(ga, gw, acc, steps);
                }
            }
        released:
            __syncwarp();
            if (lane == 0) {                                  // release the slot; the last of the warps refills it
                if ((atom_add_acq_rel_cta(&cnt[slot], 1) + 1) % Cfg::kWarps == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    if (step + kStages < total_steps) issue(step + kStages);
                }
            }
        }
        if constexpr (Cfg::kSmemReduce) {
            float * const red = reinterpret_cast<float *>(smem + Cfg::kRedOff) + warp * 32 * kRedLd;
#pragma unroll
            for (int sl = 0; sl < Cfg::kNAcc / 32; sl++) {
                __syncwarp();                                 // the previous slice's (or tile's) reads are done
#pragma unroll
                for (int j = 0; j < 32; j++) red[j * kRedLd + lane] = acc[sl * 32 + j];
                __syncwarp();
                float a[32];
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const float4 t = *reinterpret_cast<const float4 *>(red + lane * kRedLd + q * 4);
                    a[4 * q] = t.x; a[4 * q + 1] = t.y; a[4 * q + 2] = t.z; a[4 * q + 3] = t.w;
                }
                const int i = sl * 32 + lane;                 // = mi * OT + oi
                const int m = m0 + wm * 8 + i / OT, o = o0 + wo * OT + i % OT;
                const float r = lane_tree_reduce_local(a);
                if (m < M && o < O) matmul_epilogue(ep, m, o, r);
            }
        } else {
            static_assert(Cfg::kNAcc == 64, "the butterfly combines 64 outputs");
            const int base = butterfly_reduce64(acc, lane);    // outputs base, base+1 of the warp tile (index = mi*8 + oi)
            const int m = m0 + wm * 8 + (base >> 3), o = o0 + wo * 8 + (base & 7);
            if (m < M) {
                if (o < O) matmul_epilogue(ep, m, o, acc[0]);
                if (o + 1 < O) matmul_epilogue(ep, m, o + 1, acc[1]);
            }
        }
    }
}

template <typename T, typename Cfg>
static void launch_tiled(const DMat & W, const void * act, int act_gs, int rows, const MatmulEpilogue & ep, int n_sm, cudaStream_t s) {
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured))
        BARK_CUDA_CHECK(cudaFuncSetAttribute(lane_gemm_tiled_kernel<T, Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) Cfg::kSmem));
    const int n_tiles = ((W.n_out + Cfg::kBO - 1) / Cfg::kBO) * ((rows + Cfg::kBM - 1) / Cfg::kBM);
    const int grid = min(n_tiles, Cfg::MINB * n_sm);            // persistent: as many CTAs as fit at once (registers, shared memory)
    BARK_LAUNCH((lane_gemm_tiled_kernel<T, Cfg>), grid, Cfg::kThreads, Cfg::kSmem, s, (const T *) W.p_gm, W.K, W.o_pad * kGmGroup, W.n_out,
                (const T *) act, act_gs, rows, ep);
}

int lane_gemm_tiled(const DMat & W, const void * act, int act_gs, int rows, const MatmulEpilogue & ep, cudaStream_t s, int variant) {
    if (!W.p_gm) { fprintf(stderr, "bark_b200: matrix has no group-major copy for the tiled mat-mul\n"); throw std::runtime_error("unsupported configuration (see the message above)"); }
    if (W.o_pad % kGemmOPad) { fprintf(stderr, "bark_b200: group-major rows padded to %d, need a multiple of %d\n", W.o_pad, kGemmOPad); throw std::runtime_error("unsupported configuration (see the message above)"); }
    int dev = 0, n_sm = 0;
    BARK_CUDA_CHECK(cudaGetDevice(&dev));
    BARK_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    // f16: the 32 x 32 tile (a third fewer bytes per FMA) was measured ahead on 15 of the bench clip's 17 GEMM shapes, the 91-row
    // coarse windows included although their 72 tiles leave SMs idle, and at most 2 % behind on the other two (DESIGN §4.5).
    // f32 has only the 32 x 16 tile it has always had (DESIGN §4.5: at the fine-pass shapes it is 13-19 % faster than before).
    if (variant == 0) variant = W.type == W_F16 ? 2 : 1;
    if (W.type == W_F16) {
        if (variant == 1) launch_tiled<__half, Tile32x16>(W, act, act_gs, rows, ep, n_sm, s);
        else if (variant == 2) launch_tiled<__half, Tile32x32>(W, act, act_gs, rows, ep, n_sm, s);
        else return 0;
    } else if (W.type == W_F32) {
        if (variant == 1) launch_tiled<float, Tile32x16>(W, act, act_gs, rows, ep, n_sm, s);
        else return 0;
    } else return 0;
    return variant;
}

// ------------------------------------------------------------------------------------------------
// attention, multi-row (bark.cpp:1302-1339 / 1495-1530): scores, scale, causal mask, soft_max and P.V of one (head, 32-query tile)
// in one CTA; the tile's score rows never leave shared memory
// ------------------------------------------------------------------------------------------------
// Scores: lane = query, so a thread owns a (query, key) output, runs its 32 lane chains in registers against its query row (also in
// registers) and reduces them with lane_tree_reduce_local: the additions of GGML_F32x8_REDUCE without a shuffle.  The key row is a
// shared-memory broadcast; K streams through a 2-stage ring of 64-key tiles (cp.async), warp w taking keys w*8 .. w*8+7 of each.
// P.V: attn chains as the reference's vec_dot_f32 over the probability row: warp = 8 queries x 8 head columns, lane v walks
// k = v, v+32, ... below n_kv & ~31, butterfly_reduce64, then pv_leftovers.  V streams through the same ring in chunks of up to 512
// keys x 16 head columns (4 x 2 warp tiles); a CTA reads each element of its head's K and V from L2 once.
constexpr int kAttnQ = 32, kAttnKT = 64, kAttnVK = 512, kAttnVW = 16;
constexpr int kAttnVLd = kAttnVW + 4;      // V chunk row stride (floats): 8 consecutive rows' 16-byte reads hit 8 different bank quads

// score row stride (floats): odd, so the 32 lanes' stores of one key land in 32 different banks
__host__ __device__ inline int attn_ld(int n_kv) { return ((n_kv + 31) & ~31) + 1; }
__host__ __device__ inline int attn_ring_off(int n_kv) { return (kAttnQ * attn_ld(n_kv) + 3) & ~3; }

namespace {
__device__ __forceinline__ void cp_async_16(void * dst, const float * src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_prev() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }    // all but the latest group
}  // namespace

template <int DSTEPS>
__global__ void __launch_bounds__(256, 1) attn_fused_kernel(const float * __restrict__ Q, const float * __restrict__ Kc, const float * __restrict__ Vc,
                                                            int N, int n_kv, int n_past, int E, float scale, int causal,
                                                            void * __restrict__ act, int wt, int Kp) {
    constexpr int D = DSTEPS * 32;
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h = blockIdx.y, q0 = blockIdx.x * kAttnQ;
    const int ld = attn_ld(n_kv);
    float * const P = sm;                                    // [kAttnQ][ld] scores -> probabilities
    float * const ring = sm + attn_ring_off(n_kv);           // 2 K tiles [kAttnKT][D], later 2 V chunks [vk][kAttnVLd]
    const float * const kh = Kc + h * D, * const vh = Vc + h * D;
    const float ninf = __int_as_float(0xff800000);

    // ---- scores ----
    float qr[D];
    {
        const float4 * qrow = reinterpret_cast<const float4 *>(Q + (size_t) min(q0 + lane, N - 1) * E + h * D);
#pragma unroll
        for (int i = 0; i < D / 4; i++) { const float4 t = __ldg(qrow + i); qr[4 * i] = t.x; qr[4 * i + 1] = t.y; qr[4 * i + 2] = t.z; qr[4 * i + 3] = t.w; }
    }
    const int n_kt = (n_kv + kAttnKT - 1) / kAttnKT;
    auto issue_k = [&](int t) {
        if (t < n_kt) {
            float * const dst = ring + (t & 1) * kAttnKT * D;
            for (int i = tid; i < kAttnKT * D / 4; i += 256) {
                const int r = i / (D / 4), c = i % (D / 4), k = t * kAttnKT + r;
                if (k < n_kv) cp_async_16(dst + r * D + c * 4, kh + (size_t) k * E + c * 4);
            }
        }
        cp_async_commit();                                   // (an empty group past the last tile keeps the wait count uniform)
    };
    issue_k(0); issue_k(1);
    const int k_vis = n_past + min(q0 + kAttnQ, N) - 1;      // causal: the last key any query of the tile sees
    for (int t = 0; t < n_kt; t++) {
        cp_async_wait_prev();
        __syncthreads();
        const float * const kt = ring + (t & 1) * kAttnKT * D;
        for (int j = 0; j < 8; j++) {
            const int kl = warp * 8 + j, k = t * kAttnKT + kl;
            if (k >= n_kv) break;
            float r = ninf;
            if (!causal || k <= k_vis) {
                float a[32];
#pragma unroll
                for (int v = 0; v < 32; v++) a[v] = 0.0f;
#pragma unroll
                for (int c = 0; c < DSTEPS; c++)
#pragma unroll
                    for (int v4 = 0; v4 < 8; v4++) {
                        const float4 kk = *reinterpret_cast<const float4 *>(kt + kl * D + c * 32 + v4 * 4);
                        a[v4 * 4]     = __fmaf_rn(kk.x, qr[c * 32 + v4 * 4],     a[v4 * 4]);
                        a[v4 * 4 + 1] = __fmaf_rn(kk.y, qr[c * 32 + v4 * 4 + 1], a[v4 * 4 + 1]);
                        a[v4 * 4 + 2] = __fmaf_rn(kk.z, qr[c * 32 + v4 * 4 + 2], a[v4 * 4 + 2]);
                        a[v4 * 4 + 3] = __fmaf_rn(kk.w, qr[c * 32 + v4 * 4 + 3], a[v4 * 4 + 3]);
                    }
                r = __fmul_rn(lane_tree_reduce_local(a), scale);                  // ggml_scale_inplace
                if (causal && k > n_past + q0 + lane) r = ninf;                   // ggml_diag_mask_inf
            }
            P[lane * ld + k] = r;
        }
        __syncthreads();
        issue_k(t + 2);
    }

    // ---- V chunks: D / 16 rounds of 16 head columns, each over keys [0, np) ----
    const int np = n_kv & ~31;
    const int vk = min(kAttnVK, np), n_ch = vk ? (np + vk - 1) / vk : 0;
    auto issue_v = [&](int i) {
        if (i < n_ch * (D / kAttnVW)) {
            const int rd = i / n_ch, k0 = (i % n_ch) * vk, rows = min(vk, np - k0);
            float * const dst = ring + (i & 1) * vk * kAttnVLd;
            for (int e = tid; e < rows * 4; e += 256)
                cp_async_16(dst + (e >> 2) * kAttnVLd + (e & 3) * 4, vh + (size_t)(k0 + (e >> 2)) * E + rd * kAttnVW + (e & 3) * 4);
        }
        cp_async_commit();
    };
    issue_v(0); issue_v(1);

    // ---- soft_max of the tile's rows, in place, while the first V chunks arrive ----
    for (int r = warp; r < min(kAttnQ, N - q0); r += 8) softmax_row(P + r * ld, n_kv);
    __syncthreads();                                         // (P.V below may run no chunk at all when n_kv < 32)

    // ---- P.V ----
    const int qs = warp & 3, cs = warp >> 2;
    const float * const pw = P + qs * 8 * ld;               // this warp's 8 probability rows
    int i = 0;
    for (int rd = 0; rd < D / kAttnVW; rd++) {
        float acc[64];
#pragma unroll
        for (int a = 0; a < 64; a++) acc[a] = 0.0f;
        for (int c = 0; c < n_ch; c++, i++) {
            const int k0 = c * vk, rows = min(vk, np - k0);
            cp_async_wait_prev();
            __syncthreads();
            const float * const vt = ring + (i & 1) * vk * kAttnVLd + cs * 8;
            for (int kl = lane; kl < rows; kl += 32) {
                const float4 v0 = *reinterpret_cast<const float4 *>(vt + kl * kAttnVLd);
                const float4 v1 = *reinterpret_cast<const float4 *>(vt + kl * kAttnVLd + 4);
                const float vf[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                for (int qi = 0; qi < 8; qi++) {
                    const float p = pw[qi * ld + k0 + kl];
#pragma unroll
                    for (int di = 0; di < 8; di++) acc[qi * 8 + di] = __fmaf_rn(vf[di], p, acc[qi * 8 + di]);
                }
            }
            __syncthreads();
            issue_v(i + 2);
        }
        const int base = butterfly_reduce64(acc, lane);
        const int q = q0 + qs * 8 + (base >> 3), d = rd * kAttnVW + cs * 8 + (base & 7);
        if (q < N) {
            const float * const p = P + (q - q0) * ld;
#pragma unroll
            for (int j = 0; j < 2; j++) store_act(act, wt, Kp, q, h * D + d + j, pv_leftovers(acc[j], vh + d + j, p, np, n_kv, E));
        }
    }
}

// Few query rows (the causal models' prefills, the per-op decode path): the fused kernel's grid of (N / 32) x H CTAs would leave
// most SMs idle, so three kernels spread the same arithmetic over (n_kv / 64) x (N / 8) x H CTAs and pass the scores through
// memory instead: 8 x 8 tiles per warp, the lane mapping of the fused kernel's P.V for both contractions.
// scores[h][q][k] = vec_dot_f32(D, K[k][h], Q[q][h]) * scale, -inf where k > n_past + q (causal)
template <int DSTEPS>
__global__ void __launch_bounds__(256) attn_scores_tiled_kernel(const float * __restrict__ Q, const float * __restrict__ Kc, int N, int n_kv, int n_past, int E,
                                                                float scale, int causal, float * __restrict__ S) {
    constexpr int D = DSTEPS * 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h = blockIdx.z, q0 = blockIdx.y * 8, k0 = (blockIdx.x * 8 + warp) * 8;
    if (k0 >= n_kv) return;
    float qf[8][DSTEPS], kf[8][DSTEPS];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int q = min(q0 + i, N - 1), k = min(k0 + i, n_kv - 1);
#pragma unroll
        for (int c = 0; c < DSTEPS; c++) {
            qf[i][c] = __ldg(Q + (size_t) q * E + h * D + c * 32 + lane);
            kf[i][c] = __ldg(Kc + (size_t) k * E + h * D + c * 32 + lane);
        }
    }
    float acc[64];
#pragma unroll
    for (int qi = 0; qi < 8; qi++)
#pragma unroll
        for (int ki = 0; ki < 8; ki++) {
            float a = 0.0f;
#pragma unroll
            for (int c = 0; c < DSTEPS; c++) a = __fmaf_rn(kf[ki][c], qf[qi][c], a);
            acc[qi * 8 + ki] = a;
        }
    const int base = butterfly_reduce64(acc, lane);
    const int q = q0 + (base >> 3), k = k0 + (base & 7);
    if (q < N) {
        float * row = S + ((size_t) blockIdx.z * N + q) * n_kv;
#pragma unroll
        for (int j = 0; j < 2; j++) if (k + j < n_kv) {
            float r = __fmul_rn(acc[j], scale);                                       // ggml_scale_inplace
            if (causal && k + j > n_past + q) r = __int_as_float(0xff800000);         // ggml_diag_mask_inf
            row[k + j] = r;
        }
    }
}

// KQV[q][h*D+d] = vec_dot_f32(n_kv, V^T[d], P[q]) -> activation operand for c_proj.  Warp = 8 queries x 8 head columns;
// lane v walks k = v, v+32, ...  D / 8 warps: up to 512 threads for 128-wide heads.
__global__ void __launch_bounds__(512) attn_pv_tiled_kernel(const float * __restrict__ S, const float * __restrict__ Vc, int N, int n_kv, int E, int D,
                                                            void * __restrict__ act, int wt, int Kp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h = blockIdx.y, q0 = blockIdx.x * 8, d0 = warp * 8;
    if (d0 >= D) return;
    const float * prow[8];
#pragma unroll
    for (int qi = 0; qi < 8; qi++) prow[qi] = S + ((size_t) h * N + min(q0 + qi, N - 1)) * n_kv;
    const float * vbase = Vc + h * D + d0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.0f;
    const int np = n_kv & ~31;
    for (int k = lane; k < np; k += 32) {
        const float4 v0 = __ldg(reinterpret_cast<const float4 *>(vbase + (size_t) k * E));
        const float4 v1 = __ldg(reinterpret_cast<const float4 *>(vbase + (size_t) k * E) + 1);
        const float vf[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int qi = 0; qi < 8; qi++) {
            const float p = __ldg(prow[qi] + k);
#pragma unroll
            for (int di = 0; di < 8; di++) acc[qi * 8 + di] = __fmaf_rn(vf[di], p, acc[qi * 8 + di]);
        }
    }
    const int base = butterfly_reduce64(acc, lane);
    const int q = q0 + (base >> 3), d = d0 + (base & 7);
    if (q >= N) return;
    const float * p = S + ((size_t) h * N + q) * n_kv;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        store_act(act, wt, Kp, q, h * D + d + j, pv_leftovers(acc[j], Vc + h * D + d + j, p, np, n_kv, E));
    }
}

// soft_max of the score matrix, one warp per row
__global__ void attn_softmax_kernel(float * __restrict__ S, int rows, int n_kv) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    softmax_row(S + (size_t) row * n_kv, n_kv);
}

// the same, counting the rows that took the sequential replay (bark_b200_parity_rows)
__global__ void softmax_rows_kernel(float * __restrict__ S, int rows, int n, unsigned * __restrict__ replays) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    softmax_row(S + (size_t) row * n, n, replays);
}

void softmax_rows(float * S, int rows, int n, unsigned * replays, cudaStream_t s) {
    BARK_LAUNCH(softmax_rows_kernel, (rows + 7) / 8, 256, 0, s, S, rows, n, replays);
}

int attn_tiled_max_rows(int H, int n_sm) { return kAttnQ * ((n_sm + H - 1) / H - 1); }

void attention(const float * Q, const float * Kc, const float * Vc, int N, int n_kv, int n_past, int E, int H, bool causal,
               float * scores, void * act, WType wt, int Kp, cudaStream_t s, AttnPath path) {
    const int D = E / H;
    if (E % H || D < 32 || D % 32 || D > 128 || N < 1 || n_kv < 1 || n_kv > 1024) {
        fprintf(stderr, "bark_b200: attention needs a head size of 32, 64, 96 or 128 and 1..1024 keys (got %d heads of %d, %d keys)\n", H, D, n_kv);
        throw std::runtime_error("unsupported configuration (see the message above)");
    }
    const float scale = 1.0f / sqrtf((float) E / (float) H);                 // bark.cpp:1318
    int dev = 0, n_sm = 0;
    BARK_CUDA_CHECK(cudaGetDevice(&dev));
    BARK_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    if (path == ATTN_TILED || (path == ATTN_AUTO && N <= attn_tiled_max_rows(H, n_sm))) {
        if (N > attn_tiled_max_rows(H, n_sm)) {
            fprintf(stderr, "bark_b200: %d rows exceed the score buffer of the three-kernel attention (%d)\n", N, attn_tiled_max_rows(H, n_sm));
            throw std::runtime_error("unsupported configuration (see the message above)");
        }
        const int rows = H * N, c = causal ? 1 : 0;
        const dim3 grid((n_kv + 63) / 64, (N + 7) / 8, H);
        g_next_bytes = 4.0 * ((double) n_kv * E + (double) N * E + (double) H * N * n_kv); g_next_flops = 2.0 * (double) N * n_kv * E;
        if (D == 64)      BARK_LAUNCH(attn_scores_tiled_kernel<2>, grid, 256, 0, s, Q, Kc, N, n_kv, n_past, E, scale, c, scores);
        else if (D == 32) BARK_LAUNCH(attn_scores_tiled_kernel<1>, grid, 256, 0, s, Q, Kc, N, n_kv, n_past, E, scale, c, scores);
        else if (D == 96) BARK_LAUNCH(attn_scores_tiled_kernel<3>, grid, 256, 0, s, Q, Kc, N, n_kv, n_past, E, scale, c, scores);
        else              BARK_LAUNCH(attn_scores_tiled_kernel<4>, grid, 256, 0, s, Q, Kc, N, n_kv, n_past, E, scale, c, scores);
        g_next_bytes = 8.0 * (double) rows * n_kv;
        BARK_LAUNCH(attn_softmax_kernel, (rows + 7) / 8, 256, 0, s, scores, rows, n_kv);
        g_next_bytes = 4.0 * ((double) n_kv * E + (double) H * N * n_kv + (double) N * E); g_next_flops = 2.0 * (double) N * n_kv * E;
        BARK_LAUNCH(attn_pv_tiled_kernel, dim3((N + 7) / 8, H), 32 * ((D + 7) / 8), 0, s, scores, Vc, N, n_kv, E, D, act, (int) wt, Kp);
        return;
    }
    const int np = n_kv & ~31;
    const size_t ring = std::max((size_t) 2 * kAttnKT * D, (size_t) 2 * std::min(kAttnVK, np) * kAttnVLd);
    const size_t smem = ((size_t) attn_ring_off(n_kv) + ring) * 4;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) {
        const size_t most = ((size_t) attn_ring_off(1024) + std::max(2 * kAttnKT * 128, 2 * kAttnVK * kAttnVLd)) * 4;
        BARK_CUDA_CHECK(cudaFuncSetAttribute(attn_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) most));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(attn_fused_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) most));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(attn_fused_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) most));
        BARK_CUDA_CHECK(cudaFuncSetAttribute(attn_fused_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) most));
    }
    const dim3 grid((N + kAttnQ - 1) / kAttnQ, H);
    g_next_bytes = 4.0 * (2.0 * N * E + 2.0 * n_kv * E); g_next_flops = 4.0 * N * (double) n_kv * E;
    const int c = causal ? 1 : 0;
    if (D == 64)      BARK_LAUNCH(attn_fused_kernel<2>, grid, 256, smem, s, Q, Kc, Vc, N, n_kv, n_past, E, scale, c, act, (int) wt, Kp);
    else if (D == 32) BARK_LAUNCH(attn_fused_kernel<1>, grid, 256, smem, s, Q, Kc, Vc, N, n_kv, n_past, E, scale, c, act, (int) wt, Kp);
    else if (D == 96) BARK_LAUNCH(attn_fused_kernel<3>, grid, 256, smem, s, Q, Kc, Vc, N, n_kv, n_past, E, scale, c, act, (int) wt, Kp);
    else              BARK_LAUNCH(attn_fused_kernel<4>, grid, 256, smem, s, Q, Kc, Vc, N, n_kv, n_past, E, scale, c, act, (int) wt, Kp);
}
}  // namespace bark
