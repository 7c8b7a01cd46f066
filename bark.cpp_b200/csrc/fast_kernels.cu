// FAST MODE (BARK_B200_MODE=fast, opt-in): the dense contractions of the hot path on the Hopper tensor cores (wgmma).
//
// The fine model's 1024-row passes (bark.cpp:1416-1584; mul_mat sites bark.cpp:1278,1344,1371,1380,1403 and the non-causal
// attention bark.cpp:1495-1530) are genuine GEMMs.  The parity path (gemm_kernels.cu) must replay the reference's 32 IEEE FMA chains
// per output and therefore runs on the fp32 pipe; wgmma accumulates in a different order, so this path cannot be bit-identical
// and is validated by kernel tests with exact answers and by teacher forcing instead (tests/test_fast_mode.py).
//
//   wgmma_gemm_kernel  C[M][N] = A[M][K] * W[N][K]^T, f16 operands, f32 accumulate in registers.  Block tile 128 x BN.
//                      warp 8: TMA producer (cp.async.bulk.tensor 2-D tiles, 128-byte swizzle, mbarrier complete_tx ring)
//                      warpgroups 0-1: 64 rows each, wgmma.mma_async m64nBNk16 from shared-memory descriptors, one stage kept in
//                              flight; fused epilogue from the accumulator registers: f16 store (+ V^T for the attention kernel),
//                              residual add, GELU -> f16, plain f32 store
//   flash_attn_kernel  non-causal attention of one (head, 128-query tile) over all keys in blocks of 128: each warpgroup owns 64
//                      queries, S = Q K^T into registers (wgmma), online soft_max in registers, P (f16) stays in registers as the
//                      A operand of O += P V (wgmma with A from registers); no score matrix ever reaches shared memory or HBM.
//   ln_rows_f16_kernel LayerNorm -> f16 row-major operand (float statistics; the parity path's double sums are not needed here)
#include "gpt_kernels.h"
#include "epilogue.cuh"

#include <cuda.h>

namespace bark {

namespace {

// ---- PTX helpers ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// bounded wait: a protocol bug traps (the launch fails with an error) instead of hanging the GPU.  No printf here: a function call
// inside the MMA warpgroups' loop makes ptxas serialize every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    const long long t0 = clock64();
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) break;
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap * map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap * map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }
// programmatic dependent launch: wait for the preceding kernel's results / let the following kernel start its prologue
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- wgmma (sm_90a) ---------------------------------------------------------------------------------------------------
// Accumulator fragment of an m64nN tile, thread t of the warpgroup (w = t / 32, g = (t % 32) / 4, c = t % 4):
//   d[4j + 0], d[4j + 1] = row 16w + g,     columns 8j + 2c, 8j + 2c + 1
//   d[4j + 2], d[4j + 3] = row 16w + g + 8, same columns
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs that read / write them
template <int R> __device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i]) :: "memory");
}
// D[64][64] (+)= A[64][16] * B[64][16]^T, both operands K-major in shared memory (descriptors); scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d));
}
// D[64][128] (+)= A[64][16] * B[128][16]^T, both operands K-major in shared memory (descriptors); scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(scale_d));
}
// D[64][256] (+)= A[64][16] * B[256][16]^T, both operands K-major in shared memory (descriptors); scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t da, uint64_t db, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(da), "l"(db), "r"(scale_d));
}
// D[64][64] += A[64][16] * B[64][16]^T with A in registers (four f16x2 per thread, the accumulator fragment layout), B K-major in shared memory
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 0;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// Shared-memory matrix descriptor (sm_90 wgmma) of a K-major operand tile written by TMA with the 128-byte swizzle: rows of 64 f16
// (128 B), 8-row groups 1024 B apart (stride byte offset), one swizzle atom along K (leading byte offset unused), layout type 1 =
// SWIZZLE_128B.  Advancing by one MMA (K = 16 elements = 32 B) adds 2 to the encoded start address.  Tiles are 1024-byte aligned.
__device__ __forceinline__ uint64_t kmajor_sw128_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}

template <int BN> struct WgmmaN;
template <> struct WgmmaN<64>  { __device__ __forceinline__ static void mma(float (&d)[32], uint64_t a, uint64_t b, int sc)  { wgmma_ss_n64(d, a, b, sc); } };
template <> struct WgmmaN<128> { __device__ __forceinline__ static void mma(float (&d)[64], uint64_t a, uint64_t b, int sc)  { wgmma_ss_n128(d, a, b, sc); } };
template <> struct WgmmaN<256> { __device__ __forceinline__ static void mma(float (&d)[128], uint64_t a, uint64_t b, int sc) { wgmma_ss_n256(d, a, b, sc); } };

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&h);
}

constexpr int kBM = 128, kBK = 64;                 // CTA tile rows; K elements per pipeline stage (= one 128-byte swizzle atom)
constexpr int kGemmThreads = 288;                  // warpgroups 0-1: MMA + epilogue; warp 8: TMA producer

}  // namespace

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
// GELU as the reference's table defines it (ggml.c:2546-2571: f16(x) -> 0.5 x (1 + tanh(sqrt(2/pi) x (1 + 0.044715 x^2))) -> f16), evaluated
// in closed form instead of a 64 K-entry table: dependent table look-ups per output would dominate the fc GEMM's epilogue.
// It uses 0.5 x (1 + tanh y) = x / (1 + 2^(-2 y log2(e))), which does not cancel for negative x: 1 + tanh y does, and there the
// ~2^-11 relative error of tanh.approx becomes thousands of f16 ulps of the small result.  ex2.approx and the fast reciprocal are
// accurate to ~2^-22 relative, so for every f16 input the result is within one f16 ulp of the table, or within 2^-22 where the
// table's own float tanh is quantised near -1 (tests/test_fast_mode.py).
// For x <= -10 the denominator exceeds 2^126 or is infinite and the result is -0, as the table's 0.
__device__ __forceinline__ float gelu_fast(float v) {
    const float x = __half2float(__float2half_rn(v));
    const float y = 0.79788456080286535588f * x * (1.0f + 0.044715f * x * x);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-2.88539008177792681f * y));       // 2^(-2 y log2(e)) = e^(-2y)
    return __fdividef(x, 1.0f + e);
}

// two horizontally adjacent outputs (m, n), (m, n + 1) of the fused epilogue
__device__ __forceinline__ void fast_epilogue_pair(const FastEpi & ep, int m, int n, int N, float v0, float v1) {
    const bool two = n + 1 < N, vec = two && (ep.ldo & 1) == 0;
    if (ep.mode == FEPI_F32 || ep.mode == FEPI_RESID) {
        float * dst = ep.out32 + (size_t) m * ep.ldo + n;
        if (vec) {
            float2 o = make_float2(v0, v1);
            if (ep.mode == FEPI_RESID) { const float2 x = *reinterpret_cast<const float2 *>(dst); o.x += x.x; o.y += x.y; }
            *reinterpret_cast<float2 *>(dst) = o;
        } else {
            dst[0] = ep.mode == FEPI_RESID ? v0 + dst[0] : v0;
            if (two) dst[1] = ep.mode == FEPI_RESID ? v1 + dst[1] : v1;
        }
    } else if (ep.mode == FEPI_QKV16 && n >= ep.v_col0) {      // V^T for the attention kernel (v_col0 is even: a pair never straddles it)
        ep.vt[(size_t)(n - ep.v_col0) * ep.vt_ld + m] = __float2half_rn(v0);
        if (two) ep.vt[(size_t)(n + 1 - ep.v_col0) * ep.vt_ld + m] = __float2half_rn(v1);
    } else {
        if (ep.mode == FEPI_GELU16) { v0 = gelu_fast(v0); v1 = gelu_fast(v1); }
        __half * dst = ep.out16 + (size_t) m * ep.ldo + n;
        if (vec) *reinterpret_cast<uint32_t *>(dst) = pack_half2(v0, v1);
        else {
            dst[0] = __float2half_rn(v0);
            if (two) dst[1] = __float2half_rn(v1);
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1) wgmma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                      int M, int N, int K, FastEpi ep) {
    constexpr int kStages = BN >= 256 ? 4 : BN >= 128 ? 6 : 8;
    constexpr int kABytes = kBM * kBK * 2, kBBytes = BN * kBK * 2, kStageBytes = kABytes + kBBytes;
    extern __shared__ unsigned char smem_raw[];
    unsigned char * smem = (unsigned char *)(((uintptr_t) smem_raw + 1023) & ~(uintptr_t) 1023);      // swizzle-128B tiles need 1024-byte alignment
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + kStages * kStageBytes);                      // full[kStages], empty[kStages]
    const uint32_t full0 = smem_u32(bars), empty0 = full0 + kStages * 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * BN;
    const int nk = K / kBK;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < kStages; s++) { mbar_init(full0 + s * 8, 1); mbar_init(empty0 + s * 8, 8); }   // empty: lane 0 of each MMA warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();                                  // the next kernel of the chain may begin its prologue on SMs as they free up
    pdl_wait();                                               // everything above overlapped the previous kernel's tail; its outputs are needed from here on

    if (warp == 8) {
        if (lane == 0) {                                      // ===== TMA producer =====
            for (int kb = 0; kb < nk; kb++) {
                const int s = kb % kStages;
                mbar_wait(empty0 + s * 8, ((kb / kStages) & 1) ^ 1);
                const uint32_t dst = smem_u32(smem + (size_t) s * kStageBytes);
                mbar_expect_tx(full0 + s * 8, kStageBytes);
                tma_load_2d(dst, &tmA, kb * kBK, m0, full0 + s * 8);
                tma_load_2d(dst + kABytes, &tmB, kb * kBK, n0, full0 + s * 8);
            }
        }
        return;
    }
    // ===== warpgroup wg: rows m0 + 64 wg .. + 63 of the tile =====
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.0f;
    for (int kb = 0; kb < nk; kb++) {
        const int s = kb % kStages;
        mbar_wait(full0 + s * 8, (kb / kStages) & 1);
        const uint32_t a = smem_u32(smem + (size_t) s * kStageBytes);
        const uint64_t da = kmajor_sw128_desc(a + wg * 64 * 128), db = kmajor_sw128_desc(a + kABytes);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; k++) WgmmaN<BN>::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                      // stage kb stays in flight; stage kb - 1 is complete
        fence_regs(acc);
        if (kb > 0 && lane == 0) mbar_arrive(empty0 + ((kb - 1) % kStages) * 8);
    }
    wgmma_wait<0>();
    fence_regs(acc);
    const int w = warp & 3, g = lane >> 2, c = lane & 3;
    const int r0 = m0 + wg * 64 + w * 16 + g;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int n = n0 + 8 * j + 2 * c;
        if (n >= N) continue;
        if (r0 < M)     fast_epilogue_pair(ep, r0, n, N, acc[4 * j], acc[4 * j + 1]);
        if (r0 + 8 < M) fast_epilogue_pair(ep, r0 + 8, n, N, acc[4 * j + 2], acc[4 * j + 3]);
    }
}

// ------------------------------------------------------------------------------------------------
// attention (non-causal, head size 64, keys in blocks of 128)
// ------------------------------------------------------------------------------------------------
constexpr int kKeyBlk = 128, kHeadD = 64, kKvStages = 4;
struct FlashSmem {
    static constexpr int q = 0;                                    // [128 queries][64] f16, swizzled K-major                16 KB
    static constexpr int k = q + 128 * 128;                        // kKvStages x [128 keys][64] f16                         64 KB
    static constexpr int v = k + kKvStages * kKeyBlk * 128;        // kKvStages x 2 atoms x [64 d][64 keys] f16              64 KB
    static constexpr int bars = v + kKvStages * kKeyBlk * 128;     // q_full, kv_full[kKvStages], kv_empty[kKvStages]
    static constexpr int total = bars + (1 + 2 * kKvStages) * 8;
};

// tmQK: the [N][ldq] f16 buffer holding Q (columns h*64) and K (columns k_col0 + h*64), box 64 x 128;  tmVT: V^T [E][N] f16, box 64 keys x 64 rows
__global__ void __launch_bounds__(kGemmThreads, 1) flash_attn_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmVT,
                                                                      int n_keys, int k_col0, float scale_log2e, __half * __restrict__ out, int ldo) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char * smem = (unsigned char *)(((uintptr_t) smem_raw + 1023) & ~(uintptr_t) 1023);
    const uint32_t b0 = smem_u32(smem + FlashSmem::bars);
    const uint32_t q_full = b0, kv_full0 = b0 + 8, kv_empty0 = b0 + 8 + kKvStages * 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h = blockIdx.y, q0 = blockIdx.x * 128;
    const int nblk = n_keys / kKeyBlk;
    constexpr uint32_t kStage = kKeyBlk * 128;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmQK); prefetch_tmap(&tmVT);
        mbar_init(q_full, 1);
        for (int s = 0; s < kKvStages; s++) { mbar_init(kv_full0 + s * 8, 1); mbar_init(kv_empty0 + s * 8, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t sQ = smem_u32(smem + FlashSmem::q), sK = smem_u32(smem + FlashSmem::k), sV = smem_u32(smem + FlashSmem::v);

    if (warp == 8) {
        if (lane == 0) {                                      // ===== TMA producer =====
            mbar_expect_tx(q_full, 128 * 128);
            tma_load_2d(sQ, &tmQK, h * kHeadD, q0, q_full);
            for (int j = 0; j < nblk; j++) {
                const int s = j % kKvStages;
                mbar_wait(kv_empty0 + s * 8, ((j / kKvStages) & 1) ^ 1);
                mbar_expect_tx(kv_full0 + s * 8, 2 * kStage);
                tma_load_2d(sK + s * kStage, &tmQK, k_col0 + h * kHeadD, j * kKeyBlk, kv_full0 + s * 8);
                for (int a = 0; a < 2; a++) tma_load_2d(sV + s * kStage + a * 64 * 128, &tmVT, j * kKeyBlk + a * 64, h * kHeadD, kv_full0 + s * 8);
            }
        }
        return;
    }
    // ===== warpgroup wg: queries q0 + 64 wg .. + 63; this thread holds rows g and g + 8 of its warp's 16 =====
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, c = lane & 3;
    float o[kHeadD / 2], sc[kKeyBlk / 2];
#pragma unroll
    for (int i = 0; i < kHeadD / 2; i++) o[i] = 0.0f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};        // l_run: this thread's share of the row sums
    const uint64_t dq = kmajor_sw128_desc(sQ + wg * 64 * 128);
    mbar_wait(q_full, 0);
    for (int j = 0; j < nblk; j++) {
        const int s = j % kKvStages;
        mbar_wait(kv_full0 + s * 8, (j / kKvStages) & 1);
        // S = Q K^T  (64 x 128, K = 64)
        const uint64_t dk = kmajor_sw128_desc(sK + s * kStage);
        fence_regs(sc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kHeadD / 16; k++) wgmma_ss_n128(sc, dq + 2 * k, dk + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(sc);
        // online soft_max of rows g (r = 0) and g + 8 (r = 1): a row lives in the four threads of a quad
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            float mx = m_run[r];
#pragma unroll
            for (int i = 0; i < kKeyBlk / 8; i++) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * r], sc[4 * i + 2 * r + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            alpha[r] = exp2f((m_run[r] - mx) * scale_log2e);
            m_run[r] = mx;
        }
        // P (f16) as the A operand of P V: k-step kk covers keys 16 kk .. 16 kk + 15 = accumulator column groups 2 kk, 2 kk + 1
        uint32_t pa[kKeyBlk / 16][4];
        float sum[2] = {0.0f, 0.0f};
#pragma unroll
        for (int i = 0; i < kKeyBlk / 8; i++) {
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const __half2 hp = __floats2half2_rn(exp2f((sc[4 * i + 2 * r] - m_run[r]) * scale_log2e), exp2f((sc[4 * i + 2 * r + 1] - m_run[r]) * scale_log2e));
                sum[r] += __low2float(hp) + __high2float(hp);         // the sum of what the tensor core will actually multiply
                pa[i >> 1][(i & 1) * 2 + r] = *reinterpret_cast<const uint32_t *>(&hp);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; r++) l_run[r] = l_run[r] * alpha[r] + sum[r];
#pragma unroll
        for (int i = 0; i < kHeadD / 8; i++) { o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0]; o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1]; }
        // O += P V  (64 x 64, K = 128 keys): V^T atom kk / 4, 32-byte step kk % 4
        fence_regs(o);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kKeyBlk / 16; kk++) wgmma_rs_n64(o, pa[kk], kmajor_sw128_desc(sV + s * kStage + (kk >> 2) * 64 * 128) + 2 * (kk & 3));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
        if (lane == 0) mbar_arrive(kv_empty0 + s * 8);        // this warp's reads of stage s are complete
    }
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[r] = 1.0f / l;
    }
    const int row = q0 + wg * 64 + w * 16 + g;
#pragma unroll
    for (int i = 0; i < kHeadD / 8; i++) {
        const int col = h * kHeadD + 8 * i + 2 * c;
        *reinterpret_cast<uint32_t *>(out + (size_t) row * ldo + col) = pack_half2(o[4 * i] * inv[0], o[4 * i + 1] * inv[0]);
        *reinterpret_cast<uint32_t *>(out + (size_t)(row + 8) * ldo + col) = pack_half2(o[4 * i + 2] * inv[1], o[4 * i + 3] * inv[1]);
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm -> f16 row-major operand: one warp per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ln_rows_f16_kernel(const float * __restrict__ x, int rows, int E, const float * __restrict__ g, const float * __restrict__ b, __half * __restrict__ out) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    pdl_launch_dependents();
    pdl_wait();
    if (row >= rows) return;
    const float * xr = x + (size_t) row * E;
    float s = 0.0f;
    for (int i = lane; i < E; i += 32) s += xr[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float) E;
    float s2 = 0.0f;
    for (int i = lane; i < E; i += 32) { const float d = xr[i] - mean; s2 += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    const float sc = 1.0f / sqrtf(s2 / (float) E + 1e-5f);
    for (int i = lane; i < E; i += 32) {
        float y = (xr[i] - mean) * sc * g[i];
        if (b) y += b[i];
        out[(size_t) row * E + i] = __float2half_rn(y);
    }
}

// ------------------------------------------------------------------------------------------------
// weight conversion at load: one matrix of the file's type -> row-major f16 (the GEMMs' W operand)
// ------------------------------------------------------------------------------------------------
// Rows are whole blocks of 32, so the flat [n_out][K] index of an element is its index in the source as well.  The f16 is the round to
// nearest even of the weight (f32) or of dequantize_row_<t>'s value (dequant_element).  non_finite (device) is increased by the number
// of results that are inf or NaN: a source NaN / inf, or a value of magnitude >= 65520.
__global__ void __launch_bounds__(256) convert_f16_kernel(const unsigned char * __restrict__ src, WType t, size_t n, __half * __restrict__ dst,
                                                          int * __restrict__ non_finite) {
    const size_t e = (size_t) blockIdx.x * 256 + threadIdx.x;
    bool bad = false;
    if (e < n) {
        const float v = t == W_F32 ? reinterpret_cast<const float *>(src)[e] : dequant_element(src, t, e);
        const __half h = __float2half_rn(v);
        dst[e] = h;
        bad = (__half_as_ushort(h) & 0x7c00) == 0x7c00;
    }
    const unsigned nb = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && nb) atomicAdd(non_finite, __popc(nb));
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void * p = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        return (EncodeTiledFn) p;
    }();
    return fn;
}

// 2-D f16 row-major [rows][ld] view starting at column 0, `cols` columns visible; box = 64 columns (128 bytes, swizzled) x box_rows
static bool make_map(CUtensorMap * m, const void * base, int rows, int cols, int ld, int box_rows) {
    EncodeTiledFn fn = encode_tiled();
    if (!fn) { fprintf(stderr, "bark_b200 fast mode: cuTensorMapEncodeTiled is not available from this driver\n"); return false; }
    const cuuint64_t dims[2] = {(cuuint64_t) cols, (cuuint64_t) rows};
    const cuuint64_t strides[1] = {(cuuint64_t) ld * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t) box_rows}, estr[2] = {1, 1};
    const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { fprintf(stderr, "bark_b200 fast mode: cuTensorMapEncodeTiled failed (%d) for a [%d][%d] view, ld %d\n", (int) r, rows, cols, ld); return false; }
    return true;
}

template <int BN>
static bool launch_gemm(const __half * A, int lda, const __half * W, int ldw, int M, int N, int K, const FastEpi & ep, cudaStream_t s) {
    constexpr int kStages = BN >= 256 ? 4 : BN >= 128 ? 6 : 8;
    const size_t smem = (size_t) kStages * (kBM * kBK * 2 + BN * kBK * 2) + 2 * kStages * 8 + 1024;
    static std::atomic<unsigned long long> configured{0};     // kernel attributes are per device (one host thread per GPU may share this process)
    if (first_use_on_this_device(configured)) BARK_CUDA_CHECK(cudaFuncSetAttribute(wgmma_gemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    CUtensorMap ta, tb;
    if (!make_map(&ta, A, M, K, lda, kBM) || !make_map(&tb, W, N, K, ldw, BN)) return false;
    const dim3 grid((N + BN - 1) / BN, (M + kBM - 1) / kBM);
    g_next_flops = 2.0 * M * N * (double) K;
    g_next_bytes = 2.0 * ((double) M * K + (double) N * K) + (double) M * N * (ep.mode == FEPI_F32 ? 4 : ep.mode == FEPI_RESID ? 8 : 2);
    BARK_LAUNCH_PDL((wgmma_gemm_kernel<BN>), grid, dim3(kGemmThreads), smem, s, ta, tb, M, N, K, ep);
    return true;
}

// C = A W^T on the tensor cores.  A [M][lda] f16, W [N][ldw] f16 (both K-contiguous), K % 64 == 0.  bn = 0 lets the cost model below
// pick the tile width; 64 / 128 / 256 force it (tests).  Returns the tile width launched, 0 on failure.
int fast_gemm(const __half * A, int lda, const __half * W, int ldw, int M, int N, int K, const FastEpi & ep, int n_sm, int bn, cudaStream_t s) {
    if (K % kBK != 0 || K < kBK || M < 1 || N < 1) { fprintf(stderr, "bark_b200 fast mode: unsupported GEMM shape %d x %d x %d\n", M, N, K); return 0; }
    if (bn != 0 && bn != 64 && bn != 128 && bn != 256) { fprintf(stderr, "bark_b200 fast mode: tile width %d is not 64, 128 or 256\n", bn); return 0; }
    // Tile width.  These GEMMs are a few microseconds each, so the choice is about filling the SMs, one CTA per SM at a time:
    //   time(BN) ~ waves x (fixed per-CTA cost + operand bytes of one CTA / per-SM fill rate)
    // with an assumed ~3 us of prologue + epilogue drain per CTA and ~64 B/clk (~120 GB/s) from L2 into one SM's shared memory.
    // Narrow tiles re-read the 128 activation rows for every column tile, wide tiles leave SMs idle.
    const int tiles_m = (M + kBM - 1) / kBM;
    auto cost = [&](int bn) {
        const int tiles = tiles_m * ((N + bn - 1) / bn);
        return (double)((tiles + n_sm - 1) / n_sm) * (3.0 + (double)(kBM + bn) * K * 2.0 / 120e3);
    };
    int best = bn;
    if (best == 0) {
        best = 256;
        for (int b : {128, 64})
            if (cost(b) < cost(best) - 1e-9) best = b;
    }
    const bool ok = best == 256 ? launch_gemm<256>(A, lda, W, ldw, M, N, K, ep, s)
                  : best == 128 ? launch_gemm<128>(A, lda, W, ldw, M, N, K, ep, s)
                                : launch_gemm<64>(A, lda, W, ldw, M, N, K, ep, s);
    return ok ? best : 0;
}

// att[N][E] (f16) = soft_max(Q K^T / sqrt(64)) V per head; qk: [N][ldq] f16 with Q at column h*64 and K at k_col0 + h*64; vt: V^T [E][N] f16
bool fast_attention(const __half * qk, int ldq, int k_col0, const __half * vt, int n, int E, int H, __half * out, cudaStream_t s) {
    if (E / H != kHeadD || n % kKeyBlk != 0 || n < kKeyBlk) { fprintf(stderr, "bark_b200 fast mode: attention needs head size 64 and a multiple of %d positions (got %d heads of %d, %d positions)\n", kKeyBlk, H, E / H, n); return false; }
    const size_t smem = (size_t) FlashSmem::total + 1024;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_this_device(configured)) BARK_CUDA_CHECK(cudaFuncSetAttribute(flash_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    CUtensorMap tqk, tvt;
    if (!make_map(&tqk, qk, n, k_col0 + E, ldq, 128) || !make_map(&tvt, vt, E, n, n, 64)) return false;
    const float scale_log2e = (1.0f / sqrtf((float) kHeadD)) * 1.4426950408889634f;
    g_next_flops = 4.0 * (double) n * n * E;
    g_next_bytes = 2.0 * 4.0 * (double) n * E;
    BARK_LAUNCH_PDL(flash_attn_kernel, dim3(n / 128, H), dim3(kGemmThreads), smem, s, tqk, tvt, n, k_col0, scale_log2e, out, E);
    return true;
}

void fast_layernorm(const float * x, int rows, int E, const float * g, const float * b, __half * out, cudaStream_t s) {
    BARK_LAUNCH_PDL(ln_rows_f16_kernel, dim3((rows + 7) / 8), dim3(256), (size_t) 0, s, x, rows, E, g, b, out);
}

void fast_convert(const void * src, WType t, int n_out, int K, __half * dst, int * non_finite, cudaStream_t s) {
    const size_t n = (size_t) n_out * K;
    g_next_bytes = (double) n * 2 + (t == W_F32 ? (double) n * 4 : (double)(n / 32) * (t == W_Q4_0 ? 18 : qx_block_bytes(t)));
    BARK_LAUNCH(convert_f16_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, (const unsigned char *) src, t, n, dst, non_finite);
}

}  // namespace bark
