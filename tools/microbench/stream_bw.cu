// How fast can G SMs stream weights?  Decides whether the decode step can run inside ONE 16-CTA cluster (DSMEM exchanges, ~0.3 us per
// dependency) instead of across all CTAs through L2: the weight stream of a token (188 MB) must then come
// through 16 SMs' L2->shared-memory paths.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a tools/microbench/stream_bw.cu -o /tmp/stream_bw
// Each CTA: lane 0 of warp 0 issues cp.async.bulk copies of `chunk` bytes into a ring of shared-memory stages (mbarrier complete_tx);
// the other warps wait for each stage, touch it (one LDS per thread) and release it.  Every CTA streams its own region (cold: HBM).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)
typedef unsigned long long u64;
__device__ __forceinline__ u64 gtime() { u64 t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint32_t s32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mwait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0; long long t0 = clock64();
    while (!done) { asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
                    if (!done && clock64() - t0 > 4000000000ll) __trap(); }
}
template <int STAGES>
__global__ void __launch_bounds__(512, 1) stream_kernel(const unsigned char * src, size_t per_cta, int chunk, long long * out, float * sink) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ __align__(8) u64 full[STAGES], empty[STAGES];
    const int tid = threadIdx.x;
    if (tid == 0) { for (int s = 0; s < STAGES; s++) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&full[s]))); asm volatile("mbarrier.init.shared::cta.b64 [%0], 15;" ::"r"(s32(&empty[s]))); }
                    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    const int n = (int)(per_cta / chunk);
    const unsigned char * mine = src + (size_t) blockIdx.x * per_cta;
    float acc = 0.f;
    const u64 t0 = gtime();
    if (tid < 32) {
        if (tid == 0) for (int i = 0; i < n; i++) {
            const int s = i % STAGES;
            mwait(s32(&empty[s]), ((i / STAGES) & 1) ^ 1);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&full[s])), "r"((uint32_t) chunk) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(sm + (size_t) s * chunk)), "l"(mine + (size_t) i * chunk), "r"((uint32_t) chunk), "r"(s32(&full[s])) : "memory");
        }
    } else {
        for (int i = 0; i < n; i++) {
            const int s = i % STAGES;
            mwait(s32(&full[s]), (i / STAGES) & 1);
            acc += reinterpret_cast<const float *>(sm + (size_t) s * chunk)[tid];
            __syncwarp();
            if ((tid & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(&empty[s])) : "memory");
        }
    }
    __syncthreads();
    if (tid == 0) out[blockIdx.x] = (long long)(gtime() - t0);
    if (acc == 1234.5f) sink[0] = acc;
}
int main() {
    CK(cudaSetDevice(0));
    const size_t total = (size_t) 3 << 30;
    unsigned char * d; CK(cudaMalloc(&d, total)); CK(cudaMemset(d, 1, total));
    long long * d_out; CK(cudaMalloc(&d_out, 1024 * 8)); float * d_sink; CK(cudaMalloc(&d_sink, 4));
    const int STAGES = 12;
    CK(cudaFuncSetAttribute(stream_kernel<STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * 16384));
    printf("# G CTAs (one per SM) streaming disjoint cold regions through a %d-stage shared-memory ring (cp.async.bulk)\n", STAGES);
    for (int chunk : {16384, 4096}) for (int G : {1, 4, 8, 16, 32, 64, 132}) {
        const size_t per = ((size_t) 16 << 20);
        CK(cudaMemset(d, 2, total));                     // evict the L2 (3 GB written)
        stream_kernel<STAGES><<<G, 512, STAGES * 16384>>>(d, per, chunk, d_out, d_sink);
        CK(cudaDeviceSynchronize());
        std::vector<long long> h(G); CK(cudaMemcpy(h.data(), d_out, G * 8, cudaMemcpyDeviceToHost));
        long long mx = 0; for (long long v : h) mx = v > mx ? v : mx;
        printf("chunk %5d B  G %3d : %7.1f GB/s total, %6.1f GB/s per SM   (%.1f us for %zu MB per CTA)\n", chunk, G, G * (double) per / mx, (double) per / mx, mx / 1e3, per >> 20);
    }
    // L2-resident source (second pass over the same 64 MB): what the KV cache / re-read operands see
    for (int G : {8, 16, 32}) {
        const size_t per = ((size_t) 4 << 20);
        for (int rep = 0; rep < 2; rep++) { stream_kernel<STAGES><<<G, 512, STAGES * 16384>>>(d, per, 16384, d_out, d_sink); CK(cudaDeviceSynchronize()); }
        std::vector<long long> h(G); CK(cudaMemcpy(h.data(), d_out, G * 8, cudaMemcpyDeviceToHost));
        long long mx = 0; for (long long v : h) mx = v > mx ? v : mx;
        printf("L2-resident  G %3d : %7.1f GB/s total, %6.1f GB/s per SM\n", G, G * (double) per / mx, (double) per / mx);
    }
    return 0;
}
