// Micro-benchmarks of the primitives the persistent decode step is built from (DESIGN.md §9): run on the GPU BEFORE redesigning
// the step, ~10 s in total.
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo tools/microbench/exchange_bench.cu -o /tmp/exchange_bench
//   /tmp/exchange_bench
//
// 1. tagged exchange: P producer CTAs publish W 8-byte {value, epoch} words each (st.relaxed.gpu) at a common start time; every CTA
//    of the grid then needs ALL P*W words (ld.relaxed.gpu polling, as consume_to_smem does).  Reported: time from the publish instant to
//    the last consumer being done, for different poll back-offs and for consumers that start polling EARLY (a given time before the
//    publish) — the situation of the residual exchanges, where the decode step measured 1.5-2 us instead of 0.6 us.
// 2. grid-wide barrier (cooperative groups grid.sync) round trip.
// 3. thread-block cluster: barrier.cluster arrive+wait round trip and a DSMEM store -> remote load hand-off, cluster sizes 2/4/8.
// 4. __nanosleep(n): what a sleep of n ns really costs.
// 5. one elected thread issuing k TMA bulk copies (cp.async.bulk) of 1536 B: issue cost per copy and completion latency.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>

namespace cg = cooperative_groups;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

typedef unsigned long long u64;
__device__ __forceinline__ u64 gtime() { u64 t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void publish(u64 * p, float v, uint32_t tag) { const u64 w = ((u64) tag << 32) | (u64) __float_as_uint(v); asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory"); }
__device__ __forceinline__ u64 peek(const u64 * p) { u64 w; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory"); return w; }

// ---- 1. tagged exchange ------------------------------------------------------------------------------------------
// words: [n_words] tagged slots.  Every CTA: wait until t_start - early_ns, then poll all words (512 threads, 2 words each for 768
// words); producers (CTAs < n_prod... all CTAs own words_per_cta consecutive words) publish at t_start.  out[cta] = done time - t_start.
__global__ void __launch_bounds__(512, 1) exchange_kernel(u64 * words, int n_words, uint32_t tag, u64 t_start, unsigned early_ns, unsigned poll_ns, long long * out) {
    const int tid = threadIdx.x, cta = blockIdx.x, G = gridDim.x;
    const int base = n_words / G, rem = n_words % G;
    const int w0 = cta * base + min(cta, rem), w1 = w0 + base + (cta < rem ? 1 : 0);
    // producer part: lane 0 of warp (w - w0) publishes word w at t_start (like lane 0 of a row-owning warp)
    const int warp = tid >> 5, lane = tid & 31;
    const bool is_prod = lane == 0 && w0 + warp < w1;
    if (is_prod) {
        while (gtime() < t_start) { }
        publish(words + w0 + warp, 1.0f, tag);
    } else {
        while (gtime() + early_ns < t_start) { }                       // consumers start polling `early_ns` before the publish instant
    }
    __syncwarp();
    for (int i = tid; i < n_words; i += 512) {
        u64 w = peek(words + i);
        const u64 ts = gtime();
        while ((uint32_t)(w >> 32) != tag && gtime() - ts < 20ull * 1000 * 1000) { if (poll_ns) __nanosleep(poll_ns); w = peek(words + i); }   // bounded: a bug must not hang the box
    }
    __syncthreads();
    if (tid == 0) out[cta] = (long long) gtime() - (long long) t_start;
}

// ---- 2. grid barrier -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512, 1) gridsync_kernel(int iters, long long * out) {
    cg::grid_group g = cg::this_grid();
    g.sync();
    const u64 t0 = gtime();
    for (int i = 0; i < iters; i++) g.sync();
    if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = (long long)(gtime() - t0) / iters;
}

// ---- 3. cluster barrier / DSMEM hand-off -------------------------------------------------------------------------
// ping-pong between ranks 0 and 1 of the cluster: 1 KB of payload written into the partner's shared memory by 256 threads, then a flag;
// the partner's thread 0 spins on its LOCAL flag, the block reads the payload and answers.  Every spin is bounded (kSpinLimitNs).
constexpr u64 kSpinLimitNs = 20ull * 1000 * 1000;
__global__ void __launch_bounds__(512, 1) cluster_kernel(int iters, long long * out) {
    cg::cluster_group cl = cg::this_cluster();
    __shared__ unsigned flag;
    __shared__ float payload[256];
    if (threadIdx.x == 0) flag = 0;
    cl.sync();
    u64 t0 = gtime();
    for (int i = 0; i < iters; i++) cl.sync();
    const long long t_bar = (long long)(gtime() - t0) / iters;
    const unsigned r = cl.block_rank();
    long long t_ring = 0; float acc = 0.f;
    if (r < 2 && cl.num_blocks() >= 2) {
        float * peer_payload = cl.map_shared_rank(payload, r ^ 1);
        unsigned * peer_flag = cl.map_shared_rank(&flag, r ^ 1);
        t0 = gtime();
        for (int i = 1; i <= iters; i++) {
            if (r == 0) {                                                // send, then wait for the answer
                if (threadIdx.x < 256) peer_payload[threadIdx.x] = acc + i;
                __syncthreads();
                if (threadIdx.x == 0) { asm volatile("fence.acq_rel.cluster;" ::: "memory"); *(volatile unsigned *) peer_flag = (unsigned) i; }
            }
            if (threadIdx.x == 0) { const u64 ts = gtime(); while (*(volatile unsigned *) &flag < (unsigned) i && gtime() - ts < kSpinLimitNs) { } asm volatile("fence.acq_rel.cluster;" ::: "memory"); }
            __syncthreads();
            acc += payload[threadIdx.x & 255];
            __syncthreads();
            if (r == 1) {                                                // answer
                if (threadIdx.x < 256) peer_payload[threadIdx.x] = acc;
                __syncthreads();
                if (threadIdx.x == 0) { asm volatile("fence.acq_rel.cluster;" ::: "memory"); *(volatile unsigned *) peer_flag = (unsigned) i; }
            }
        }
        t_ring = (long long)(gtime() - t0);
    }
    cl.sync();
    if (threadIdx.x == 0 && r == 0 && blockIdx.x == 0) { out[0] = t_bar; out[1] = t_ring / (2ll * iters); out[2] = (long long) acc; }
}

// ---- 4. nanosleep -------------------------------------------------------------------------------------------------
__global__ void nanosleep_kernel(unsigned ns, int iters, long long * out) {
    const u64 t0 = gtime();
    for (int i = 0; i < iters; i++) __nanosleep(ns);
    if (threadIdx.x == 0) out[0] = (long long)(gtime() - t0) / iters;
}

// ---- 5. TMA bulk-copy issue cost -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512, 1) tma_kernel(const unsigned char * src, int copies, long long * out) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ __align__(8) u64 bar;
    const uint32_t b = (uint32_t) __cvta_generic_to_shared(&bar), dst = (uint32_t) __cvta_generic_to_shared(sm);
    if (threadIdx.x == 0) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b)); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    if (threadIdx.x == 0) {
        const u64 t0 = gtime();
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)(copies * 1536)) : "memory");
        for (int c = 0; c < copies; c++)
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst + c * 1536), "l"(src + (size_t)(blockIdx.x * copies + c) * 1536), "r"(1536u), "r"(b) : "memory");
        const u64 t1 = gtime();
        asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(b) : "memory");
        const u64 t2 = gtime();
        if (blockIdx.x == 0) { out[0] = (long long)(t1 - t0); out[1] = (long long)(t2 - t0); }
    }
}

__global__ void read_timer(u64 * out) { *out = gtime(); }

int main() {
    int dev = 0; CK(cudaSetDevice(dev));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
    const int n_sm = prop.multiProcessorCount;
    printf("device %s, %d SMs\n", prop.name, n_sm);
    long long * d_out; CK(cudaMalloc(&d_out, 1024 * 8));
    u64 * d_t; CK(cudaMalloc(&d_t, 8));
    std::vector<long long> h(1024);

    // 1. exchange
    {
        const int n_words = 768;
        u64 * d_words; CK(cudaMalloc(&d_words, n_words * 8)); CK(cudaMemset(d_words, 0, n_words * 8));
        uint32_t tag = 1;
        printf("\n# 1. tagged exchange of %d words, %d CTAs x 512 threads (us from the publish instant to the last consumer done; median / max over CTAs)\n", n_words, n_sm);
        const unsigned earlies[] = {0, 500, 1000, 2000, 4000};
        const unsigned polls[] = {0, 40, 200, 1000};
        for (unsigned early : earlies) for (unsigned poll : polls) {
            double med = 0, mx = 0; const int reps = 5;
            for (int rep = 0; rep < reps; rep++, tag++) {
                read_timer<<<1, 1>>>(d_t); u64 t_now; CK(cudaMemcpy(&t_now, d_t, 8, cudaMemcpyDeviceToHost));
                const u64 t_start = t_now + 300000 + early;              // 0.3 ms ahead: every CTA is resident and spinning by then
                void * args[] = {(void *) &d_words, (void *) &n_words, (void *) &tag, (void *) &t_start, (void *) &early, (void *) &poll, (void *) &d_out};
                CK(cudaLaunchCooperativeKernel((const void *) exchange_kernel, dim3(n_sm), dim3(512), args, 0, 0));
                CK(cudaMemcpy(h.data(), d_out, n_sm * 8, cudaMemcpyDeviceToHost));
                std::vector<long long> v(h.begin(), h.begin() + n_sm); std::sort(v.begin(), v.end());
                med += v[n_sm / 2] / 1e3 / reps; mx += v[n_sm - 1] / 1e3 / reps;
            }
            printf("consumers start %4u ns early, poll back-off %4u ns: median %6.2f  max %6.2f\n", early, poll, med, mx);
        }
        CK(cudaFree(d_words));
    }
    // 2. grid.sync
    {
        int iters = 200; void * args[] = {(void *) &iters, (void *) &d_out};
        CK(cudaLaunchCooperativeKernel((const void *) gridsync_kernel, dim3(n_sm), dim3(512), args, 0, 0));
        CK(cudaMemcpy(h.data(), d_out, 8, cudaMemcpyDeviceToHost));
        printf("\n# 2. cooperative grid.sync, %d CTAs x 512: %.2f us per barrier\n", n_sm, h[0] / 1e3);
    }
    // 3. clusters
    printf("\n# 3. thread-block cluster (512 threads per CTA): barrier round trip, and 1 KB DSMEM store + flag -> neighbour read, per hop\n");
    for (int cs : {2, 4, 8}) {
        cudaLaunchConfig_t cfg = {}; cfg.gridDim = dim3(cs * 8); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = 0; cfg.stream = 0;
        cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        int iters = 200;
        cudaError_t e = cudaLaunchKernelEx(&cfg, cluster_kernel, iters, d_out);
        if (e != cudaSuccess) { printf("cluster size %d: launch failed (%s)\n", cs, cudaGetErrorString(e)); (void) cudaGetLastError(); continue; }
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), d_out, 24, cudaMemcpyDeviceToHost));
        printf("cluster size %d: barrier %.2f us, 1 KB DSMEM hand-off %.2f us per hop\n", cs, h[0] / 1e3, h[1] / 1e3);
    }
    // 4. nanosleep
    printf("\n# 4. __nanosleep(n), one thread: average cost\n");
    for (unsigned ns : {0u, 20u, 40u, 100u, 200u, 500u, 1000u, 2000u}) {
        nanosleep_kernel<<<1, 1>>>(ns, 200, d_out); CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), d_out, 8, cudaMemcpyDeviceToHost));
        printf("nanosleep(%4u): %6lld ns\n", ns, h[0]);
    }
    // 5. TMA issue
    {
        unsigned char * d_src; const size_t bytes = (size_t) n_sm * 64 * 1536; CK(cudaMalloc(&d_src, bytes)); CK(cudaMemset(d_src, 1, bytes));
        CK(cudaFuncSetAttribute(tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1536));
        printf("\n# 5. one thread issuing k bulk copies of 1536 B (all %d CTAs at once): issue time / time to completion, CTA 0\n", n_sm);
        for (int k : {1, 2, 4, 8, 16, 32}) {
            tma_kernel<<<n_sm, 512, 64 * 1536>>>(d_src, k, d_out); CK(cudaDeviceSynchronize());
            CK(cudaMemcpy(h.data(), d_out, 16, cudaMemcpyDeviceToHost));
            printf("k = %2d: issue %5lld ns, complete %5lld ns\n", k, h[0], h[1]);
        }
        CK(cudaFree(d_src));
    }
    return 0;
}
