// Chained grid-wide exchange rounds: what ONE tagged exchange of the persistent decode step costs, and what replication buys.
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo tools/microbench/exchange_rounds.cu -o /tmp/exchange_rounds
//
// Every round: each CTA publishes its share of W tagged 8-byte {value, epoch} words (lane 0 of the row-owning warps, as run_phase does),
// then every CTA gathers ALL W words into shared memory (512 threads, as consume_to_smem does), block barrier, next round.  The time per
// round is the cost of one grid-wide dependency.  R replicas: the producer's lanes 0..R-1 store the same word into R copies of the
// vector; CTA c reads copy c % R, so every L2 line has n_cta / R readers instead of n_cta.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)
typedef unsigned long long u64;
__device__ __forceinline__ u64 gtime() { u64 t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void publish(u64 * p, float v, uint32_t tag) { const u64 w = ((u64) tag << 32) | (u64) __float_as_uint(v); asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory"); }
__device__ __forceinline__ u64 peek(const u64 * p) { u64 w; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory"); return w; }
__device__ __forceinline__ void peek2(const u64 * p, u64 & a, u64 & b) { asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory"); }

constexpr int kSpinLimit = 4 * 1000 * 1000;        // a bug must not hang the box: every spin is bounded
__device__ int g_timeout;

// mode 0: one word per load (consume_to_smem);  mode 1: two adjacent words per 16-byte load
template <int MAXJ>
__global__ void __launch_bounds__(512, 1) rounds_kernel(u64 * words, int W, int R, int rounds, uint32_t tag0, unsigned poll_ns, int mode, int work_ns, long long * out, float * sink) {
    extern __shared__ float sm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, cta = blockIdx.x, G = gridDim.x;
    const int base = W / G, rem = W % G;
    const int w0 = cta * base + min(cta, rem), w1 = w0 + base + (cta < rem ? 1 : 0);
    const int n = w1 - w0;
    const int a = w0 + ((warp * n) >> 4), b = w0 + (((warp + 1) * n) >> 4);      // this warp's words, like warp_rows
    float acc = 0.f;
    const u64 t_begin = gtime();
    for (int r = 0; r < rounds; r++) {
        const uint32_t tag = tag0 + r;
        u64 * buf = words + (size_t)(r & 1) * 37 * 4096;          // two buffers: a CTA one round ahead must not overwrite words others still wait for
        const u64 * mine = buf + (size_t)(cta % R) * W;
        if (work_ns) { const long long t = clock64(); while (clock64() - t < (long long) work_ns * 2) { } }   // ~2 cycles per ns
        for (int w = a; w < b; w++) if (lane < R) publish(buf + (size_t) lane * W + w, (float)(w + r), tag);
        if (mode == 0) {
            u64 v[MAXJ];
#pragma unroll
            for (int j = 0; j < MAXJ; j++) { const int i = tid + j * 512; if (i < W) v[j] = peek(mine + i); }
#pragma unroll
            for (int j = 0; j < MAXJ; j++) {
                const int i = tid + j * 512;
                if (i < W) {
                    int spins = 0;                         // (no %globaltimer reads in the rounds: one read costs far more than a poll)
                    while ((uint32_t)(v[j] >> 32) != tag) { if (poll_ns) __nanosleep(poll_ns); v[j] = peek(mine + i); if (++spins > kSpinLimit) { g_timeout = 1; break; } }
                    sm[i] = __uint_as_float((uint32_t) v[j]);
                }
            }
        } else {
            u64 v[MAXJ][2];
#pragma unroll
            for (int j = 0; j < (MAXJ + 1) / 2; j++) { const int i = 2 * (tid + j * 512); if (i < W) peek2(mine + i, v[j][0], v[j][1]); }
#pragma unroll
            for (int j = 0; j < (MAXJ + 1) / 2; j++) {
                const int i = 2 * (tid + j * 512);
                if (i < W) {
                    int spins = 0;
                    while ((uint32_t)(v[j][0] >> 32) != tag || (uint32_t)(v[j][1] >> 32) != tag) { if (poll_ns) __nanosleep(poll_ns); peek2(mine + i, v[j][0], v[j][1]); if (++spins > kSpinLimit) { g_timeout = 1; break; } }
                    sm[i] = __uint_as_float((uint32_t) v[j][0]); sm[i + 1] = __uint_as_float((uint32_t) v[j][1]);
                }
            }
        }
        __syncthreads();
        acc += sm[(tid * 7 + r) % W];
        __syncthreads();
    }
    const u64 t_end = gtime();
    if (tid == 0) out[cta] = (long long)(t_end - t_begin);
    if (acc == -1.f) sink[0] = acc;
}

int main() {
    CK(cudaSetDevice(0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int n_sm = prop.multiProcessorCount;
    printf("device %s, %d SMs\n", prop.name, n_sm);
    long long * d_out; CK(cudaMalloc(&d_out, 1024 * 8));
    float * d_sink; CK(cudaMalloc(&d_sink, 4));
    const int maxR = 37, maxW = 4096;
    u64 * d_words; CK(cudaMalloc(&d_words, (size_t) 2 * maxR * maxW * 8)); CK(cudaMemset(d_words, 0, (size_t) 2 * maxR * maxW * 8));
    CK(cudaFuncSetAttribute(rounds_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxW * 4));
    uint32_t tag = 1;
    const int rounds = 400;
    printf("# chained exchange rounds (%d rounds, %d CTAs x 512 threads): us per round = cost of one grid-wide tagged dependency\n", rounds, n_sm);
    for (int W : {768, 1024, 3072, 4096}) for (int mode : {0, 1}) for (unsigned poll : {0u, 40u}) for (int R : {1, 2, 4, 8, 16, 32}) for (int ctas : {n_sm, 96}) {
        if (ctas != n_sm && (R != 1 && R != 8)) continue;
        if (poll == 0 && mode == 1) continue;
        int work = 0;
        void * args[] = {(void *) &d_words, (void *) &W, (void *) &R, (void *) &rounds, (void *) &tag, (void *) &poll, (void *) &mode, (void *) &work, (void *) &d_out, (void *) &d_sink};
        CK(cudaLaunchCooperativeKernel((const void *) rounds_kernel<8>, dim3(ctas), dim3(512), args, (size_t) maxW * 4, 0));
        CK(cudaDeviceSynchronize());
        std::vector<long long> h(ctas); CK(cudaMemcpy(h.data(), d_out, ctas * 8, cudaMemcpyDeviceToHost));
        long long mx = 0; for (long long v : h) mx = v > mx ? v : mx;
        int to = 0; CK(cudaMemcpyFromSymbol(&to, g_timeout, 4));
        printf("W %4d  load %s  poll %3u ns  replicas %2d  CTAs %3d : %6.3f us per round%s\n", W, mode ? "16B" : " 8B", poll, R, ctas, mx / 1e3 / rounds, to ? "  TIMEOUT" : "");
        tag += rounds;
        if (to) { int z = 0; CK(cudaMemcpyToSymbol(g_timeout, &z, 4)); }
    }
    // with 1 us of independent work between publish rounds (stragglers / skew absorb part of the latency)
    for (int W : {768, 3072}) for (int R : {1, 8}) {
        int work = 1000, mode = 0; unsigned poll = 40;
        void * args[] = {(void *) &d_words, (void *) &W, (void *) &R, (void *) &rounds, (void *) &tag, (void *) &poll, (void *) &mode, (void *) &work, (void *) &d_out, (void *) &d_sink};
        CK(cudaLaunchCooperativeKernel((const void *) rounds_kernel<8>, dim3(n_sm), dim3(512), args, (size_t) maxW * 4, 0));
        CK(cudaDeviceSynchronize());
        std::vector<long long> h(n_sm); CK(cudaMemcpy(h.data(), d_out, n_sm * 8, cudaMemcpyDeviceToHost));
        long long mx = 0; for (long long v : h) mx = v > mx ? v : mx;
        printf("W %4d  replicas %2d  + 1000 ns of work per round: %6.3f us per round (exchange = this - 1.0)\n", W, R, mx / 1e3 / rounds);
        tag += rounds;
    }
    return 0;
}
