// Dependent-chain latencies on one warp (cycles per operation): DADD, DFMA, FADD, 32-bit SHFL, 64-bit SHFL (two 32-bit), SHFL + DADD level
// (one level of the LayerNorm warp tree), bar.sync with 16 warps.  Build: nvcc -O3 -arch=sm_90a -o lat lat.cu
#include <cstdio>
#include <cuda_runtime.h>
template <int MODE>
__global__ void k(double * out, long long * cyc, int n) {
    double d = threadIdx.x * 1e-3 + 1.0; float f = threadIdx.x * 1e-3f + 1.0f; const double inc = 1e-9;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < n; i++) {
        if (MODE == 0) d = __dadd_rn(d, inc);
        if (MODE == 1) d = __fma_rn(d, 1.0000001, inc);
        if (MODE == 2) f = __fadd_rn(f, 1e-7f);
        if (MODE == 3) f = __shfl_xor_sync(0xffffffffu, f, 1);
        if (MODE == 4) d = __shfl_xor_sync(0xffffffffu, d, 1);
        if (MODE == 5) d = __dadd_rn(d, __shfl_xor_sync(0xffffffffu, d, 1));
        if (MODE == 6) __syncthreads();
        if (MODE == 7) f = __fadd_rn(f, __shfl_xor_sync(0xffffffffu, f, 1));
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) { cyc[0] = t1 - t0; }
    out[threadIdx.x] = d + f;
}
int main() {
    double * out; long long * cyc; cudaMalloc(&out, 4096 * 8); cudaMalloc(&cyc, 8);
    const char * names[] = {"DADD", "DFMA", "FADD", "SHFL32", "SHFL64", "SHFL64+DADD (one tree level)", "bar.sync", "SHFL32+FADD"};
    const int n = 4096;
    for (int threads : {32, 512}) {
        for (int m = 0; m < 8; m++) {
            long long h = 0;
            for (int rep = 0; rep < 2; rep++) {
                switch (m) {
                    case 0: k<0><<<1, threads>>>(out, cyc, n); break; case 1: k<1><<<1, threads>>>(out, cyc, n); break;
                    case 2: k<2><<<1, threads>>>(out, cyc, n); break; case 3: k<3><<<1, threads>>>(out, cyc, n); break;
                    case 4: k<4><<<1, threads>>>(out, cyc, n); break; case 5: k<5><<<1, threads>>>(out, cyc, n); break;
                    case 6: k<6><<<1, threads>>>(out, cyc, n); break; case 7: k<7><<<1, threads>>>(out, cyc, n); break;
                }
                cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
            }
            printf("%4d threads  %-30s %7.1f cycles per op\n", threads, names[m], (double) h / n);
        }
    }
    return 0;
}
