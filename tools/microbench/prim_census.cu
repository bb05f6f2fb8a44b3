// Developer tool: each arithmetic primitive of the Hades kernel alone in a loop, so that tools/sass_census.py --loops
// gives the per-primitive SASS instruction mix (and so that variants of one primitive can be compared without a GPU).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -cubin -o /tmp/prim.cubin prim_census.cu
//   python tools/sass_census.py /tmp/prim.cubin --loops
// Run on a GPU it also times them (modmul/s), one dependent chain per thread at the kernel's occupancy.
#include <cstdio>
#include <cuda_runtime.h>
#include "../../poseidon252_b200/csrc/hades_device.cuh"

static int sm_count() {   // SMs of device 0 (132 on an H100 SXM)
    static int n = 0;
    if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

using namespace p252;

template <int MODE>
__global__ void __launch_bounds__(128, 5) prim(uint32_t* io, int iters) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (MODE <= 2) {
        uint32_t x[8], y[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = io[tid * 8 + k] & 0x3fffffff, y[k] = (io[(tid ^ 1) * 8 + k] + k) & 0x3fffffff;
#pragma unroll 1
        for (int it = 0; it < iters; ++it) {
            uint32_t r[8];
            if (MODE == 0) montmul(r, y, x);
            if (MODE == 1) montsqr(r, x);
            if (MODE == 2) sbox(r, x);
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = r[k];
            x[7] &= 0x3fffffff;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) io[tid * 8 + k] = x[k];
    } else {
        uint32_t s[5][8];
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int k = 0; k < 8; ++k) s[i][k] = io[(tid * 5 + i) * 8 + k] & 0x3fffffff;
#pragma unroll 1
        for (int it = 0; it < iters; ++it) {
            if (MODE == 3) mix(s, 1 + (it & 63));
            if (MODE == 4) hades_permute(s, 0x1fu);
        }
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int k = 0; k < 8; ++k) io[(tid * 5 + i) * 8 + k] = s[i][k];
    }
}

template <int MODE>
void run(const char* name, uint32_t* d, int blocks, int iters, double units) {
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    prim<MODE><<<blocks, 128>>>(d, 2);
    cudaEventRecord(a);
    prim<MODE><<<blocks, 128>>>(d, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double per_warp_cycles = ms * 1e-3 * khz * 1e3 / ((double)iters * blocks * 4 / ((double)sm_count() * 4));
    printf("%-10s %8.3f ms  %.3e /s   %.0f cycles per warp-op per sub-partition\n", name, ms,
           (double)blocks * 128 * iters * units / (ms * 1e-3), per_warp_cycles);
}

int main() {
    const int blocks = sm_count() * 5 * 4;
    uint32_t* d;
    cudaMalloc(&d, (size_t)blocks * 128 * 40 * 4);
    cudaMemset(d, 0x5a, (size_t)blocks * 128 * 40 * 4);
    run<0>("montmul", d, blocks, 2000, 1);
    run<1>("montsqr", d, blocks, 2000, 1);
    run<2>("sbox", d, blocks, 1000, 1);
    run<3>("mix", d, blocks, 1000, 1);
    run<4>("permute", d, blocks, 8, 1);
    printf("status: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
