// Microbenchmark: Montgomery multiply / square throughput, current 8x32-bit carry-chain PTX vs the radix-2^29
// unsaturated prototype (plain IMAD.WIDE, no carry chains).  Dependent chain per thread; many warps.
#include <cstdio>
#include <cuda_runtime.h>
#include "../../poseidon252_b200/csrc/fr_ptx.cuh"
#include "fr29_proto.cuh"

static int sm_count() {   // SMs of device 0 (132 on an H100 SXM)
    static int n = 0;
    if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

__device__ __forceinline__ void montmul32(uint32_t (&r)[8], const uint32_t (&x)[8], const uint32_t (&y)[8]) {
    uint32_t a[8], b[8];
    p252::fr_row_first(a, b, x, y[0]); p252::fr_row(b, a, x, y[1]); p252::fr_row(a, b, x, y[2]); p252::fr_row(b, a, x, y[3]);
    p252::fr_row(a, b, x, y[4]); p252::fr_row(b, a, x, y[5]); p252::fr_row(a, b, x, y[6]); p252::fr_row(b, a, x, y[7]);
    p252::fr_merge(r, b, a);
}
__device__ __forceinline__ void montsqr32(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    uint32_t t[16];
    p252::fr_sqr_wide(t, a);
    p252::fr_redc_wide(r, t);
}

template <int MODE>
__global__ void __launch_bounds__(128, 5) kern(uint32_t* io, int iters) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (MODE < 2) {
        uint32_t x[8], y[8];
        for (int k = 0; k < 8; ++k) x[k] = io[tid * 8 + k] & 0x3fffffff, y[k] = (io[(tid ^ 1) * 8 + k] + k) & 0x3fffffff;
        for (int it = 0; it < iters; ++it) {
            uint32_t r[8];
            if (MODE == 0) montmul32(r, y, x); else montsqr32(r, x);
            for (int k = 0; k < 8; ++k) x[k] = r[k];
            x[7] &= 0x3fffffff;
        }
        for (int k = 0; k < 8; ++k) io[tid * 8 + k] = x[k];
    } else {
        uint32_t x[9], y[9];
        for (int k = 0; k < 9; ++k) x[k] = io[tid * 8 + (k & 7)] & fr29::MASK, y[k] = (io[(tid ^ 1) * 8 + (k & 7)] + k) & fr29::MASK;
        for (int it = 0; it < iters; ++it) {
            uint32_t r[9];
            if (MODE == 2) fr29::montmul(r, x, y); else fr29::montsqr(r, x);
            for (int k = 0; k < 9; ++k) x[k] = r[k];
        }
        for (int k = 0; k < 8; ++k) io[tid * 8 + k] = x[k] + x[8];
    }
}

template <int MODE>
void run(const char* name, uint32_t* d, int blocks) {
    const int iters = 2000;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    kern<MODE><<<blocks, 128>>>(d, 10);
    cudaEventRecord(a);
    kern<MODE><<<blocks, 128>>>(d, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    printf("%-32s %8.3f ms  %.3e modmul/s\n", name, ms, (double)blocks * 128 * iters / (ms * 1e-3));
}

int main() {
    const int blocks = sm_count() * 5 * 4;
    uint32_t* d;
    cudaMalloc(&d, (size_t)blocks * 128 * 8 * 4);
    cudaMemset(d, 0x5a, (size_t)blocks * 128 * 8 * 4);
    run<0>("montmul 8x32 carry chains", d, blocks);
    run<1>("montsqr 8x32 carry chains", d, blocks);
    run<2>("montmul 9x29 unsaturated", d, blocks);
    run<3>("montsqr 9x29 unsaturated", d, blocks);
    printf("status: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
