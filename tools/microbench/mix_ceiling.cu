// Microbenchmark (developer tool): how busy can the IMAD pipe stay when the real Montgomery row (15 IMAD-class
// + 7 ALU instructions) is diluted with independent ALU / FP64 work, as in the full permutation kernel
// (1 IMAD.WIDE per ~3 issued instructions)?  Prints cycles per IMAD-class instruction per sub-partition.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../poseidon252_b200/csrc/fr_ptx.cuh"

static int sm_count() {   // SMs of device 0 (132 on an H100 SXM)
    static int n = 0;
    if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

template <int NALU, int NDFMA>
__global__ void __launch_bounds__(128, 5) kern(uint32_t* out, uint32_t b, int iters) {
    uint32_t e[8], o[8], x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) e[k] = threadIdx.x + k, o[k] = blockIdx.x + 3 * k, x[k] = b + k;
    double d[4] = {1.0 + threadIdx.x, 1.5, 2.5, 3.5};
    uint32_t s[8] = {1, 2, 3, 4, 5, 6, 7, 8};
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            p252::fr_row(e, o, x, b + r);
#pragma unroll
            for (int q = 0; q < NALU; ++q)      // dependent only on itself: one chain per register
                asm volatile("add.u32 %0, %0, %1;" : "+r"(s[q & 7]) : "r"(e[q & 7]));
#pragma unroll
            for (int q = 0; q < NDFMA; ++q)
                asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[q & 3]) : "d"(1.0000001), "d"(0.5));
        }
    }
    uint32_t acc = (uint32_t)(d[0] + d[1] + d[2] + d[3]);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += e[k] + o[k] + s[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int NALU, int NDFMA>
void run(uint32_t* d_out) {
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const int iters = 1000;
    const int blocks = sm_count() * 5;      // 5 warps per sub-partition, like the shipped kernels
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    kern<NALU, NDFMA><<<blocks, 128>>>(d_out, 12345u, 10);
    cudaEventRecord(a);
    kern<NALU, NDFMA><<<blocks, 128>>>(d_out, 12345u, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const double cycles = ms * 1e-3 * khz * 1e3;
    const double imads = (double)iters * 16 * 15 * 5;          // per sub-partition
    const double per_row = 22 + NALU + NDFMA;
    printf("row + %2d ALU + %2d DFMA  (%.2f instr per IMAD)  %.2f cycles per IMAD  -> pipe busy %.0f%% (4 cyc/IMAD.WIDE, 2/IMAD.HI)\n",
           NALU, NDFMA, per_row / 15.0, cycles / imads, 100.0 * (14 * 4 + 2) / 15.0 / (cycles / imads));
}

int main() {
    uint32_t* d_out;
    cudaMalloc(&d_out, sm_count() * 5 * 128 * sizeof(uint32_t));
    run<0, 0>(d_out);
    run<6, 0>(d_out);
    run<12, 0>(d_out);
    run<0, 6>(d_out);
    run<6, 6>(d_out);
    run<12, 6>(d_out);
    run<16, 6>(d_out);
    run<24, 8>(d_out);
    printf("status: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
