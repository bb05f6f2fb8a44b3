// Microbenchmark (developer tool): cycles per IMAD.WIDE.U32 on one SM sub-partition, for
//   A: independent plain mad.wide (no carry; operands vary so that ptxas cannot strength-reduce them)      B: carry chains (mad.lo.cc/madc.hi.cc -> IMAD.WIDE.X)
//   C: the real interleaved Montgomery row (fr_row) D: A + one DFMA per wide   E: A + two IADD3 per wide
// as a function of resident warps per sub-partition.  nvcc -gencode arch=compute_90a,code=sm_90a -O3
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../poseidon252_b200/csrc/fr_ptx.cuh"

static int sm_count() {   // SMs of device 0 (132 on an H100 SXM)
    static int n = 0;
    if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

constexpr int REP = 32;

template <int MODE>
__global__ void kern(uint32_t* out, uint32_t b, int iters) {
    uint32_t e[8], o[8], x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) e[k] = threadIdx.x + k, o[k] = blockIdx.x + 3 * k, x[k] = b + k;
    uint64_t w[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k] = threadIdx.x * 7 + k;
    double d0 = threadIdx.x, d1 = 1.5, d2 = 2.5, d3 = 3.5;
    uint32_t s0 = 1, s1 = 2, s2 = 3, s3 = 4;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int r = 0; r < REP; ++r) {
            if (MODE == 0 || MODE == 3 || MODE == 4) {
                // 8 independent 64-bit accumulators, plain wide MAD (no carry)
#pragma unroll
                for (int k = 0; k < 8; ++k)   // multiplier taken from a neighbouring accumulator: not loop-invariant
                    asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[k]) : "r"((uint32_t)w[(k + 3) & 7]), "r"(x[k]));
                if (MODE == 3) {
                    asm volatile("fma.rn.f64 %0, %0, %4, %5; fma.rn.f64 %1, %1, %4, %5; fma.rn.f64 %2, %2, %4, %5; fma.rn.f64 %3, %3, %4, %5;"
                                 "fma.rn.f64 %0, %0, %4, %5; fma.rn.f64 %1, %1, %4, %5; fma.rn.f64 %2, %2, %4, %5; fma.rn.f64 %3, %3, %4, %5;"
                                 : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3) : "d"(1.0000001), "d"(0.5));
                }
                if (MODE == 4) {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        asm volatile("add.u32 %0, %0, %4; add.u32 %1, %1, %4; add.u32 %2, %2, %4; add.u32 %3, %3, %4;"
                                     : "+r"(s0), "+r"(s1), "+r"(s2), "+r"(s3) : "r"(b));
                }
            } else if (MODE == 1) {
                // two carry chains of 4 wide MADs each
                asm volatile("mad.lo.cc.u32 %0, %8, %12, %0; madc.hi.cc.u32 %1, %8, %12, %1; madc.lo.cc.u32 %2, %9, %12, %2; madc.hi.cc.u32 %3, %9, %12, %3;"
                             "madc.lo.cc.u32 %4, %10, %12, %4; madc.hi.cc.u32 %5, %10, %12, %5; madc.lo.cc.u32 %6, %11, %12, %6; madc.hi.u32 %7, %11, %12, %7;"
                             : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7])
                             : "r"(x[0]), "r"(x[2]), "r"(x[4]), "r"(x[6]), "r"(b));
                asm volatile("mad.lo.cc.u32 %0, %8, %12, %0; madc.hi.cc.u32 %1, %8, %12, %1; madc.lo.cc.u32 %2, %9, %12, %2; madc.hi.cc.u32 %3, %9, %12, %3;"
                             "madc.lo.cc.u32 %4, %10, %12, %4; madc.hi.cc.u32 %5, %10, %12, %5; madc.lo.cc.u32 %6, %11, %12, %6; madc.hi.u32 %7, %11, %12, %7;"
                             : "+r"(o[0]), "+r"(o[1]), "+r"(o[2]), "+r"(o[3]), "+r"(o[4]), "+r"(o[5]), "+r"(o[6]), "+r"(o[7])
                             : "r"(x[1]), "r"(x[3]), "r"(x[5]), "r"(x[7]), "r"(b));
            } else if (MODE == 2) {
                p252::fr_row(e, o, x, b + r);     // 15 IMAD-class + 6 IADD3, as in montmul
            }
        }
    }
    uint32_t acc = s0 + s1 + s2 + s3 + (uint32_t)(d0 + d1 + d2 + d3);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += e[k] + o[k] + (uint32_t)w[k] + (uint32_t)(w[k] >> 32);
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int MODE>
void run(const char* name, int wides_per_rep, uint32_t* d_out) {
    int dev_clock_khz = 0;
    cudaDeviceGetAttribute(&dev_clock_khz, cudaDevAttrClockRate, 0);
    const int iters = 2000;
    for (int w = 1; w <= 6; ++w) {
        const int threads = 128 * w;   // w warps per sub-partition
        if (threads > 1024) break;
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        kern<MODE><<<sm_count(), threads>>>(d_out, 12345u, 10);
        cudaEventRecord(a);
        kern<MODE><<<sm_count(), threads>>>(d_out, 12345u, iters);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        const double cycles = ms * 1e-3 * dev_clock_khz * 1e3;
        const double wides = (double)iters * REP * wides_per_rep * w;   // per sub-partition
        printf("%-28s warps/SMSP=%d  %.2f cycles per IMAD.WIDE per sub-partition (%.3f ms)\n", name, w, cycles / wides, ms);
    }
}

int main() {
    uint32_t* d_out;
    cudaMalloc(&d_out, sm_count() * 1024 * sizeof(uint32_t));
    run<0>("A plain wide, independent", 8, d_out);
    run<1>("B carry chains (2 x 4)", 8, d_out);
    run<2>("C real Montgomery row", 15, d_out);
    run<3>("D plain wide + 1 DFMA/wide", 8, d_out);
    run<4>("E plain wide + 2 ADD/wide", 8, d_out);
    cudaError_t e = cudaDeviceSynchronize();
    printf("status: %s\n", cudaGetErrorString(e));
    return 0;
}
