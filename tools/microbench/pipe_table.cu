// Microbenchmark (developer tool): issue cost per warp instruction per SM sub-partition for the opcodes the Hades
// kernel is made of, alone and in pairs, at 5 resident warps per sub-partition (the kernel's occupancy).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipe_table pipe_table.cu && ./pipe_table
// Every test body is REP copies of one asm block over 8 independent accumulators; check the SASS with
//   cuobjdump -sass pipe_table | grep -A40 'kernILi<k>E'
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

static int sm_count() {   // SMs of device 0 (132 on an H100 SXM)
    static int n = 0;
    if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
    return n;
}

constexpr int REP = 16;

#define ACC8(op)                                                                                       \
    op(0) op(1) op(2) op(3) op(4) op(5) op(6) op(7)


// one IMAD.WIDE.U32 Rd(pair), Ra, Rb|imm|UR, Rd(pair): the mad.lo.cc/madc.hi pair the kernel uses
#define WIDE_RR(k) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(q[2 * (k)]), "+r"(q[2 * (k) + 1]) : "r"(q[2 * (((k) + 3) & 7)]), "r"(x[k]))
#define WIDE_RI(k) asm volatile("mad.lo.cc.u32 %0, %2, 0x53bda402, %0; madc.hi.u32 %1, %2, 0x53bda402, %1;" : "+r"(q[2 * (k)]), "+r"(q[2 * (k) + 1]) : "r"(q[2 * (((k) + 3) & 7)]))
#define WIDE_RU(k) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(q[2 * (k)]), "+r"(q[2 * (k) + 1]) : "r"(q[2 * (((k) + 3) & 7)]), "r"(b))

template <int MODE>
__global__ void __launch_bounds__(128) kern(uint32_t* out, uint32_t b, int iters) {
    uint32_t q[16];
    uint32_t x[8], s[8];
    double d[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        q[2 * k] = threadIdx.x * 7 + k, q[2 * k + 1] = k;
        x[k] = b + k * 77 + threadIdx.x;
        s[k] = threadIdx.x + k;
        d[k] = threadIdx.x + 0.5 * k;
    }
    const double dc = 1.0000001, de = 0.5;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int r = 0; r < REP; ++r) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (MODE == 0)   // IMAD.WIDE.U32 R,R,R,R  (both multiplicands vector registers, one loop-variant)
                    WIDE_RR(k);
                if (MODE == 1)   // IMAD.WIDE.U32 R,R,imm,R
                    WIDE_RI(k);
                if (MODE == 2)   // IMAD.WIDE.U32 R,R,UR,R  (kernel parameter -> uniform register)
                    WIDE_RU(k);
                if (MODE == 3)   // IMAD.HI.U32
                    asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                if (MODE == 4)   // IMAD (lo)
                    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                if (MODE == 5)   // IADD3 (three live inputs)
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                if (MODE == 6)   // DFMA
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                if (MODE == 7)   // LOP3
                    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                if (MODE == 8)   // SHF
                    asm volatile("shf.l.wrap.b32 %0, %0, %1, 3;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]));
                if (MODE == 9) {   // wide(reg) + 1 IADD3
                    WIDE_RR(k);
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                }
                if (MODE == 10) {  // wide(reg) + 2 IADD3
                    WIDE_RR(k);
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(s[(k + 1) & 7]) : "r"(s[(k + 5) & 7]), "r"(x[k]));
                }
                if (MODE == 11) {  // wide(reg) + 1 DFMA
                    WIDE_RR(k);
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                }
                if (MODE == 12) {  // wide(reg) + 1 IMAD lo  (same pipe?)
                    WIDE_RR(k);
                    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                }
                if (MODE == 13) {  // wide(reg) + 3 ALU
                    WIDE_RR(k);
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(s[(k + 1) & 7]) : "r"(s[(k + 5) & 7]), "r"(x[k]));
                    asm volatile("shf.l.wrap.b32 %0, %0, %1, 3;" : "+r"(s[(k + 2) & 7]) : "r"(s[(k + 6) & 7]));
                }
                if (MODE == 14) {  // wide(imm) + 2 ALU
                    WIDE_RI(k);
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(s[(k + 1) & 7]) : "r"(s[(k + 5) & 7]), "r"(x[k]));
                }
                if (MODE == 15) {  // wide(reg) + 1 DFMA + 2 ALU
                    WIDE_RR(k);
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(s[(k + 1) & 7]) : "r"(s[(k + 5) & 7]), "r"(x[k]));
                }

                if (MODE == 20) {  // IMAD lo + IADD3 (fma pipe + alu pipe, both rt=2): 2 cycles per pair if the pipes overlap
                    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(q[k]) : "r"(q[(k + 3) & 7]), "r"(x[k]));
                }
                if (MODE == 21) {  // DFMA + IADD3
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(q[k]) : "r"(q[(k + 3) & 7]), "r"(x[k]));
                }
                if (MODE == 22) {  // DFMA + IMAD lo
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                }
                if (MODE == 23) {  // wide + IADD3 with one register source (imm + RZ)
                    WIDE_RR(k);
                    asm volatile("add.u32 %0, %0, 0x1234567;" : "+r"(s[k]));
                }
                if (MODE == 24) {  // wide + 2-register IADD3
                    WIDE_RR(k);
                    asm volatile("add.u32 %0, %0, %1;" : "+r"(s[k]) : "r"(x[k]));
                }
                if (MODE == 25) {  // wide + 2 x (one-register IADD3)
                    WIDE_RR(k);
                    asm volatile("add.u32 %0, %0, 0x1234567;" : "+r"(s[k]));
                    asm volatile("xor.b32 %0, %0, 0x7654321;" : "+r"(x[k]));
                }
                if (MODE == 26) {  // IMAD lo + IADD3 + DFMA: three pipes
                    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(s[k]) : "r"(s[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(q[k]) : "r"(q[(k + 3) & 7]), "r"(x[k]));
                    asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[k]) : "d"(dc), "d"(de));
                }
                if (MODE == 27) {  // wide with zero addend (mul.wide): 2 register reads
                    asm volatile("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(q[2 * k]), "=r"(q[2 * k + 1]) : "r"(s[k]), "r"(x[k]));
                    asm volatile("add.u32 %0, %0, %1;" : "+r"(s[k]) : "r"(q[2 * k + 1]));
                }
                if (MODE == 16)  // I2F.F64.U32
                    asm volatile("{.reg .f64 t; cvt.rn.f64.u32 t, %1; add.f64 %0, %0, t;}" : "+d"(d[k]) : "r"(s[k] + r));
                if (MODE == 17)  // DADD
                    asm volatile("add.f64 %0, %0, %1;" : "+d"(d[k]) : "d"(dc));
            }

            // ---- review item (iii): what a DFMA-based (FP64-limb) squaring PRODUCT would issue vs the IMAD one ----
            // Synthetic instruction mixes with the counts of DESIGN.md 4.1 (independent accumulators: an optimistic
            // throughput bound for both).  30: 36 IMAD.WIDE + 40 ALU (the shipped 8x32-bit squaring product).
            // 31: 72 DFMA + 24 DADD + 116 ALU (16-bit split of one operand, conversions by magic-number DADD, column
            // recombination).  32: blocks alternate 30 / 31, i.e. both pipes loaded on every sub-partition.
            if (MODE == 30 || (MODE == 32 && (blockIdx.x & 1) == 0)) {
                if (r % 2 == 0) {
#pragma unroll
                    for (int z = 0; z < 36; ++z) WIDE_RR(z & 7);
#pragma unroll
                    for (int q = 0; q < 20; ++q) {
                        asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[q & 7]) : "r"(s[(q + 3) & 7]), "r"(x[q & 7]));
                        asm volatile("shf.l.wrap.b32 %0, %0, %1, 1;" : "+r"(s[(q + 1) & 7]) : "r"(s[(q + 5) & 7]));
                    }
                }
            }
            if (MODE == 31 || (MODE == 32 && (blockIdx.x & 1) == 1)) {
                if (r % 2 == 0) {
#pragma unroll
                    for (int q = 0; q < 72; ++q) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[q & 7]) : "d"(dc), "d"(de));
#pragma unroll
                    for (int q = 0; q < 24; ++q) asm volatile("add.f64 %0, %0, %1;" : "+d"(d[q & 7]) : "d"(dc));
#pragma unroll
                    for (int q = 0; q < 58; ++q) {
                        asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(s[q & 7]) : "r"(s[(q + 3) & 7]), "r"(x[q & 7]));
                        asm volatile("shf.l.wrap.b32 %0, %0, %1, 1;" : "+r"(s[(q + 1) & 7]) : "r"(s[(q + 5) & 7]));
                    }
                }
            }
            if (MODE == 18) {  // carry chain: 4 IMAD.WIDE.X per chain, two chains
                asm volatile("mad.lo.cc.u32 %0, %8, %12, %0; madc.hi.cc.u32 %1, %8, %12, %1; madc.lo.cc.u32 %2, %9, %12, %2; madc.hi.cc.u32 %3, %9, %12, %3;"
                             "madc.lo.cc.u32 %4, %10, %12, %4; madc.hi.cc.u32 %5, %10, %12, %5; madc.lo.cc.u32 %6, %11, %12, %6; madc.hi.u32 %7, %11, %12, %7;"
                             : "+r"(s[0]), "+r"(s[1]), "+r"(s[2]), "+r"(s[3]), "+r"(s[4]), "+r"(s[5]), "+r"(s[6]), "+r"(s[7])
                             : "r"(x[0]), "r"(x[2]), "r"(x[4]), "r"(x[6]), "r"(x[1] + r));
                asm volatile("mad.lo.cc.u32 %0, %8, %12, %0; madc.hi.cc.u32 %1, %8, %12, %1; madc.lo.cc.u32 %2, %9, %12, %2; madc.hi.cc.u32 %3, %9, %12, %3;"
                             "madc.lo.cc.u32 %4, %10, %12, %4; madc.hi.cc.u32 %5, %10, %12, %5; madc.lo.cc.u32 %6, %11, %12, %6; madc.hi.u32 %7, %11, %12, %7;"
                             : "+r"(q[0]), "+r"(q[1]), "+r"(q[2]), "+r"(q[3]), "+r"(q[4]), "+r"(q[5]), "+r"(q[6]), "+r"(q[7])
                             : "r"(x[1]), "r"(x[3]), "r"(x[5]), "r"(x[7]), "r"(x[0] + r));
            }
        }
    }
    uint32_t acc = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += s[k] + q[2 * k] + q[2 * k + 1] + (uint32_t)d[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int MODE>
void run(const char* name, double inst_per_rep, uint32_t* d_out) {
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const int iters = 4000;
    for (int w : {1, 2, 5, 8}) {
        const int blocks = sm_count() * w;     // 128-thread blocks: one warp per sub-partition each
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        kern<MODE><<<blocks, 128>>>(d_out, 12345u, 10);
        cudaEventRecord(a);
        kern<MODE><<<blocks, 128>>>(d_out, 12345u, iters);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        const double cycles = ms * 1e-3 * khz * 1e3;
        const double groups = (double)iters * REP * w;     // per sub-partition
        printf("%-34s warps/SMSP=%d  %6.2f cycles per group of %.0f instr  (%.2f cyc/instr)\n", name, w, cycles / groups,
               inst_per_rep, cycles / groups / inst_per_rep);
    }
}

int main() {
    uint32_t* d_out;
    cudaMalloc(&d_out, sm_count() * 8 * 128 * sizeof(uint32_t));
    run<0>("IMAD.WIDE reg,reg", 8, d_out);
    run<1>("IMAD.WIDE reg,imm", 8, d_out);
    run<2>("IMAD.WIDE reg,uniform", 8, d_out);
    run<3>("IMAD.HI", 8, d_out);
    run<4>("IMAD lo", 8, d_out);
    run<5>("IADD3", 8, d_out);
    run<6>("DFMA", 8, d_out);
    run<7>("LOP3", 8, d_out);
    run<8>("SHF", 8, d_out);
    run<9>("WIDE + IADD3", 16, d_out);
    run<10>("WIDE + IADD3 + LOP3", 24, d_out);
    run<11>("WIDE + DFMA", 16, d_out);
    run<12>("WIDE + IMAD lo", 16, d_out);
    run<13>("WIDE + 3 ALU", 32, d_out);
    run<14>("WIDE(imm) + 2 ALU", 24, d_out);
    run<15>("WIDE + DFMA + 2 ALU", 32, d_out);
    run<16>("I2F.F64.U32 + DADD", 16, d_out);
    run<17>("DADD", 8, d_out);
    run<18>("IMAD.WIDE.X chains (2x4)", 8, d_out);
    run<20>("IMAD lo + IADD3", 16, d_out);
    run<21>("DFMA + IADD3", 16, d_out);
    run<22>("DFMA + IMAD lo", 16, d_out);
    run<23>("WIDE + IADD3(1 reg)", 16, d_out);
    run<24>("WIDE + IADD3(2 reg)", 16, d_out);
    run<25>("WIDE + 2 x 1-reg ALU", 24, d_out);
    run<26>("IMAD lo + IADD3 + DFMA", 24, d_out);
    run<27>("mul.wide(2 reads) + IADD3", 16, d_out);
    // per "squaring product": REP/2 = 8 products per loop iteration -> pass 1/8 of a group as the unit
    run<30>("IMAD sqr product (36W+40ALU) x8", 8, d_out);
    run<31>("FP64 sqr product (72DFMA+24DADD+116ALU) x8", 8, d_out);
    run<32>("both, alternating blocks x8", 8, d_out);
    printf("status: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
