// Device-side Hades permutation for BLS12-381 Fr on sm_90a -- one width-5 state per thread, all
// 40 state words in registers.
//
// Replaces, on the batch path, the reference's scalar loop
//   Hades::perm                      src/hades/permutation.rs:105-123
//   add_round_constants / quintic_s_box / mul_matrix
//                                    src/hades/permutation/scalar.rs:39-64
// with the bit-exact "scaled lazy" formulation derived in tools/hades_model.py:
//   * 300 unreduced Montgomery products + 65 products by a table constant ("constant folds", 78 instead of 120
//     IMAD.WIDE each) per permutation (carry chains, fr_ptx.cuh) instead of the reference's 2000 (dense 25-multiply
//     MDS every round);
//   * the MDS layer is 25 small-integer (<= 17 bit) multiply-adds per round, computed EXACTLY in FP64
//     (DFMA on the otherwise idle FP64 pipe; column sums < 2^52) followed by ONE Montgomery row per
//     lane; round constants ride inside that same accumulation;
//   * values stay in [0, 2^256) with no modular correction at all between the first round's add and the
//     final output (bound analysis: DESIGN.md "Operand bounds"; asserted by the emulator and the model).
// Input and output are BlsScalar.0 (4 x u64 LE limbs, Montgomery form, < p), bit-exact.
#pragma once
#include <stdint.h>

#include "fr_ptx.cuh"

#ifndef P252_CONST_SMEM
#define P252_CONST_SMEM 0     // 1: round tables staged into shared memory with one TMA bulk copy per block
#endif

namespace p252 {

#include "hades_tables.inc"

#if P252_CONST_SMEM
// Experiment (north_star's suggestion): stage kA|kGT into shared memory once per block with cp.async.bulk
// (TMA, completion on an mbarrier) and read them with broadcast LDS instead of LDCU from the constant bank.
__device__ __forceinline__ const uint32_t* stage_round_tables(uint32_t* s_tab, uint64_t* mbar) {
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(mbar);
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(s_tab);
    constexpr uint32_t kBytes = P252_TAB_WORDS * 4;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(kBytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                     "l"(gRoundTab), "r"(kBytes), "r"(bar)
                     : "memory");
    }
    uint32_t done = 0;
    while (!done) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done)
                     : "r"(bar)
                     : "memory");
    }
    return s_tab;
}
#define P252_TAB_ARG , const uint32_t* tab
#define P252_TAB_PASS , tab
#define P252_A_ROW(round, lane) (tab + ((round) * 5 + (lane)) * 12)
#define P252_G_ROW(idx) (tab + P252_TAB_A_WORDS + (idx) * 64)
#else
#define P252_TAB_ARG
#define P252_TAB_PASS
#define P252_A_ROW(round, lane) (kA[round][lane])
#define P252_G_ROW(idx) (&kGT[idx][0][0])
#endif

// hades_tables.inc defines, in the constant bank (statically initialised at module load):
//   kA0[5][8], kA[69][5][12]  per-round additive constants (scaled)   kGT[60][8][8]  lane-4 correction (fold table)
//   kFT[8][8]     final multiplier (fold table)             kDenseArc / kDenseMds  dense tables
// Every thread of a warp reads the same word in the same instruction (the round index is
// warp-uniform), which the constant cache serves as a broadcast operand.

constexpr int kRounds = 68;
constexpr int kHalfFull = 4;
constexpr int kPartial = 60;

// Work per permutation in this formulation (see hades_permute below): 100 S-boxes (5 per full round, 1 per partial
// round) = 200 squarings + 100 products; 60 lane-4 corrections and 5 final products as constant folds; 68 mixes of 5
// Montgomery rows.
constexpr int kSboxPerPerm = 2 * kHalfFull * 5 + kPartial;
constexpr int kMontSqrPerPerm = 2 * kSboxPerPerm;
constexpr int kMontMulPerPerm = kSboxPerPerm;
constexpr int kFoldPerPerm = kPartial + 5;
constexpr int kWideMulPerPerm = kMontSqrPerPerm * (kWideOps_fr_sqr_wide + kWideOps_fr_redc_wide) +
                                kMontMulPerPerm * (kWideOps_fr_row_first + 7 * kWideOps_fr_row) +
                                kFoldPerPerm * kWideOps_fr_cfold + kRounds * 5 * kWideOps_fr_arc_redc1;
constexpr int kDfmaPerPerm = kRounds * 5 * 5 * 8;

// r = (x*y + m p) / 2^256.  Row operand x must satisfy x + p <= 2^256; y < 2^256.
__device__ __forceinline__ void montmul(uint32_t (&r)[8], const uint32_t (&x)[8],
                                        const uint32_t (&y)[8]) {
    uint32_t a[8], b[8];
    fr_row_first(a, b, x, y[0]);
    fr_row(b, a, x, y[1]);
    fr_row(a, b, x, y[2]);
    fr_row(b, a, x, y[3]);
    fr_row(a, b, x, y[4]);
    fr_row(b, a, x, y[5]);
    fr_row(a, b, x, y[6]);
    fr_row(b, a, x, y[7]);
    fr_merge(r, b, a);
}

// r = (a*a + m p) / 2^256: 36-product square, then eight Montgomery rows on the low half + high half.
__device__ __forceinline__ void montsqr(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    uint32_t t[16];
    fr_sqr_wide(t, a);
    fr_redc_wide(r, t);
}

// z = u^5 / R^4 (unreduced): two squarings and one product like quintic_s_box
// (src/hades/permutation/scalar.rs:50-52).  u < 1.0003 p  =>  z < 1.89 p.
__device__ __forceinline__ void sbox(uint32_t (&z)[8], const uint32_t (&u)[8]) {
    uint32_t a[8], b[8];
    montsqr(a, u);             // < 1.4533 p
    montsqr(b, a);             // < 1.9564 p
    montmul(z, u, b);          // row operand u (u + p <= 2^256), result < 1.8861 p
}

__device__ __forceinline__ void load_const(uint32_t (&d)[8], const uint32_t* c) {
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = c[k];
}

// r = C w / R (mod p) for a constant C given by its fold table tab[8 j + k] = limb k of C 2^(32j - 192) mod p
// (gen_tables.py): S = sum_j w_j T_j < 8 * 2^32 p < 2^290 over the 32-bit limbs w_j of w, then two Montgomery rows,
// r = (S + m0 p + m1 p 2^32) / 2^64 < p + 2^226.  The same residue as montmul(C, w) (so the scale bookkeeping is
// unchanged) for 64 + 2 * 7 multiplier instructions instead of 8 * 15.  w < 2^256, any value.  The table index is
// warp-uniform, so every limb is a broadcast constant operand.
__device__ __forceinline__ void cfold(uint32_t (&r)[8], const uint32_t* tab, const uint32_t (&w)[8]) {
    uint32_t ev[9], od[9], t[8];
    load_const(t, tab);
    fr_fold_row_first(ev, od, t, w[0]);
#pragma unroll
    for (int j = 1; j < 8; ++j) {
        load_const(t, tab + 8 * j);
        fr_fold_row(ev, od, t, w[j]);
    }
    uint32_t s[10], u[9];
    fr_fold_merge(s, ev, od);
    fr_redc1_10(u, s);
    fr_redc1(r, u);
}

// Partial-round S-box of lane 4 with its correction: z = G u^5 / R^5 = montmul(cfold(G, u), u^4 / R^3).  The fold
// g = G u / R depends on u alone, so it runs alongside the two squarings instead of after the S-box; g < p + 2^226
// keeps the row-operand condition g + p <= 2^256 of the last product.  z < 1.887 p.
__device__ __forceinline__ void sbox_partial(uint32_t (&z)[8], const uint32_t (&u)[8], const uint32_t* gtab) {
    uint32_t g[8], a[8], b[8];
    cfold(g, gtab, u);
    montsqr(a, u);             // < 1.4533 p
    montsqr(b, a);             // < 1.9564 p
    montmul(z, g, b);
}

constexpr double kTwo52 = 4503599627370496.0;

// s <- redc1(C s + A[next_round]) in place -- mul_matrix (+ the next add_round_constants) of the reference,
// src/hades/permutation/scalar.rs:39-48,54-64.
//
// The 25 products per round are (<= 17 bit constant) x (32-bit limb); a column sum over the five lanes is
// below 268697 * 2^32 < 2^50.1, i.e. EXACT in an IEEE double.  The FP64 pipe is left idle by the integer
// S-box, so the column sums are formed with DFMA there (concurrently with the IMAD.WIDE carry
// chains on the fmaheavy pipe) instead of 40 IMAD.WIDE per lane:
//   limb -> double      : I2F.F64.U32 (exact)
//   acc = 2^52 + sum_j c_ij * limb_j   (five DFMA; every partial sum is an integer < 2^53: no rounding)
//   raw bits of acc     = 0x43300000_00000000 + column sum
// Limb-major: for limb k the five lanes' limbs are converted once and the five raw columns are folded straight
// into the 9-limb totals t[i] (column k overlaps column k+1 by its upper word).  The exponent words are not
// masked off: their sum K_off is pre-subtracted (mod 2^288) from the 9-limb round constant kA[next_round][i],
// and the addition inside fr_arc_redc1 wraps to the true integer C s + A < 2^288.
__device__ __forceinline__ void mix(uint32_t (&s)[5][8], int next_round P252_TAB_ARG) {
    uint32_t t[5][9];
    uint32_t hi_prev[5] = {0, 0, 0, 0, 0}, carry[5] = {0, 0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        double d[5];
#pragma unroll
        for (int j = 0; j < 5; ++j) d[j] = (double)s[j][k];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            double acc = kTwo52;
#pragma unroll
            for (int j = 0; j < 5; ++j) acc = fma((double)hades_cmat(i, j), d[j], acc);
            const uint64_t sum = (uint64_t)(uint32_t)__double2loint(acc) + hi_prev[i] + carry[i];
            t[i][k] = (uint32_t)sum;
            carry[i] = (uint32_t)(sum >> 32);
            hi_prev[i] = (uint32_t)__double2hiint(acc);
        }
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        t[i][8] = hi_prev[i] + carry[i];
        uint32_t c[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) c[k] = P252_A_ROW(next_round, i)[k];
        fr_arc_redc1(s[i], t[i], c);
    }
}

// In-register Hades permutation, standard Montgomery form in and out (both < p).
// out_lanes: bit i set = lane i of the result is needed.  The last permutation of a sponge is only ever read through
// the rate lanes it squeezes (a Merkle digest: lane 1), so the output multiplication + final subtraction of the other
// lanes is skipped (warp-uniform branch); lanes not asked for are left in the internal scaled form and must not be used.
__device__ __forceinline__ void hades_permute(uint32_t (&s)[5][8], uint32_t out_lanes P252_TAB_ARG) {
    uint32_t c[8];
    // first add_round_constants: explicit, then one full conditional subtraction
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        load_const(c, kA0[i]);
        uint32_t t[8];
        fr_add_lazy(t, s[i], c);
        fr_condsub(t);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[i][k] = t[k];
    }
#pragma unroll 1
    for (int r = 0; r < kRounds; ++r) {
        const bool full = (r < kHalfFull) || (r >= kHalfFull + kPartial);
        if (full) {
            // one S-box code instance on slot 4, run five times, rotating the lanes through slot 4
#pragma unroll 1
            for (int it = 0; it < 5; ++it) {
                uint32_t w[8];
                sbox(w, s[4]);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    s[4][k] = s[3][k];
                    s[3][k] = s[2][k];
                    s[2][k] = s[1][k];
                    s[1][k] = s[0][k];
                    s[0][k] = w[k];
                }
            }
        } else {
            sbox_partial(s[4], s[4], P252_G_ROW(r - kHalfFull));
        }
        mix(s, r + 1 P252_TAB_PASS);      // r + 1 == kRounds: row 68 of kA carries no round constants
    }
    // leave the scaled domain: out = F v / R (constant fold) fully reduced
#pragma unroll 1
    for (int it = 0; it < 5; ++it) {
        uint32_t w[8];
        if ((out_lanes >> (4 - it)) & 1u) {            // slot 4 holds lane 4 - it
            cfold(w, &kFT[0][0], s[4]);
            fr_condsub(w);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) w[k] = s[4][k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            s[4][k] = s[3][k];
            s[3][k] = s[2][k];
            s[2][k] = s[1][k];
            s[1][k] = s[0][k];
            s[0][k] = w[k];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Lane-split permutation for SMALL batches: five threads per state, thread `li` of a group holds lane `li`.
//
// One permutation on one thread is a chain of ~106 k dependent-ish instructions (a single warp
// cannot issue its IMAD.WIDEs back to back); a batch that does not fill the machine (the top
// levels of a Merkle tree, a single Hash::digest) is bound by that latency, not by throughput.  Splitting the
// state over five threads takes the four idle S-boxes of a full round and four of the five mix rows off the
// critical path:  full round = 1 S-box + 1 mix row per thread (instead of 5 + 5), partial round = lane 4's
// S-box and correction + 1 mix row (instead of + 5 rows).  The mix needs every lane's limbs: 5 x 8 warp shuffles.
// Same integer arithmetic, same tables, same bounds as hades_permute() -> bit-identical results (tests compare the
// two paths and the oracle).  Throughput per state is ~3x worse (6 states per warp instead of 32), so the
// launchers use it only below kCoopMaxItems.
//   li   : lane of the state this thread owns (0..4; the reference's S-box lane in partial rounds is 4,
//          src/hades/permutation.rs:68)
//   g0   : warp lane of the group's thread 0 (groups are 5 consecutive lanes; lanes 30,31 of a warp idle)
//   crow : this thread's row of the small-integer MDS as doubles, crow[j] = hades_cmat(li, j)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void coop_load_row(uint32_t (&c)[12], const uint32_t* row) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(row)), b = __ldg(reinterpret_cast<const uint4*>(row) + 1),
                d = __ldg(reinterpret_cast<const uint4*>(row) + 2);
    c[0] = a.x, c[1] = a.y, c[2] = a.z, c[3] = a.w, c[4] = b.x, c[5] = b.y, c[6] = b.z, c[7] = b.w;
    c[8] = d.x, c[9] = d.y, c[10] = d.z, c[11] = d.w;
}

__device__ __forceinline__ void coop_mix(uint32_t (&s)[8], int next_round, int li, int g0, const double (&crow)[5]) {
    uint32_t a12[12];
    coop_load_row(a12, gA[next_round][li]);          // issued first: its latency hides behind the shuffles
    uint32_t t[9];
    uint32_t hi_prev = 0, carry = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        double acc = kTwo52;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const uint32_t z = __shfl_sync(0xffffffffu, s[k], g0 + j);
            acc = fma(crow[j], (double)z, acc);
        }
        const uint64_t sum = (uint64_t)(uint32_t)__double2loint(acc) + hi_prev + carry;
        t[k] = (uint32_t)sum;
        carry = (uint32_t)(sum >> 32);
        hi_prev = (uint32_t)__double2hiint(acc);
    }
    t[8] = hi_prev + carry;
    uint32_t c[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) c[k] = a12[k];
    fr_arc_redc1(s, t, c);
}

__device__ __forceinline__ void hades_permute_coop(uint32_t (&s)[8], int li, int g0, const double (&crow)[5]) {
    {
        // first add_round_constants + one full conditional subtraction, exactly as hades_permute()
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(gA0[li])), b = __ldg(reinterpret_cast<const uint4*>(gA0[li]) + 1);
        const uint32_t c[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        uint32_t t[8];
        fr_add_lazy(t, s, c);
        fr_condsub(t);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] = t[k];
    }
#pragma unroll 1
    for (int r = 0; r < kRounds; ++r) {
        const bool full = (r < kHalfFull) || (r >= kHalfFull + kPartial);
        // every thread runs the S-box; in partial rounds only lane 4 keeps it
        if (full) {
            uint32_t w[8];
            sbox(w, s);
#pragma unroll
            for (int k = 0; k < 8; ++k) s[k] = w[k];
        } else {
            uint32_t z[8];
            sbox_partial(z, s, &kGT[r - kHalfFull][0][0]);   // always the constant bank (warp-uniform index)
#pragma unroll
            for (int k = 0; k < 8; ++k) s[k] = (li == 4) ? z[k] : s[k];
        }
        coop_mix(s, r + 1, li, g0, crow);
    }
    uint32_t w[8];
    cfold(w, &kFT[0][0], s);
    fr_condsub(w);
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = w[k];
}

// ---------------------------------------------------------------------------------------------
// Modular add / sub on fully reduced operands (Safe::add, Encryption::subtract,
// src/hades/permutation/scalar.rs:33-35,69-75)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void fr_add_mod(uint32_t (&r)[8], const uint32_t (&a)[8],
                                           const uint32_t (&b)[8]) {
    fr_add_lazy(r, a, b);
    fr_condsub(r);
}

// Montgomery form -> canonical integer in [0,p): x / R, i.e. the eight reduction rows alone applied to (x, 0)
// (no product needed), then one conditional subtraction (Scalar::reduce)
__device__ __forceinline__ void fr_to_canonical(uint32_t (&r)[8], const uint32_t (&x)[8]) {
    uint32_t t[16];
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] = x[k], t[8 + k] = 0;
    fr_redc_wide(r, t);        // (x + m p) / 2^256 < p + 1
    fr_condsub(r);
}

// canonical integer (any 256-bit value) -> Montgomery form of (c mod p): c * R^2 / R
__device__ __forceinline__ void fr_from_canonical(uint32_t (&r)[8], const uint32_t (&c)[8]) {
    const uint32_t r2[8] = {0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u,
                            0x0748d9d9u};   // R^2 mod p
    montmul(r, r2, c);         // row operand R^2 < p; c < 2^256  =>  result < 2p
    fr_condsub(r);
}

// c < p ?  (borrow of c - p)
__device__ __forceinline__ bool fr_is_canonical(const uint32_t (&c)[8]) {
    uint32_t t[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] = c[k];
    fr_condsub(t);             // t = c - p if c >= p else c   (valid for c < 2p; c >= 2p also changes t)
    bool same = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) same = same && (t[k] == c[k]);
    return same;
}

// ---------------------------------------------------------------------------------------------
// Dense formulation: the reference's algorithm verbatim on the device (25 full products per MDS,
// full reduction after every operation).  Cross-check / "what a straight port would cost".
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void dense_mul(uint32_t (&r)[8], const uint32_t (&x)[8],
                                          const uint32_t (&y)[8]) {
    montmul(r, x, y);          // x < p  => x + p < 2^256
    fr_condsub(r);
}

__device__ __forceinline__ void dense_permute(uint32_t (&s)[5][8]) {
#pragma unroll 1
    for (int r = 0; r < kRounds; ++r) {
        const bool full = (r < kHalfFull) || (r >= kHalfFull + kPartial);
        uint32_t c[8], t[8];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            load_const(c, kDenseArc[r * 5 + i]);
            fr_add_mod(t, s[i], c);
#pragma unroll
            for (int k = 0; k < 8; ++k) s[i][k] = t[k];
        }
#pragma unroll 1
        for (int it = 0; it < 5; ++it) {
            uint32_t w[8];
            if (full || it == 0) {
                uint32_t a[8], b[8];
                dense_mul(a, s[4], s[4]);
                dense_mul(b, a, a);
                dense_mul(w, s[4], b);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = s[4][k];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                s[4][k] = s[3][k];
                s[3][k] = s[2][k];
                s[2][k] = s[1][k];
                s[1][k] = s[0][k];
                s[0][k] = w[k];
            }
        }
        uint32_t acc[5][8];
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[i][k] = 0;
#pragma unroll 1
        for (int j = 0; j < 5; ++j) {
            // column j of the matrix times lane j; rotate the lanes so indexing stays static
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                load_const(c, kDenseMds[i * 5 + j]);
                uint32_t pr[8], sum[8];
                dense_mul(pr, c, s[0]);
                fr_add_mod(sum, acc[i], pr);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[i][k] = sum[k];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                uint32_t t0 = s[0][k];
                s[0][k] = s[1][k];
                s[1][k] = s[2][k];
                s[2][k] = s[3][k];
                s[3][k] = s[4][k];
                s[4][k] = t0;
            }
        }
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int k = 0; k < 8; ++k) s[i][k] = acc[i][k];
    }
}

}  // namespace p252
