// Device-side JubJub arithmetic on the BLS12-381 Fr primitives of fr_ptx.cuh / hades_device.cuh: one scalar
// multiplication per thread, for the key exchange dhke(secret, public) = [s] public (p252_dhke_batch).
//
// The curve: a u^2 + v^2 = 1 + d u^2 v^2 over Fr (the same p as the permutation), a = -1,
// d = -10240/10241.  d is a non-square and -1 a square, so the unified addition law is complete: no identity,
// doubling or small-order exceptions.  Points are kept in extended twisted-Edwards coordinates (X : Y : Z : T) with
// u = X/Z, v = Y/Z, uv = T/Z (Hisil-Wong-Carter-Dawson 2008, a = -1).
//
// Operand bounds: every value this file produces is FULLY reduced (< p).  fr_add_mod / fr_sub_mod take and give [0, p);
// fmul / fsqr take operands < p, so the row operand satisfies x + p < 2p < 2^256 (the precondition of montmul in
// hades_device.cuh), the Montgomery product is < (p^2 + (2^256 - 1) p) / 2^256 < 2p (square: < 1.46 p), and one
// fr_condsub brings it below p.  No lazy reduction: the condsub costs ~17 instructions next to ~130 per product.
//
// Secret independence: the scalar only ever reaches a 4-bit digit that drives masked selects over the whole table
// (every entry is read, at addresses fixed by the loop counters), so neither a branch nor a memory address depends
// on a secret bit.  The inversion's chain is the fixed bit pattern of p - 2.
#pragma once
#include <stdint.h>

#include "hades_device.cuh"

namespace p252 {
namespace jj {

// Montgomery images (x R mod p, 8 x u32 LE) of the constants
__device__ __forceinline__ void set_one(uint32_t (&r)[8]) {
    const uint32_t c[8] = {0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau,
                           0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u};
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = c[k];
}
__device__ __forceinline__ void set_d(uint32_t (&r)[8]) {     // d = -10240/10241
    const uint32_t c[8] = {0xb974f6b0u, 0x2a522455u, 0x0d9acab3u, 0xfc6cc9efu,
                           0xc27628d1u, 0x7a08fb94u, 0xfe0e262eu, 0x57f8f6a8u};
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = c[k];
}
__device__ __forceinline__ void set_2d(uint32_t (&r)[8]) {
    const uint32_t c[8] = {0x72e9ed5fu, 0x54a448acu, 0x1b373967u, 0xa51befdbu,
                           0x7b4a799eu, 0xc0d81f21u, 0xd27ecf14u, 0x3c0445feu};
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = c[k];
}
// Order of the prime subgroup r_J (canonical, not Montgomery: 252 bits) and p - 2, the Fermat exponent of the inversion
// (255 bits, 164 of them set).  Immediates, not __constant__ data: indexed only by unrolled or public loop counters.
#define P252_JJ_ORDER {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau}
#define P252_JJ_PM2 {0xffffffffu, 0xfffffffeu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u}
constexpr int kPm2Bits = 255, kPm2Ones = 164;

// Products per scalar multiplication (montmul + montsqr), following the schedule below:
//   on-curve check 4, T and 2d T of the input 2, table entries 2..15 14 x (8 + 1), 63 windows x (3 doublings without T
//   x 7 + 1 doubling with T x 8 + 1 addition without T x 7), inversion (kPm2Bits - 1) squarings + (kPm2Ones - 1)
//   products, affine conversion 2.
constexpr int kWindows = 63;
constexpr int kProductsPerDhke = 4 + 2 + 14 * 9 + kWindows * (3 * 7 + 8 + 7) + (kPm2Bits - 1) + (kPm2Ones - 1) + 2;
static_assert(kProductsPerDhke == 2819, "product count of DESIGN.md section 4");

__device__ __forceinline__ void fmul(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    montmul(r, a, b);          // a < p  =>  a + p < 2^256; result < 2p
    fr_condsub(r);
}
__device__ __forceinline__ void fsqr(uint32_t (&r)[8], const uint32_t (&a)[8]) {
    montsqr(r, a);             // a < p  =>  result < 1.46 p
    fr_condsub(r);
}
__device__ __forceinline__ void fcopy(uint32_t (&r)[8], const uint32_t (&a)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = a[k];
}
// a == b for fully reduced a, b
__device__ __forceinline__ bool feq(const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    uint32_t x = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) x |= a[k] ^ b[k];
    return x == 0;
}
// c < r_J for 256-bit little-endian words (borrow of c - r_J)
__device__ __forceinline__ bool below_order(const uint32_t (&c)[8]) {
    const uint32_t m[8] = P252_JJ_ORDER;
    uint32_t borrow = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t t = (uint64_t)c[k] - m[k] - borrow;
        borrow = (uint32_t)(t >> 63);
    }
    return borrow != 0;
}

struct Ext {                    // extended coordinates, every coordinate < p
    uint32_t X[8], Y[8], Z[8], T[8];
};
struct Cached {                 // an addend prepared for add(): (Y - X, Y + X, 2d T, 2 Z)
    uint32_t ymx[8], ypx[8], kt[8], z2[8];
};

// on-curve check of an affine (u, v), u, v < p: -u^2 + v^2 == 1 + d u^2 v^2   (4 products)
__device__ __forceinline__ bool on_curve(const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    uint32_t uu[8], vv[8], w[8], c[8], lhs[8], rhs[8];
    fsqr(uu, u);
    fsqr(vv, v);
    fr_sub_mod(lhs, vv, uu);
    fmul(w, uu, vv);
    set_d(c);
    fmul(rhs, w, c);
    set_one(c);
    fr_add_mod(w, rhs, c);
    return feq(lhs, w);
}

__device__ __forceinline__ void to_cached(Cached& c, const Ext& p) {   // 1 product
    uint32_t k[8];
    fr_sub_mod(c.ymx, p.Y, p.X);
    fr_add_mod(c.ypx, p.Y, p.X);
    set_2d(k);
    fmul(c.kt, p.T, k);
    fr_add_mod(c.z2, p.Z, p.Z);
}

// r = p + q, unified and complete (add-2008-hwcd-3): 8 products, 7 without T3
template <bool kWantT>
__device__ __forceinline__ void add(Ext& r, const Ext& p, const Cached& q) {
    uint32_t a[8], b[8], c[8], d[8], e[8], f[8], g[8], h[8];
    fr_sub_mod(e, p.Y, p.X);
    fmul(a, e, q.ymx);          // A = (Y1 - X1)(Y2 - X2)
    fr_add_mod(e, p.Y, p.X);
    fmul(b, e, q.ypx);          // B = (Y1 + X1)(Y2 + X2)
    fmul(c, p.T, q.kt);         // C = T1 2d T2
    fmul(d, p.Z, q.z2);         // D = Z1 2 Z2
    fr_sub_mod(e, b, a);        // E = B - A
    fr_sub_mod(f, d, c);        // F = D - C
    fr_add_mod(g, d, c);        // G = D + C
    fr_add_mod(h, b, a);        // H = B + A
    fmul(r.X, e, f);
    fmul(r.Y, g, h);
    fmul(r.Z, f, g);
    if (kWantT) fmul(r.T, e, h);
}

// r = 2 p (dbl-2008-hwcd, a = -1): 4 squarings + 4 products, 3 without T3.  T of the input is not read.
template <bool kWantT>
__device__ __forceinline__ void dbl(Ext& r, const Ext& p) {
    uint32_t a[8], b[8], c[8], e[8], f[8], g[8], h[8];
    fsqr(a, p.X);               // A = X^2
    fsqr(b, p.Y);               // B = Y^2
    fsqr(c, p.Z);
    fr_add_mod(c, c, c);        // C = 2 Z^2
    fr_add_mod(e, p.X, p.Y);
    fsqr(h, e);
    fr_sub_mod(e, h, a);
    fr_sub_mod(e, e, b);        // E = (X + Y)^2 - A - B
    fr_sub_mod(g, b, a);        // G = D + B = B - A   (D = a A = -A)
    fr_sub_mod(f, g, c);        // F = G - C
    fr_add_mod(h, a, b);
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    fr_sub_mod(h, zero, h);     // H = D - B = -(A + B)
    fmul(r.X, e, f);
    fmul(r.Y, g, h);
    fmul(r.Z, f, g);
    if (kWantT) fmul(r.T, e, h);
}

// One cached table entry as 8 x 16 bytes (ymx, ypx, kt, z2), in thread-local memory.
struct Entry {
    uint4 w[8];
};
__device__ __forceinline__ void store_entry(Entry& e, const Cached& c) {
    const uint32_t* src[4] = {c.ymx, c.ypx, c.kt, c.z2};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        e.w[2 * q] = make_uint4(src[q][0], src[q][1], src[q][2], src[q][3]);
        e.w[2 * q + 1] = make_uint4(src[q][4], src[q][5], src[q][6], src[q][7]);
    }
}

// c = tab[digit], digit in [0, 16): every entry is read and masked in, so the access pattern is the same for all digits
__device__ __forceinline__ void select_entry(Cached& c, const Entry (&tab)[16], uint32_t digit) {
    uint32_t acc[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[k] = 0;
#pragma unroll 1
    for (int j = 0; j < 16; ++j) {             // j is the public loop counter: the same 16 addresses for every digit
        const uint32_t m = 0u - (uint32_t)(digit == (uint32_t)j);
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const uint4 x = tab[j].w[w];
            acc[4 * w + 0] |= x.x & m;
            acc[4 * w + 1] |= x.y & m;
            acc[4 * w + 2] |= x.z & m;
            acc[4 * w + 3] |= x.w & m;
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) c.ymx[k] = acc[k], c.ypx[k] = acc[8 + k], c.kt[k] = acc[16 + k], c.z2[k] = acc[24 + k];
}

// r = z^(p-2) = 1/z for z != 0 (Fermat), left to right over the public bits of p - 2
__device__ __forceinline__ void inverse(uint32_t (&r)[8], const uint32_t (&z)[8]) {
    fcopy(r, z);                // the top bit
#pragma unroll 1
    for (int i = kPm2Bits - 2; i >= 0; --i) {
        uint32_t t[8];
        fsqr(t, r);
        const uint32_t e[8] = P252_JJ_PM2;
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) word = (k == (i >> 5)) ? e[k] : word;
        if ((word >> (i & 31)) & 1u)
            fmul(r, t, z);
        else
            fcopy(r, t);
    }
}

// c = tab[digit] for a PUBLIC digit: one entry read at the digit's address (8 loads instead of 16 x 8 masked ones)
__device__ __forceinline__ void load_entry(Cached& c, const Entry& e) {
    uint32_t* dst[4] = {c.ymx, c.ypx, c.kt, c.z2};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 a = e.w[2 * q], b = e.w[2 * q + 1];
        dst[q][0] = a.x, dst[q][1] = a.y, dst[q][2] = a.z, dst[q][3] = a.w;
        dst[q][4] = b.x, dst[q][5] = b.y, dst[q][6] = b.z, dst[q][7] = b.w;
    }
}

// One window of the walk, most significant first: acc = 16 acc + tab[digit w of s], 3 x 7 + 8 + 7 products (8 with
// kWantT).  kPublic: the digit indexes the table directly (load_entry); otherwise every entry is read (select_entry).
template <bool kPublic, bool kWantT>
__device__ __forceinline__ void window_step(Ext& acc, Cached& c, const Entry (&tab)[16], const uint32_t (&s)[8], int w) {
    uint32_t limb = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) limb = (k == (w >> 3)) ? s[k] : limb;   // w is the public loop counter
    const uint32_t digit = (limb >> ((w & 7) * 4)) & 15u;
    Ext t;
    dbl<false>(t, acc);
    dbl<false>(acc, t);
    dbl<false>(t, acc);
    dbl<true>(acc, t);
    if (kPublic)
        load_entry(c, tab[digit]);
    else
        select_entry(c, tab, digit);
    add<kWantT>(t, acc, c);
    acc = t;
}

// tab[j] = [j] (u, v), j < 16, in cached form, for an on-curve (u, v) with u, v < p (Montgomery): T and 2d T of the input
// 2, entries 2..15 14 x (8 + 1) products.  acc and c are the build's temporaries.
__device__ __forceinline__ void var_table(Entry (&tab)[16], Ext& acc, Cached& c, const uint32_t (&u)[8],
                                          const uint32_t (&v)[8]) {
    // tab[0] = identity (0 : 1 : 1 : 0) cached = (1, 1, 0, 2)
    set_one(c.ymx);
    set_one(c.ypx);
#pragma unroll
    for (int k = 0; k < 8; ++k) c.kt[k] = 0;
    fr_add_mod(c.z2, c.ymx, c.ymx);
    store_entry(tab[0], c);
    // tab[1] = P = (u : v : 1 : uv)
    Cached pc;
    fcopy(acc.X, u);
    fcopy(acc.Y, v);
    set_one(acc.Z);
    fmul(acc.T, u, v);
    to_cached(pc, acc);
    store_entry(tab[1], pc);
    // tab[j] = tab[j - 1] + P
#pragma unroll 1
    for (int j = 2; j < 16; ++j) {
        Ext t;
        add<true>(t, acc, pc);
        acc = t;
        to_cached(c, acc);
        store_entry(tab[j], c);
    }
}

// acc = [s] P from the identity over the table of P (var_table), 63 window_steps; c is the windows' temporary.
template <bool kPublic, bool kLastT>
__device__ __forceinline__ void var_walk(Ext& acc, Cached& c, const Entry (&tab)[16], const uint32_t (&s)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) acc.X[k] = 0, acc.T[k] = 0;
    set_one(acc.Y);
    set_one(acc.Z);
#pragma unroll 1
    for (int w = kWindows - 1; w >= (kLastT ? 1 : 0); --w) window_step<kPublic, false>(acc, c, tab, s, w);
    if (kLastT) window_step<kPublic, true>(acc, c, tab, s, 0);
}

// acc = [s] (u, v) in extended coordinates for s < 2^252 (canonical words) and an on-curve (u, v) with u, v < p
// (Montgomery).  Fixed 4-bit window: the 16-entry table of (u, v) in thread-local memory, then 63 window_steps.
// kPublic: s is public (signature verification), so each window reads only its entry; a secret s (the key exchange)
// must not, and reads all 16.  kLastT: the last window also computes T, for a caller that adds another point to acc.
template <bool kPublic, bool kLastT>
__device__ __forceinline__ void scalar_mul_ext(Ext& acc, const uint32_t (&s)[8], const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    Entry tab[16];
    Cached c;
    var_table(tab, acc, c, u, v);
    var_walk<kPublic, kLastT>(acc, c, tab, s);
}

// (ou, ov) = [s] (u, v), affine, for a secret s: scalar_mul_ext with masked table reads, then one inversion.
__device__ __forceinline__ void scalar_mul(uint32_t (&ou)[8], uint32_t (&ov)[8], const uint32_t (&s)[8],
                                           const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    Ext acc;
    scalar_mul_ext<false, false>(acc, s, u, v);
    uint32_t zi[8];
    inverse(zi, acc.Z);
    fmul(ou, acc.X, zi);
    fmul(ov, acc.Y, zi);
}

// ---- fixed base: [s] B for one public base B shared by a batch (p252_fixed_base_batch) -------------------------------
// s < 2^252 is recoded into 64 signed digits e_w in [-8, 8), s = sum e_w 16^w, so [s] B = sum_w [e_w] (16^w B): one
// mixed addition per window from a precomputed table, no doublings.  The table holds, for w = 0..63 and j = 1..8, the
// affine point j 16^w B in "Niels" form (v - u, v + u, 2d u v), 6 x 16 bytes per entry, 48 KB in all; the digit's sign is
// applied by the negation -(u, v) = (-u, v), i.e. swap the first two coordinates and negate the third.
constexpr int kFbWindows = 64, kFbEntries = 8, kFbEntryWords = 6;   // uint4 per entry
constexpr int kFbTableWords = kFbWindows * kFbEntries * kFbEntryWords;
// Products per item: 63 mixed additions with T3 x 7, the last without x 6, the inversion, the affine conversion 2.
constexpr int kProductsPerFixedBase = (kFbWindows - 1) * 7 + 6 + (kPm2Bits - 1) + (kPm2Ones - 1) + 2;
static_assert(kProductsPerFixedBase == 866, "product count of DESIGN.md section 4");

struct Niels {                  // an affine addend (v - u, v + u, 2d u v), every coordinate < p
    uint32_t ymx[8], ypx[8], kt[8];
};

// r = p + q for an affine q (Z2 = 1): add() with D = 2 Z1 instead of a product, 7 products, 6 without T3
template <bool kWantT>
__device__ __forceinline__ void madd(Ext& r, const Ext& p, const Niels& q) {
    uint32_t a[8], b[8], c[8], d[8], e[8], f[8], g[8], h[8];
    fr_sub_mod(e, p.Y, p.X);
    fmul(a, e, q.ymx);          // A = (Y1 - X1)(v2 - u2)
    fr_add_mod(e, p.Y, p.X);
    fmul(b, e, q.ypx);          // B = (Y1 + X1)(v2 + u2)
    fmul(c, p.T, q.kt);         // C = T1 2d u2 v2
    fr_add_mod(d, p.Z, p.Z);    // D = 2 Z1
    fr_sub_mod(e, b, a);
    fr_sub_mod(f, d, c);
    fr_add_mod(g, d, c);
    fr_add_mod(h, b, a);
    fmul(r.X, e, f);
    fmul(r.Y, g, h);
    fmul(r.Z, f, g);
    if (kWantT) fmul(r.T, e, h);
}

// Signed 4-bit recoding, least significant window first: the low nibble of s plus the carry, in [0, 16] -> a digit in
// [-8, 8) and the next carry; s is shifted down by 4 (consumed).  Arithmetic only, no indexing by the window.  The last
// window (bits 252..255, zero for s < 2^252) takes the final carry, a digit in {0, 1}.
__device__ __forceinline__ int32_t recode_digit(uint32_t (&s)[8], uint32_t& carry) {
    const uint32_t x = (s[0] & 15u) + carry;
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = __funnelshift_r(s[k], s[k + 1], 4);
    s[7] >>= 4;
    carry = (x + 8u) >> 4;
    return (int32_t)x - (int32_t)(carry << 4);
}

// q = sign(e) (|e| 16^w B) from window w of the table: every entry of the window is read, at addresses fixed by w and the
// entry counter, and masked in (|e| = 0 selects the identity (1, 1, 0)); the sign is a masked swap and negation.
template <bool kLdg>
__device__ __forceinline__ void select_niels(Niels& q, const uint4* tab, int w, int32_t e) {
    const uint32_t neg = (uint32_t)e >> 31;
    const uint32_t mag = (uint32_t)((e ^ -(int32_t)neg) + (int32_t)neg);
    uint32_t acc[24], one[8];
    set_one(one);
    const uint32_t m0 = 0u - (uint32_t)(mag == 0);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = one[k] & m0, acc[8 + k] = one[k] & m0, acc[16 + k] = 0;
    const uint4* win = tab + w * (kFbEntries * kFbEntryWords);
#pragma unroll 1
    for (int j = 0; j < kFbEntries; ++j) {          // j is the public loop counter: the same 8 entries for every digit
        const uint32_t m = 0u - (uint32_t)(mag == (uint32_t)(j + 1));
#pragma unroll
        for (int q4 = 0; q4 < kFbEntryWords; ++q4) {
            const uint4 x = kLdg ? __ldg(win + j * kFbEntryWords + q4) : win[j * kFbEntryWords + q4];
            acc[4 * q4 + 0] |= x.x & m;
            acc[4 * q4 + 1] |= x.y & m;
            acc[4 * q4 + 2] |= x.z & m;
            acc[4 * q4 + 3] |= x.w & m;
        }
    }
    const uint32_t mn = 0u - neg;
    uint32_t nk[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t t = (acc[k] ^ acc[8 + k]) & mn;
        q.ymx[k] = acc[k] ^ t;
        q.ypx[k] = acc[8 + k] ^ t;
        q.kt[k] = acc[16 + k];
    }
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    fr_sub_mod(nk, zero, q.kt);
#pragma unroll
    for (int k = 0; k < 8; ++k) q.kt[k] = (q.kt[k] & ~mn) | (nk[k] & mn);
}

// t = [s] B in extended coordinates for s < 2^252 (canonical words) and the table of B (kFbTableWords uint4, built by
// fixed_base_entry).  kLdg: read the table through the read-only data path (a global table); otherwise plain loads (e.g.
// shared memory).  kLastT: the last window also computes T (64 x 7 products instead of 63 x 7 + 6), for a caller that
// adds another point to the result; without it t.T is not the result's.  t is also the windows' temporary, as it was in
// fixed_base_mul before the split, which keeps k_fixed_base's code unchanged.
// fixed_base_from: the same walk from acc (with T) instead of the identity, t = acc + [s] B; acc is the walk's
// accumulator and is overwritten.  kWin: the walk covers windows 0..kWin-1 only, for s < 2^(4 (kWin - 1)) (its last
// digit is the final carry); the default is the whole table.
template <bool kLdg, bool kLastT, int kWin = kFbWindows>
__device__ __forceinline__ void fixed_base_from(Ext& t, Ext& acc, const uint32_t (&s)[8], const uint4* tab) {
    static_assert(kWin >= 1 && kWin <= kFbWindows, "a walk over the table's windows");
    uint32_t d[8], carry = 0;
    fcopy(d, s);
    Niels q;
#pragma unroll 1
    for (int w = 0; w < kWin - 1; ++w) {
        select_niels<kLdg>(q, tab, w, recode_digit(d, carry));
        madd<true>(t, acc, q);
        acc = t;
    }
    select_niels<kLdg>(q, tab, kWin - 1, recode_digit(d, carry));
    madd<kLastT>(t, acc, q);
}

template <bool kLdg, bool kLastT>
__device__ __forceinline__ void fixed_base_ext(Ext& t, const uint32_t (&s)[8], const uint4* tab) {
    Ext acc;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc.X[k] = 0, acc.T[k] = 0;
    set_one(acc.Y);
    set_one(acc.Z);
    fixed_base_from<kLdg, kLastT>(t, acc, s, tab);
}

// (ou, ov) = [s] B, affine: fixed_base_ext without the last T, one inversion
template <bool kLdg>
__device__ __forceinline__ void fixed_base_mul(uint32_t (&ou)[8], uint32_t (&ov)[8], const uint32_t (&s)[8],
                                               const uint4* tab) {
    Ext t;
    fixed_base_ext<kLdg, false>(t, s, tab);
    uint32_t zi[8];
    inverse(zi, t.Z);
    fmul(ou, t.X, zi);
    fmul(ov, t.Y, zi);
}

// ---- stealth addresses: note_pk = [h] G + B (p252_stealth_address_batch / p252_stealth_owns_batch) -------------------
// h = hash([r] A) = hash([a] R) < 2^250 comes from the truncated digest; [h] G is fixed_base_ext with T in every window,
// then one mixed addition of B in Niels form.
//   owns:   B's Niels form is precomputed on the host; the result is compared projectively with note_pk, X == u Z and
//           Y == v Z (no inversion).
//   derive: B is read per item: on-curve check 4, Niels form 2 (u v, 2d u v); then the inversion and the affine
//           conversion.
constexpr int kProductsPerStealthOwns = kFbWindows * 7 + 6 + 2;
constexpr int kProductsPerStealthDerive = kFbWindows * 7 + 4 + 2 + 6 + (kPm2Bits - 1) + (kPm2Ones - 1) + 2;
static_assert(kProductsPerStealthOwns == 456, "product count of DESIGN.md section 4");
static_assert(kProductsPerStealthDerive == 879, "product count of DESIGN.md section 4");

// The Niels form (v - u, v + u, 2d u v) of an affine (u, v), u, v < p: 2 products
__device__ __forceinline__ void to_niels(Niels& q, const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    uint32_t uv[8], k[8];
    fr_sub_mod(q.ymx, v, u);
    fr_add_mod(q.ypx, v, u);
    fmul(uv, u, v);
    set_2d(k);
    fmul(q.kt, uv, k);
}

// ---- Schnorr signatures (p252_schnorr_sign_batch / p252_schnorr_verify_batch) ------------------------------------------
// c = challenge(R, m) < 2^250 comes from the truncated digest.
//   sign:   u = (r - c sk) mod r_J, no field product: two Montgomery products modulo r_J (order_mul) and one subtraction.
//   verify: [c] PK + [u] G == R.  PK is checked on the curve (4), [c] PK is scalar_mul_ext with public table reads and T
//           in the last window (table 2 + 14 x 9, 62 windows x 36, the last 37), then the fixed-base walk of [u] G starts
//           from it (63 x 7 + 6), and the result is compared projectively with R (2): no inversion.
constexpr int kOrderProductsPerSchnorrSign = 2;
constexpr int kProductsPerSchnorrVerify =
    4 + 2 + 14 * 9 + (kWindows - 1) * (3 * 7 + 8 + 7) + (3 * 7 + 8 + 8) + (kFbWindows - 1) * 7 + 6 + 2;
static_assert(kOrderProductsPerSchnorrSign == 2, "product count of DESIGN.md section 4");
static_assert(kProductsPerSchnorrVerify == 2850, "product count of DESIGN.md section 4");

// ---- note nullifiers (p252_nullifier_batch) ----------------------------------------------------------------------------
// h = hash([a] R) < 2^250 comes from the truncated digest.  note_sk = (h + b) mod r_J is order_add (no product),
// pk' = [note_sk] G' is fixed_base_mul, and the position's Montgomery image pos R mod p is one product by R^2 mod p
// (fr_from_canonical).
constexpr int kProductsPerNullifierKey = kProductsPerFixedBase + 1;
static_assert(kProductsPerNullifierKey == 867, "product count of DESIGN.md section 4");

// ---- double-key Schnorr signatures (p252_schnorr_{sign,verify}_double_batch, p252_note_sign_double_batch) ---------------
// c = challenge2(R, R', m) < 2^250 comes from the truncated digest of [R.u, R.v, R'.u, R'.v, m].
//   sign:      R = [r] G and R' = [r] G' are two fixed-base walks (k_fixed_base twice), u = (r - c sk) mod r_J the two
//              order products of the single-key signer.
//   note sign: in addition [a] R_note (k_dhke) for h, note_sk = (h + b) mod r_J (order_add, no product) and
//              pk' = [note_sk] G' (fixed_base_mul).
//   verify:    the single-key check twice, [c] PK + [u] G == R and [c] PK' + [u] G' == R'.
constexpr int kProductsPerSchnorrSignDouble = 2 * kProductsPerFixedBase;   // + kOrderProductsPerSchnorrSign modulo r_J
constexpr int kProductsPerNoteSignDouble = kProductsPerSchnorrSignDouble + kProductsPerDhke + kProductsPerFixedBase;
constexpr int kProductsPerSchnorrVerifyDouble = 2 * kProductsPerSchnorrVerify;
static_assert(kProductsPerSchnorrSignDouble == 1732, "product count of DESIGN.md section 4");
static_assert(kProductsPerNoteSignDouble == 5417, "product count of DESIGN.md section 4");
static_assert(kProductsPerSchnorrVerifyDouble == 5700, "product count of DESIGN.md section 4");

// ---- note values: C = [v] G + [blinder] G' (p252_value_commit_batch, p252_note_create_batch, p252_note_open_batch) ----
// [blinder] G' is the whole fixed-base walk of G' with T in every window (64 x 7); the walk of G continues from it for
// kValueWindows windows only: a u64 v recodes to 16 signed digits in [-8, 8) and a final carry digit in {0, 1} (window 16
// of the table).  The window count is public, so every item runs the same schedule.
//   commit / create: the last window without T (6), the inversion and the affine conversion.  create also writes the
//                    message rows Fr(v), Fr(blinder), one product by R^2 mod p each (fr_from_canonical).
//   open:            the decrypted rows leave Montgomery form by two reductions (fr_to_canonical, not counted as
//                    products), then the walk and the projective comparison with C, X == u Z and Y == v Z (2): no
//                    inversion.
constexpr int kValueWindows = 17;
constexpr int kProductsPerValueCommit = kFbWindows * 7 + (kValueWindows - 1) * 7 + 6 + (kPm2Bits - 1) + (kPm2Ones - 1) + 2;
constexpr int kProductsPerNoteCreateValue = kProductsPerValueCommit + 2;
constexpr int kProductsPerNoteOpenValue = kFbWindows * 7 + (kValueWindows - 1) * 7 + 6 + 2;
static_assert(kValueWindows == 64 / 4 + 1, "a u64 in signed 4-bit digits and the final carry");
static_assert(kProductsPerValueCommit == 985, "product count of DESIGN.md section 4");
static_assert(kProductsPerNoteCreateValue == 987, "product count of DESIGN.md section 4");
static_assert(kProductsPerNoteOpenValue == 568, "product count of DESIGN.md section 4");

// ---- multi-key wallet scans (p252_wallet_scan_batch) --------------------------------------------------------------------
// per key:        B = [b] G (fixed_base_mul) and its Niels form (2).
// per pair:       [a_j] R_i by k_dhke's schedule (its own inversion), then the stealth check against B_j (456); the hash
//                 of [a_j] R_i in between is one Hades permutation (365 Montgomery products, counted with the permutation).
// per note:       the validity of R (on-curve check, 4).
// per owned note: k_nullifier_key (867) and the opening check (568); the nullifier digest (one permutation) and the
//                 decryption at L = 2 (two) come on top.
constexpr int kProductsPerWalletKey = kProductsPerFixedBase + 2;
constexpr int kProductsPerWalletPair = kProductsPerDhke + kProductsPerStealthOwns;
constexpr int kProductsPerWalletSelect = 4;
constexpr int kProductsPerWalletOwned = kProductsPerNullifierKey + kProductsPerNoteOpenValue;
static_assert(kProductsPerWalletKey == 868, "product count of DESIGN.md section 4");
static_assert(kProductsPerWalletPair == 3275, "product count of DESIGN.md section 4");
static_assert(kProductsPerWalletOwned == 1435, "product count of DESIGN.md section 4");

// ---- JubJub ElGamal (p252_elgamal_{encrypt,decrypt}_batch, p252_note_sender_{encrypt,decrypt}_batch) --------------------
// encrypt (kPairs pairs under one PK): (c1_j, c2_j) = ([r_j] G, M_j + [r_j] PK).  PK's on-curve check 4 and its 16-entry
//   table 2 + 14 x 9 once; per pair M_j's on-curve check 4, [r_j] PK by the walk with T in the last window (62 x 36 + 37),
//   M_j's Niels form 2 and one mixed addition without T 6, [r_j] G by the fixed-base walk (63 x 7 + 6); then the 2 kPairs
//   outputs become affine with one shared inversion (batch_affine).
// decrypt: M = c2 - [sk] c1 = c2 + [sk] (-c1).  Both points' on-curve checks 8, the table of -c1 (negating u costs no
//   product), the walk with T in the last window, c2's Niels form and the mixed addition, one inversion, affine 2.
// note decrypt: note_sk = (h + b) mod r_J (order_add, no product) after k_dhke and the truncated digest; the four
//   ciphertext points' on-curve checks 16; ownership [note_sk] G (63 x 7 + 6) compared projectively with note_pk (2);
//   per pair the decrypt's table, walk and addition; one shared inversion for both outputs.
template <int kN>
constexpr int batch_affine_products() { return 3 * (kN - 1) + (kPm2Bits - 1) + (kPm2Ones - 1) + 2 * kN; }
constexpr int kProductsPerVarWalkT = 2 + 14 * 9 + (kWindows - 1) * (3 * 7 + 8 + 7) + (3 * 7 + 8 + 8);
constexpr int kProductsPerFbWalk = (kFbWindows - 1) * 7 + 6;
template <int kPairs>
constexpr int elgamal_enc_products() {
    return 4 + (2 + 14 * 9) + kPairs * (4 + (kProductsPerVarWalkT - 2 - 14 * 9) + 2 + 6 + kProductsPerFbWalk) +
           batch_affine_products<2 * kPairs>();
}
constexpr int kProductsPerElGamalEnc = elgamal_enc_products<1>();
constexpr int kProductsPerSenderEnc = elgamal_enc_products<2>();
constexpr int kProductsPerElGamalDec = 8 + kProductsPerVarWalkT + 2 + 6 + batch_affine_products<1>();
constexpr int kProductsPerSenderDec = 16 + kProductsPerFbWalk + 2 + 2 * (kProductsPerVarWalkT + 2 + 6) + batch_affine_products<2>();
static_assert(kProductsPerVarWalkT == 2397, "product count of DESIGN.md section 4");
static_assert(kProductsPerElGamalEnc == 3284, "product count of DESIGN.md section 4");
static_assert(kProductsPerSenderEnc == 6022, "product count of DESIGN.md section 4");
static_assert(kProductsPerElGamalDec == 2832, "product count of DESIGN.md section 4");
static_assert(kProductsPerSenderDec == 5699, "product count of DESIGN.md section 4");

struct Proj {                   // (X : Y : Z) of a result waiting for the shared inversion
    uint32_t X[8], Y[8], Z[8];
};
__device__ __forceinline__ void park(Proj& p, const Ext& e) {
    fcopy(p.X, e.X);
    fcopy(p.Y, e.Y);
    fcopy(p.Z, e.Z);
}

// Montgomery's trick: p[k] = (X_k / Z_k, Y_k / Z_k, -) for Z_k != 0, written back into X and Y, with one inversion:
// prefix products kN - 1, the inversion, two products per step back kN - 1, affine 2 kN.  The loops run over public
// counters: the same schedule for every item.
template <int kN>
__device__ __forceinline__ void batch_affine(Proj (&p)[kN]) {
    uint32_t pre[kN][8], inv[8], zi[8], t[8];
    fcopy(pre[0], p[0].Z);
#pragma unroll
    for (int k = 1; k < kN; ++k) fmul(pre[k], pre[k - 1], p[k].Z);
    inverse(inv, pre[kN - 1]);
#pragma unroll
    for (int k = kN - 1; k >= 0; --k) {
        if (k > 0) {
            fmul(zi, inv, pre[k - 1]);      // 1 / Z_k
            fmul(t, inv, p[k].Z);           // 1 / (Z_0 ... Z_{k-1})
            fcopy(inv, t);
        } else {
            fcopy(zi, inv);
        }
        fmul(t, p[k].X, zi);
        fcopy(p[k].X, t);
        fmul(t, p[k].Y, zi);
        fcopy(p[k].Y, t);
    }
}

// Arithmetic modulo r_J on 8 x 32-bit little-endian words, Montgomery form with R = 2^256.  Constants (immediates, as
// P252_JJ_ORDER): R^2 mod r_J and kOrderInv = -r_J^-1 mod 2^32.  Constant time: no branch and no address depends on an
// operand; each final correction is a masked subtraction or addition of r_J.
#define P252_JJ_ORDER_R2 {0x95e57731u, 0x67719aa4u, 0x9ce3fc26u, 0x51b0cef0u, 0xc026e9a5u, 0x69dab7fau, 0x8d127688u, 0x04f6547bu}
constexpr uint32_t kOrderInv = 0xef788ef9u;

// r = a b / 2^256 mod r_J for a, b < r_J (word-serial Montgomery, CIOS).  After row i the accumulator is < a + r_J <
// 2 r_J < 2^253, so it fits 8 words between rows and one masked subtraction of r_J makes it < r_J.
__device__ __forceinline__ void order_mont(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t n[8] = P252_JJ_ORDER;
    uint32_t t[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {                  // t += a b_i
            c += (uint64_t)a[j] * b[i] + t[j];
            t[j] = (uint32_t)c;
            c >>= 32;
        }
        const uint32_t hi = (uint32_t)c;
        const uint32_t m = t[0] * kOrderInv;          // t + m r_J = 0 mod 2^32
        c = ((uint64_t)m * n[0] + t[0]) >> 32;
#pragma unroll
        for (int j = 1; j < 8; ++j) {                  // t = (t + m r_J) / 2^32
            c += (uint64_t)m * n[j] + t[j];
            t[j - 1] = (uint32_t)c;
            c >>= 32;
        }
        t[7] = (uint32_t)(c + hi);                      // < 2^32 by the bound above
    }
    uint32_t d[8], borrow = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t x = (uint64_t)t[k] - n[k] - borrow;
        d[k] = (uint32_t)x;
        borrow = (uint32_t)(x >> 63);
    }
    const uint32_t keep = 0u - borrow;                  // t < r_J: keep t, otherwise t - r_J
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = (t[k] & keep) | (d[k] & ~keep);
}

// r = a b mod r_J for a, b < r_J: (a b / 2^256) (2^512 mod r_J) / 2^256, two Montgomery products
__device__ __forceinline__ void order_mul(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t r2[8] = P252_JJ_ORDER_R2;
    uint32_t x[8];
    order_mont(x, a, b);
    order_mont(r, x, r2);
}

// r = a - b mod r_J for a, b < r_J: the borrow of a - b selects a masked addition of r_J
__device__ __forceinline__ void order_sub(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t n[8] = P252_JJ_ORDER;
    uint32_t borrow = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t x = (uint64_t)a[k] - b[k] - borrow;
        r[k] = (uint32_t)x;
        borrow = (uint32_t)(x >> 63);
    }
    const uint32_t m = 0u - borrow;
    uint32_t carry = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t y = (uint64_t)r[k] + (n[k] & m) + carry;
        r[k] = (uint32_t)y;
        carry = (uint32_t)(y >> 32);
    }
}

// Table entry (w, j), j in 1..8, of the base (u, v) (on the curve, u, v < p): j 16^w (u, v) by 4w doublings and j - 1
// additions, then affine and Niels form.  The base is public, so these loops branch on w and j.
__device__ __forceinline__ void fixed_base_entry(uint4* out, const uint32_t (&u)[8], const uint32_t (&v)[8], int w, int j) {
    Ext p, t;
    fcopy(p.X, u);
    fcopy(p.Y, v);
    set_one(p.Z);
    fmul(p.T, u, v);
    for (int i = 0; i < 4 * w; ++i) {
        dbl<true>(t, p);
        p = t;
    }
    Cached c;
    to_cached(c, p);
    Ext q = p;
    for (int i = 1; i < j; ++i) {
        add<true>(t, q, c);
        q = t;
    }
    uint32_t zi[8], au[8], av[8], uv[8], k[8];
    inverse(zi, q.Z);
    fmul(au, q.X, zi);
    fmul(av, q.Y, zi);
    Niels n;
    fr_sub_mod(n.ymx, av, au);
    fr_add_mod(n.ypx, av, au);
    fmul(uv, au, av);
    set_2d(k);
    fmul(n.kt, uv, k);
    const uint32_t* src[3] = {n.ymx, n.ypx, n.kt};
#pragma unroll
    for (int q3 = 0; q3 < 3; ++q3) {
        out[2 * q3] = make_uint4(src[q3][0], src[q3][1], src[q3][2], src[q3][3]);
        out[2 * q3 + 1] = make_uint4(src[q3][4], src[q3][5], src[q3][6], src[q3][7]);
    }
}

// ---- point compression: JubJubAffine::to_bytes / from_bytes (p252_points_to_bytes / p252_points_from_bytes) ------------
// Encoding: the 32 little-endian bytes of canonical v, bit 255 = the low bit of canonical u (v < p < 2^255 leaves it free).
// Decoding solves the curve equation for u: u^2 = (v^2 - 1) / (1 + d v^2).  The denominator is never 0 (d is a
// non-square, -1 a square), so the root is RFC 9380 Appendix F.2.1.1 sqrt_ratio(num, den): no inversion, and a trip count
// fixed by p alone, so every lane of a warp runs the same instructions.  With p - 1 = 2^c1 t, t odd, c1 = 32 and Z = 5 (a
// non-residue mod p), its constants are c3 = (t - 1) / 2 (222 bits, 132 set; canonical words), c6 = Z^t and
// c7 = Z^((t + 1) / 2) (Montgomery images).  Immediates, as P252_JJ_PM2.
#define P252_JJ_SQRT_C3 {0x7fffffffu, 0x7fff2dffu, 0xa9ded201u, 0x04d0ec02u, 0x199cec04u, 0x94cebea4u, 0x39f6d3a9u, 0x00000000u}
#define P252_JJ_SQRT_C6 {0x0c17f47cu, 0x9cab6d5cu, 0xfd4b71e5u, 0x1ce1e93du, 0x471dd505u, 0x0d6db230u, 0x743a3b6au, 0x3f0ee990u}
#define P252_JJ_SQRT_C7 {0xbb7b07a1u, 0xba8e19e4u, 0x92112747u, 0x0dc42383u, 0x26b941a1u, 0xdfd3d081u, 0x7a45cec5u, 0x6bb1a261u}
constexpr int kSqrtC1 = 32, kSqrtC3Bits = 222, kSqrtC3Ones = 132;

// Products of sqrt_ratio, step by step (RFC numbering): 2. den^(2^32 - 1) by the chain 2^(2k) - 1 = (2^k - 1) 2^k +
// (2^k - 1), 31 squarings + 5 products; 3.-5. 3; 6. the exponent c3, (bits - 1) squarings + (ones - 1) products; 7.-10. 4;
// 11. 31 squarings; 13.-14. 2; the loop k = 32..2, (k - 2) squarings + 3 products per round.
constexpr int kProductsPerSqrtRatio = (31 + 5) + 3 + (kSqrtC3Bits - 1) + (kSqrtC3Ones - 1) + 4 + (kSqrtC1 - 1) + 2 +
                                      (kSqrtC1 - 2) * (kSqrtC1 - 1) / 2 + 3 * (kSqrtC1 - 1);
// Decompression: v into Montgomery form 1, v^2 and d v^2 2, sqrt_ratio; the sign needs one canonical conversion (a
// reduction, no product).  Compression: the on-curve check 4 and two canonical conversions.
constexpr int kProductsPerDecompress = 1 + 2 + kProductsPerSqrtRatio;
constexpr int kProductsPerCompress = 4;
static_assert(kProductsPerSqrtRatio == 986, "product count of DESIGN.md section 4");
static_assert(kProductsPerDecompress == 989, "product count of DESIGN.md section 4");
static_assert(kProductsPerCompress == 4, "product count of DESIGN.md section 4");

// r = a^(2^k): k squarings (k public)
__device__ __forceinline__ void fsqr_n(uint32_t (&r)[8], const uint32_t (&a)[8], int k) {
    fcopy(r, a);
#pragma unroll 1
    for (int i = 0; i < k; ++i) {
        uint32_t t[8];
        fsqr(t, r);
        fcopy(r, t);
    }
}

// r = c ? a : b, masked
__device__ __forceinline__ void fsel(uint32_t (&r)[8], bool c, const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t m = 0u - (uint32_t)c;
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = (a[k] & m) | (b[k] & ~m);
}

// Returns whether num / den is a square; y = sqrt(num / den) if it is, sqrt(Z num / den) otherwise.  num, den < p,
// den != 0.  The RFC's is_square is false for num = 0 (tv4 = 0 never powers to 1); num = 0 is a square here, and y is 0
// on both paths.
__device__ __forceinline__ bool sqrt_ratio(uint32_t (&y)[8], const uint32_t (&num)[8], const uint32_t (&den)[8]) {
    uint32_t tv1[8] = P252_JJ_SQRT_C6, tv2[8], tv3[8], tv4[8], tv5[8], t[8], one[8];
    set_one(one);
    // 2. tv2 = den^(2^32 - 1)
    fcopy(tv2, den);
#pragma unroll 1
    for (int k = 1; k < kSqrtC1; k *= 2) {
        fsqr_n(t, tv2, k);
        fmul(tv3, t, tv2);
        fcopy(tv2, tv3);
    }
    fsqr(t, tv2);                   // 3. tv3 = tv2^2
    fmul(tv3, t, den);              // 4. tv3 = tv3 den
    fmul(t, num, tv3);              // 5. tv5 = num tv3
    fcopy(tv5, t);                  // 6. tv5 = tv5^c3, left to right over the public bits of c3
#pragma unroll 1
    for (int i = kSqrtC3Bits - 2; i >= 0; --i) {
        uint32_t s[8];
        fsqr(s, tv5);
        const uint32_t e[8] = P252_JJ_SQRT_C3;
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) word = (k == (i >> 5)) ? e[k] : word;
        if ((word >> (i & 31)) & 1u)
            fmul(tv5, s, t);
        else
            fcopy(tv5, s);
    }
    fmul(t, tv5, tv2);              // 7. tv5 = tv5 tv2
    fmul(tv2, t, den);              // 8. tv2 = tv5 den
    fmul(tv3, t, num);              // 9. tv3 = tv5 num
    fmul(tv4, tv3, tv2);            // 10. tv4 = tv3 tv2
    fsqr_n(tv5, tv4, kSqrtC1 - 1);  // 11. tv5 = tv4^(2^31)
    const bool is_qr = feq(tv5, one);                       // 12.
    const uint32_t c7[8] = P252_JJ_SQRT_C7;
    fmul(tv2, tv3, c7);             // 13. tv2 = tv3 c7
    fmul(tv5, tv4, tv1);            // 14. tv5 = tv4 tv1
    fsel(tv3, is_qr, tv3, tv2);     // 15.
    fsel(tv4, is_qr, tv4, tv5);     // 16.
#pragma unroll 1
    for (int k = kSqrtC1; k >= 2; --k) {                    // 17.
        fsqr_n(tv5, tv4, k - 2);    // 18.-20. tv5 = tv4^(2^(k - 2))
        const bool e1 = feq(tv5, one);                      // 21.
        fmul(tv2, tv3, tv1);        // 22.
        fsqr(t, tv1);               // 23.
        fcopy(tv1, t);
        fmul(tv5, tv4, tv1);        // 24.
        fsel(tv3, e1, tv3, tv2);    // 25.
        fsel(tv4, e1, tv4, tv5);    // 26.
    }
    fcopy(y, tv3);
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    return is_qr | feq(num, zero);
}

// (u, v) = JubJubAffine::from_bytes(b) (Montgomery), b the 8 little-endian words of the encoding.  Returns validity: the
// 255-bit v < p and u^2 a square.  kProductsPerDecompress products.  An invalid encoding runs the same schedule on v = 0
// and its (u, v) is not a point; the caller discards it.
__device__ __forceinline__ bool decompress(uint32_t (&u)[8], uint32_t (&v)[8], const uint32_t (&b)[8]) {
    uint32_t c[8], vv[8], dvv[8], num[8], den[8], r[8], one[8], k[8];
    const uint32_t sign = b[7] >> 31;
    fcopy(c, b);
    c[7] &= 0x7fffffffu;
    const bool canon = fr_is_canonical(c);
    const uint32_t mc = 0u - (uint32_t)canon;
#pragma unroll
    for (int q = 0; q < 8; ++q) c[q] &= mc;
    fr_from_canonical(v, c);
    fsqr(vv, v);
    set_d(k);
    fmul(dvv, vv, k);
    set_one(one);
    fr_sub_mod(num, vv, one);       // v^2 - 1
    fr_add_mod(den, dvv, one);      // 1 + d v^2
    const bool square = sqrt_ratio(r, num, den);
    uint32_t rc[8], nr[8];
    fr_to_canonical(rc, r);
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    fr_sub_mod(nr, zero, r);        // p - r (0 for r = 0: a set sign bit with u = 0 decodes to the same point)
    fsel(u, (rc[0] & 1u) == sign, r, nr);
    return canon & square;
}

// ---- multi-scalar multiplication: sum [s_i] P_i by buckets (p252_jubjub_msm / p252_schnorr_verify_all) -----------------
// VARIABLE TIME: every scalar is public, and its digits become bucket indexes (addresses) and branch conditions.
// c-bit signed windows, least significant first: window w takes x = bits [c w, c w + c) of s plus the carry, x in
// [0, 2^c]; the digit is x - 2^c carry' with carry' = (x + 2^(c-1)) >> c, in [-2^(c-1), 2^(c-1)).  With W(c) = ceil(253 / c)
// windows the top one holds at most c - 1 bits of s < 2^252, so its x <= 2^(c-1) is the digit itself and no carry is left.
// Digit e != 0 of window w adds sign(e) P to bucket (w, |e| - 1); bucket sums B_j (j = |e|) of a window reduce to
// sum_j j B_j by running sums, and the windows combine as sum_w 2^(c w) S_w (Horner, c doublings per window).
// Products: a row's on-curve check 4 and Niels form 2; a nonzero digit one mixed addition with T 7; a carried partial
// sum (pieces of one bucket split across threads) and each running-sum step one cached addition 1 + 8.
constexpr int kMsmMinBits = 4, kMsmMaxBits = 13;
__host__ __device__ constexpr int msm_windows(int c) { return (253 + c - 1) / c; }
constexpr int kProductsPerMsmRow = 4 + 2;
constexpr int kProductsPerMsmDigit = 7;
constexpr int kProductsPerMsmCarry = 1 + 8;
constexpr int kProductsPerMsmBucket = 2 * (1 + 8);
static_assert(kProductsPerMsmRow == 6 && kProductsPerMsmDigit == 7, "product counts of DESIGN.md section 4");
static_assert(kProductsPerMsmCarry == 9 && kProductsPerMsmBucket == 18, "product counts of DESIGN.md section 4");
static_assert(msm_windows(kMsmMaxBits) == 20 && msm_windows(kMsmMinBits) == 64, "window counts of DESIGN.md section 4");

// The next digit of s (consumed c bits at a time, c in [kMsmMinBits, kMsmMaxBits]); top: the last window, no carry out
__device__ __forceinline__ int32_t recode_window(uint32_t (&s)[8], uint32_t& carry, int c, bool top) {
    const uint32_t x = (s[0] & ((1u << c) - 1u)) + carry;
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = __funnelshift_r(s[k], s[k + 1], c);
    s[7] >>= c;
    if (top) {
        carry = 0;
        return (int32_t)x;
    }
    carry = (x + (1u << (c - 1))) >> c;
    return (int32_t)x - (int32_t)(carry << c);
}

// r = a + b mod r_J for a, b < r_J (the sum < 2^253 fits 8 words; one masked subtraction)
__device__ __forceinline__ void order_add(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
    const uint32_t n[8] = P252_JJ_ORDER;
    uint32_t s[8], d[8], carry = 0, borrow = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t x = (uint64_t)a[k] + b[k] + carry;
        s[k] = (uint32_t)x;
        carry = (uint32_t)(x >> 32);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t x = (uint64_t)s[k] - n[k] - borrow;
        d[k] = (uint32_t)x;
        borrow = (uint32_t)(x >> 63);
    }
    const uint32_t keep = 0u - borrow;                  // s < r_J
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = (s[k] & keep) | (d[k] & ~keep);
}

__device__ __forceinline__ void set_identity(Ext& p) {
#pragma unroll
    for (int k = 0; k < 8; ++k) p.X[k] = 0, p.T[k] = 0;
    set_one(p.Y);
    set_one(p.Z);
}

// r = p + q for two extended points (to_cached + add): 9 products
__device__ __forceinline__ void add_ext(Ext& r, const Ext& p, const Ext& q) {
    Cached c;
    to_cached(c, q);
    add<true>(r, p, c);
}

// An extended point as 8 x 16 bytes (X, Y, Z, T)
__device__ __forceinline__ void store_ext(uint4* d, const Ext& p) {
    const uint32_t* src[4] = {p.X, p.Y, p.Z, p.T};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        d[2 * q] = make_uint4(src[q][0], src[q][1], src[q][2], src[q][3]);
        d[2 * q + 1] = make_uint4(src[q][4], src[q][5], src[q][6], src[q][7]);
    }
}
__device__ __forceinline__ void load_ext(Ext& p, const uint4* s) {
    uint32_t* dst[4] = {p.X, p.Y, p.Z, p.T};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 a = s[2 * q], b = s[2 * q + 1];
        dst[q][0] = a.x, dst[q][1] = a.y, dst[q][2] = a.z, dst[q][3] = a.w;
        dst[q][4] = b.x, dst[q][5] = b.y, dst[q][6] = b.z, dst[q][7] = b.w;
    }
}

// r = [k] p for a small public k (left to right over its bits)
__device__ __forceinline__ void mul_small(Ext& r, const Ext& p, uint32_t k) {
    set_identity(r);
    if (k == 0) return;
    Cached c;
    to_cached(c, p);
    for (int b = 31 - __clz(k); b >= 0; --b) {
        Ext t;
        dbl<true>(t, r);
        if ((k >> b) & 1u)
            add<true>(r, t, c);
        else
            r = t;
    }
}

// b = JubJubAffine::to_bytes(u, v) as 8 little-endian words, for u, v < p (Montgomery) on the curve: canonical v with the
// low bit of canonical u in bit 255
__device__ __forceinline__ void compress(uint32_t (&b)[8], const uint32_t (&u)[8], const uint32_t (&v)[8]) {
    uint32_t uc[8];
    fr_to_canonical(uc, u);
    fr_to_canonical(b, v);
    b[7] |= uc[0] << 31;
}

}  // namespace jj
}  // namespace p252
