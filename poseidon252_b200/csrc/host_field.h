// Host-side helpers of the library: BLAKE2b-512 (RFC 7693) and the little bit of Fr arithmetic
// needed to derive sponge tags once per batch (BlsScalar::hash_to_scalar ->
// from_bytes_wide, called at src/hades/permutation/scalar.rs:29-31).
// This is per-batch bookkeeping, not a data path: no permutation is ever computed on the host.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace p252 {
namespace host {

// ---- BLAKE2b, unkeyed, 64-byte digest -----------------------------------------------------------
struct Blake2b {
    uint64_t h[8];
    uint64_t t[2];
    uint8_t buf[128];
    size_t buflen;

    static inline uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
    static inline uint64_t load64(const uint8_t* p) {
        uint64_t v = 0;
        for (int i = 7; i >= 0; --i) v = (v << 8) | p[i];
        return v;
    }

    void init() {
        static const uint64_t iv[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL,
                                       0xa54ff53a5f1d36f1ULL, 0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL,
                                       0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
        memcpy(h, iv, sizeof iv);
        h[0] ^= 0x01010000ULL ^ 64;   // digest length 64, no key, fanout = depth = 1
        t[0] = t[1] = 0;
        buflen = 0;
        memset(buf, 0, sizeof buf);
    }

    void compress(const uint8_t* block, bool last) {
        static const uint64_t iv[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL,
                                       0xa54ff53a5f1d36f1ULL, 0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL,
                                       0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
        static const uint8_t sigma[12][16] = {
            {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
            {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
            {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
            {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
            {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
            {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
        uint64_t m[16], v[16];
        for (int i = 0; i < 16; ++i) m[i] = load64(block + 8 * i);
        for (int i = 0; i < 8; ++i) v[i] = h[i], v[i + 8] = iv[i];
        v[12] ^= t[0];
        v[13] ^= t[1];
        if (last) v[14] = ~v[14];
#define P252_G(a, b, c, d, x, y)      \
    v[a] = v[a] + v[b] + (x);         \
    v[d] = rotr(v[d] ^ v[a], 32);     \
    v[c] = v[c] + v[d];               \
    v[b] = rotr(v[b] ^ v[c], 24);     \
    v[a] = v[a] + v[b] + (y);         \
    v[d] = rotr(v[d] ^ v[a], 16);     \
    v[c] = v[c] + v[d];               \
    v[b] = rotr(v[b] ^ v[c], 63);
        for (int r = 0; r < 12; ++r) {
            const uint8_t* s = sigma[r];
            P252_G(0, 4, 8, 12, m[s[0]], m[s[1]])
            P252_G(1, 5, 9, 13, m[s[2]], m[s[3]])
            P252_G(2, 6, 10, 14, m[s[4]], m[s[5]])
            P252_G(3, 7, 11, 15, m[s[6]], m[s[7]])
            P252_G(0, 5, 10, 15, m[s[8]], m[s[9]])
            P252_G(1, 6, 11, 12, m[s[10]], m[s[11]])
            P252_G(2, 7, 8, 13, m[s[12]], m[s[13]])
            P252_G(3, 4, 9, 14, m[s[14]], m[s[15]])
        }
#undef P252_G
        for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
    }

    void update(const uint8_t* in, size_t len) {
        while (len > 0) {
            if (buflen == 128) {
                t[0] += 128;
                if (t[0] < 128) t[1]++;
                compress(buf, false);
                buflen = 0;
            }
            size_t take = 128 - buflen;
            if (take > len) take = len;
            memcpy(buf + buflen, in, take);
            buflen += take;
            in += take;
            len -= take;
        }
    }

    void final(uint8_t out[64]) {
        t[0] += buflen;
        if (t[0] < buflen) t[1]++;
        memset(buf + buflen, 0, 128 - buflen);
        compress(buf, true);
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 8; ++j) out[8 * i + j] = (uint8_t)(h[i] >> (8 * j));
    }
};

inline void blake2b512(const uint8_t* in, size_t len, uint8_t out[64]) {
    Blake2b b;
    b.init();
    b.update(in, len);
    b.final(out);
}

// ---- minimal Fr (4 x u64 Montgomery) ------------------------------------------------------------
typedef unsigned __int128 u128;
static const uint64_t kMod[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL,
                                 0x73eda753299d7d48ULL};
static const uint64_t kInv = 0xfffffffeffffffffULL;
static const uint64_t kR2[4] = {0xc999e990f3f29c6dULL, 0x2b6cedcb87925c23ULL, 0x05d314967254398fULL,
                                0x0748d9d99f59ff11ULL};
static const uint64_t kR3[4] = {0xc62c1807439b73afULL, 0x1b3e0d188cf06990ULL, 0x73d13c71c7b5f418ULL,
                                0x6e2a5bb9c8db33e9ULL};

inline void cond_sub(uint64_t a[4]) {
    uint64_t t[4];
    u128 b = 0;
    for (int i = 0; i < 4; ++i) {
        u128 d = (u128)a[i] - kMod[i] - (uint64_t)b;
        t[i] = (uint64_t)d;
        b = (d >> 64) & 1;
    }
    if (!b) memcpy(a, t, sizeof t);
}

// r = a*b/2^256 mod p, a < 2^256, b < p
inline void mont_mul(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        u128 c = 0;
        for (int j = 0; j < 4; ++j) {
            c += (u128)a[j] * b[i] + t[j];
            t[j] = (uint64_t)c;
            c >>= 64;
        }
        c += t[4];
        t[4] = (uint64_t)c;
        t[5] = (uint64_t)(c >> 64);
        const uint64_t m = t[0] * kInv;
        c = ((u128)m * kMod[0] + t[0]) >> 64;
        for (int j = 1; j < 4; ++j) {
            c += (u128)m * kMod[j] + t[j];
            t[j - 1] = (uint64_t)c;
            c >>= 64;
        }
        c += t[4];
        t[3] = (uint64_t)c;
        t[4] = t[5] + (uint64_t)(c >> 64);
    }
    // a < 2^256, b < p  =>  t < 2p (t[4] may be 1 only if t >= 2^256 > 2p: impossible)
    uint64_t out[4] = {t[0], t[1], t[2], t[3]};
    cond_sub(out);
    memcpy(r, out, sizeof out);
}

inline void add_mod(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
    u128 c = 0;
    uint64_t t[4];
    for (int i = 0; i < 4; ++i) {
        c += (u128)a[i] + b[i];
        t[i] = (uint64_t)c;
        c >>= 64;
    }
    cond_sub(t);
    memcpy(r, t, sizeof t);
}

// r = a - b mod p for a, b < p
inline void sub_mod(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
    u128 bw = 0;
    uint64_t t[4];
    for (int i = 0; i < 4; ++i) {
        u128 d = (u128)a[i] - b[i] - (uint64_t)bw;
        t[i] = (uint64_t)d;
        bw = (d >> 64) & 1;
    }
    if (bw) {
        u128 c = 0;
        for (int i = 0; i < 4; ++i) {
            c += (u128)t[i] + kMod[i];
            t[i] = (uint64_t)c;
            c >>= 64;
        }
    }
    memcpy(r, t, sizeof t);
}

// a < p
inline bool is_canonical(const uint64_t a[4]) {
    u128 bw = 0;
    for (int i = 0; i < 4; ++i) bw = (((u128)a[i] - kMod[i] - (uint64_t)bw) >> 64) & 1;
    return bw != 0;
}

// d = -10240/10241 of JubJub, Montgomery
static const uint64_t kD[4] = {0x2a522455b974f6b0ULL, 0xfc6cc9ef0d9acab3ULL, 0x7a08fb94c27628d1ULL, 0x57f8f6a8fe0e262eULL};

// (u, v) (Montgomery limbs) is a JubJub point: u, v < p and -u^2 + v^2 == 1 + d u^2 v^2, d = -10240/10241
inline bool jubjub_on_curve(const uint64_t u[4], const uint64_t v[4]) {
    static const uint64_t kOne[4] = {0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL,
                                     0x1824b159acc5056fULL};
    if (!is_canonical(u) || !is_canonical(v)) return false;
    uint64_t uu[4], vv[4], lhs[4], w[4], rhs[4];
    mont_mul(uu, u, u);
    mont_mul(vv, v, v);
    sub_mod(lhs, vv, uu);
    mont_mul(w, uu, vv);
    mont_mul(rhs, w, kD);
    add_mod(rhs, rhs, kOne);
    return memcmp(lhs, rhs, sizeof lhs) == 0;
}

// The Niels form (v - u, v + u, 2d u v) of a JubJub point (u, v < p, Montgomery limbs): the addend of the device's
// mixed addition (jubjub_device.cuh, madd), as out[0..4), out[4..8), out[8..12)
inline void jubjub_niels(uint64_t out[12], const uint64_t u[4], const uint64_t v[4]) {
    uint64_t d2[4], uv[4];
    add_mod(d2, kD, kD);
    sub_mod(out, v, u);
    add_mod(out + 4, v, u);
    mont_mul(uv, u, v);
    mont_mul(out + 8, uv, d2);
}

// BlsScalar::from_bytes_wide: 64 LE bytes -> (lo + hi*2^256) mod p, Montgomery form
inline void from_bytes_wide(uint64_t r[4], const uint8_t b[64]) {
    uint64_t lo[4], hi[4], a[4], c[4];
    for (int i = 0; i < 4; ++i) {
        lo[i] = Blake2b::load64(b + 8 * i);
        hi[i] = Blake2b::load64(b + 32 + 8 * i);
    }
    mont_mul(a, lo, kR2);   // lo * R
    mont_mul(c, hi, kR3);   // hi * 2^256 * R
    add_mod(r, a, c);
}

}  // namespace host
}  // namespace p252
