// Batch kernels of the Poseidon/Hades engine (sm_90a).  One sponge state per thread, state in
// registers; global memory is touched only by 128-bit accesses: warp-cooperative, fully coalesced
// tiles staged through shared memory for the hash/permute kernels (each LDG.128/STG.128 of a warp
// covers whole 128-byte item chunks), per-thread 2 x 128-bit per scalar for encrypt/decrypt.
//
// Sponge schedule = dusk-safe 0.3 `Sponge` as driven by the reference:
//   Hash::finalize   src/hash.rs:128-155      -> k_sponge_digest (k_sponge_digest_varlen: inputs of any lengths;
//     k_mixed_keys, k_sponge_digest_mixed: items of any domains, lengths and truncation, tags derived on the device)
//   encrypt/decrypt  src/encryption.rs:62-95  -> k_crypt (k_crypt_varlen: messages of any lengths)
//   Safe::permute    src/hades/permutation/scalar.rs:25-27 -> k_permute
//   dhke             src/encryption.rs:11-43  -> k_dhke (JubJub scalar multiplication, jubjub_device.cuh)
//   stealth addresses (note_pk = [hash(shared)] G + B) -> k_stealth
//   Schnorr signatures (u = r - c sk, [u] G + [c] PK == R) -> k_schnorr_pack, k_schnorr_sign, k_schnorr_verify
//   note nullifiers (pk' = [(h + b) mod r_J] G', the digest rows [pk'.u, pk'.v, pos]) -> k_nullifier_key
//   double-key Schnorr signatures over G and G' (SignatureDouble, note signing) -> k_schnorr_pack_double,
//     k_schnorr_sign_double<Note>, k_schnorr_verify_double
//   all-or-nothing double-key verification (one MSM over G and G') -> k_msmv_prep_double, k_msmv_final_double
//   multi-key wallet scans (owner, then nullifier and opening of owned notes) -> k_wallet_keys, k_wallet_dhke,
//     k_wallet_match, k_wallet_select, k_wallet_scatter
//   JubJubAffine::from_bytes / to_bytes (point compression) -> k_points_from_bytes, k_points_to_bytes
//   BlsScalar::hash_to_scalar (BLAKE2b-512 of byte strings, then from_bytes_wide) -> k_hash_to_scalar_keys,
//     k_hash_to_scalar; BlsScalar::from_bytes_wide alone -> k_from_bytes_wide
// capacity = state[0] = tag, rate = state[1..5]; absorb adds into state[pos+1] and permutes when
// pos == 4; any absorb forces a permutation before the next squeeze.
#include "kernels.h"

#include <cstdlib>

#include "hades_device.cuh"
#include "jubjub_device.cuh"

namespace p252 {

#ifndef P252_MINBLOCKS
#define P252_MINBLOCKS 5      // resident 128-thread blocks per SM the register allocation is held to (<= 102 regs)
#endif
#ifndef P252_THREADS
#define P252_THREADS 128
#endif
constexpr int kThreads = P252_THREADS;
constexpr int kMinBlocks = P252_MINBLOCKS;
constexpr int kWarps = kThreads / 32;

#if P252_CONST_SMEM
#define P252_STAGE_TABLES                                             \
    __shared__ __align__(128) uint32_t s_round_tab[P252_TAB_WORDS];   \
    __shared__ __align__(8) uint64_t s_tab_bar;                       \
    const uint32_t* tab = stage_round_tables(s_round_tab, &s_tab_bar);
#else
#define P252_STAGE_TABLES
#endif

struct FrArg {
    uint32_t l[8];
};

__device__ __forceinline__ uint4 ldg128(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ---- warp-cooperative 128-byte-chunk gather / scatter -------------------------------------------
// 32 items, one per lane; item k's chunk lives at base + k*stride (stride multiple of 32 B).
// Global side: lane l moves 16 B; 8 consecutive lanes cover one item's 128-byte chunk, so every
// LDG.128 / STG.128 of the warp touches 4 complete 128-byte segments.  Shared side: XOR swizzle on
// the 16-byte column keeps both the row-wise (global side) and the item-per-lane (register side)
// accesses bank-conflict free.
//
// tile_row: the register side of a gather, the lane's own item (row `lane` of the tile) into four scalars v[0..3].
__device__ __forceinline__ void tile_row(uint4 (*st)[8], int lane, uint32_t (*v)[8]) {
#pragma unroll
    for (int p = 0; p < 8; ++p) {
        const uint4 x = st[lane][p ^ (lane & 7)];
        v[p >> 1][(p & 1) * 4 + 0] = x.x;
        v[p >> 1][(p & 1) * 4 + 1] = x.y;
        v[p >> 1][(p & 1) * 4 + 2] = x.z;
        v[p >> 1][(p & 1) * 4 + 3] = x.w;
    }
}

__device__ __forceinline__ void warp_gather(uint4 (*st)[8], const uint8_t* base, size_t stride, int nitems,
                                            int nscal, int lane, uint32_t (&v)[4][8]) {
    const int part = lane & 7;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int item = r * 4 + (lane >> 3);
        uint4 x = make_uint4(0, 0, 0, 0);
        if (item < nitems && (part >> 1) < nscal) x = ldg128(base + (size_t)item * stride + part * 16);
        st[item][part ^ (item & 7)] = x;
    }
    __syncwarp();
    tile_row(st, lane, v);
    __syncwarp();
}

__device__ __forceinline__ void warp_scatter(uint4 (*st)[8], uint8_t* base, size_t stride, int nitems, int nscal,
                                             int lane, const uint32_t (&v)[4][8]) {
#pragma unroll
    for (int p = 0; p < 8; ++p)
        st[lane][p ^ (lane & 7)] = make_uint4(v[p >> 1][(p & 1) * 4 + 0], v[p >> 1][(p & 1) * 4 + 1],
                                              v[p >> 1][(p & 1) * 4 + 2], v[p >> 1][(p & 1) * 4 + 3]);
    __syncwarp();
    const int part = lane & 7;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int item = r * 4 + (lane >> 3);
        if (item < nitems && (part >> 1) < nscal)
            *reinterpret_cast<uint4*>(base + (size_t)item * stride + part * 16) = st[item][part ^ (item & 7)];
    }
    __syncwarp();
}

// ---- per-thread scalar loads / stores (2 x 128-bit) ---------------------------------------------------
__device__ __forceinline__ void load_fr(uint32_t (&d)[8], const uint8_t* p) {
    const uint4 a = ldg128(p), b = ldg128(p + 16);
    d[0] = a.x, d[1] = a.y, d[2] = a.z, d[3] = a.w;
    d[4] = b.x, d[5] = b.y, d[6] = b.z, d[7] = b.w;
}
__device__ __forceinline__ void load_fr_rw(uint32_t (&d)[8], const uint8_t* p) {   // coherent (own stores)
    const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + 16);
    d[0] = a.x, d[1] = a.y, d[2] = a.z, d[3] = a.w;
    d[4] = b.x, d[5] = b.y, d[6] = b.z, d[7] = b.w;
}
__device__ __forceinline__ void store_fr(uint8_t* p, const uint32_t (&d)[8]) {
    *reinterpret_cast<uint4*>(p) = make_uint4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<uint4*>(p + 16) = make_uint4(d[4], d[5], d[6], d[7]);
}

// the lanes the last permutation of a digest must produce: only the rate lanes of the final squeeze chunk are read
__device__ __forceinline__ uint32_t last_squeeze_lanes(uint32_t out_len) {
    const uint32_t nout = (out_len + 3) / 4;
    const uint32_t left = out_len - 4 * (nout - 1);
    return ((1u << (left < 4 ? left : 4)) - 1u) << 1;
}

// ---- Hash::digest-shaped sponge: Absorb(in_len) -> Squeeze(out_len), item-major AoS ------------
// One permutation call site: step s > 0 is always preceded by a permutation; steps [0, nin) absorb
// 4-scalar chunks, steps [nin, nin+nout) squeeze 4-scalar chunks.  Permutations = nin + nout - 1
// = ceil(in_len/4) + ceil(out_len/4) - 1  (Merkle4: exactly 1).
// kTruncate: Hash::finalize_truncated (src/hash.rs:164-183) -- every squeezed scalar is taken
// out of Montgomery form and masked to 250 bits; the 4 x u64 written are the raw limbs the reference hands to
// JubJubScalar::from_raw.
// Launch shape: kT threads per block, register allocation held to kMB resident blocks per SM.  128 x 5 (96 registers,
// 20 warps/SM) is the general shape; 256 x 2 (128 registers, 16 warps/SM) serves only batches of many waves (the
// large-batch paths of launch_digest / launch_permute): below one wave its 8-warp blocks pile onto half the SMs.
template <bool kTruncate, int kT = kThreads, int kMB = kMinBlocks>
__global__ void __launch_bounds__(kT, kMB) k_sponge_digest(FrArg tag, const uint8_t* __restrict__ in, size_t n,
                                                            uint32_t in_len, uint8_t* __restrict__ out,
                                                            uint32_t out_len) {
    constexpr int kW = kT / 32;
    __shared__ uint4 stage[kW][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const size_t item0 = ((size_t)blockIdx.x * kW + warp) * 32;
    if (item0 >= n) return;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    uint4(*st)[8] = stage[warp];

    uint32_t s[5][8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        s[0][k] = tag.l[k];
        s[1][k] = s[2][k] = s[3][k] = s[4][k] = 0;
    }
    const uint32_t nin = (in_len + 3) / 4, nout = (out_len + 3) / 4;
    const uint8_t* in_w = in + item0 * (size_t)in_len * 32;
    uint8_t* out_w = out + item0 * (size_t)out_len * 32;
#pragma unroll 1
    for (uint32_t step = 0; step < nin + nout; ++step) {
        if (step > 0) {
            uint32_t need = 0x1fu;
            if (step + 1 == nin + nout) need = last_squeeze_lanes(out_len);
            hades_permute(s, need P252_TAB_PASS);
        }
        if (step < nin) {
            const uint32_t left = in_len - 4 * step;
            const int nscal = left < 4 ? (int)left : 4;
            uint32_t v[4][8];
            warp_gather(st, in_w + (size_t)step * 128, (size_t)in_len * 32, nitems, nscal, lane, v);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t t[8];
                    fr_add_mod(t, s[1 + q], v[q]);
#pragma unroll
                    for (int k = 0; k < 8; ++k) s[1 + q][k] = t[k];
                }
            }
        } else {
            const uint32_t c = step - nin;
            const uint32_t left = out_len - 4 * c;
            const int nscal = left < 4 ? (int)left : 4;
            uint32_t v[4][8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (kTruncate) {
                    fr_to_canonical(v[q], s[1 + q]);
                    v[q][7] &= 0x03ffffffu;               // TRUNCATION_MASK, src/hash.rs:167-172
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) v[q][k] = s[1 + q][k];
                }
            }
            warp_scatter(st, out_w + (size_t)c * 128, (size_t)out_len * 32, nitems, nscal, lane, v);
        }
    }
}

// ---- the same sponge for SMALL batches: five threads per item (hades_permute_coop) ----------------------------------
// 6 items per warp (lanes 0..29), 24 per 128-thread block.  Thread li of a group owns state lane li: lane 0 is the
// capacity (tag), lanes 1..4 the rate, so rate thread li absorbs input scalar 4*step + li - 1 and squeezes output
// scalar 4*c + li - 1.  Loads/stores are 2 x 128-bit per scalar per thread (tiny batches: coalescing is irrelevant).
constexpr int kCoopItemsPerWarp = 6;

// Where a thread of a lane-split kernel sits: thread li (state lane li) of group grp, which owns warp item `item`.
// mds_row fills lane li's MDS row for hades_permute_coop; the row stays a kernel-local array (held in the struct, it
// changes the kernels' SASS).
struct LaneSplit {
    int grp, li, g0;
    size_t first, item;                                          // first: the warp's first item
    __device__ __forceinline__ LaneSplit() {
        const int lane = threadIdx.x & 31;
        grp = lane / 5, li = lane - grp * 5, g0 = grp * 5;
        first = ((size_t)blockIdx.x * kWarps + (threadIdx.x >> 5)) * kCoopItemsPerWarp;
        item = first + grp;
    }
    __device__ __forceinline__ bool idle(size_t n) const { return first >= n; }   // the whole warp
    // idle threads (lanes 30, 31 and items past n) still take part in the shuffles
    __device__ __forceinline__ bool live(size_t n) const { return grp < kCoopItemsPerWarp && item < n; }
    __device__ __forceinline__ void mds_row(double (&crow)[5]) const {
#pragma unroll
        for (int j = 0; j < 5; ++j) crow[j] = (double)(HADES_LAMBDA / (uint32_t)(li + j + 5));
    }
};

__global__ void __launch_bounds__(kThreads) k_sponge_digest_coop(FrArg tag, const uint8_t* __restrict__ in, size_t n,
                                                                 uint32_t in_len, uint8_t* __restrict__ out, uint32_t out_len) {
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);

    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = (ls.li == 0) ? tag.l[k] : 0u;
    const uint32_t nin = (in_len + 3) / 4, nout = (out_len + 3) / 4;
    const uint8_t* in_i = in + (live ? ls.item : 0) * (size_t)in_len * 32;
    uint8_t* out_i = out + (live ? ls.item : 0) * (size_t)out_len * 32;
#pragma unroll 1
    for (uint32_t step = 0; step < nin + nout; ++step) {
        if (step > 0) hades_permute_coop(s, ls.li, ls.g0, crow);
        if (step < nin) {
            const uint32_t q = 4 * step + (uint32_t)ls.li - 1;   // li == 0 wraps to a huge value -> no absorb
            if (ls.li >= 1 && q < in_len) {
                uint32_t v[8], t[8];
                load_fr(v, in_i + (size_t)q * 32);
                fr_add_mod(t, s, v);
#pragma unroll
                for (int k = 0; k < 8; ++k) s[k] = t[k];
            }
        } else {
            const uint32_t q = 4 * (step - nin) + (uint32_t)ls.li - 1;
            if (live && ls.li >= 1 && q < out_len) store_fr(out_i + (size_t)q * 32, s);
        }
    }
}

// raw permutation, small batches: thread li of a group loads / stores lane li of its state (32 B)
__global__ void __launch_bounds__(kThreads) k_permute_coop(uint8_t* __restrict__ states, size_t n) {
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);
    uint8_t* p = states + (live ? ls.item : 0) * 160 + (size_t)ls.li * 32;
    uint32_t s[8];
    load_fr_rw(s, p);
    hades_permute_coop(s, ls.li, ls.g0, crow);
    if (live) store_fr(p, s);
}

// ---- raw permutation of n x 5 states in place (Safe::permute) -----------------------------------
template <bool kDense, int kT = kThreads, int kMB = kMinBlocks>
__global__ void __launch_bounds__(kT, kDense ? 1 : kMB) k_permute(uint8_t* __restrict__ states, size_t n) {
    constexpr int kW = kT / 32;
    __shared__ uint4 stage[kW][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const size_t item0 = ((size_t)blockIdx.x * kW + warp) * 32;
    if (item0 >= n) return;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    uint4(*st)[8] = stage[warp];
    uint8_t* base = states + item0 * 160;

    uint32_t s[5][8];
    {
        uint32_t v[4][8];
        warp_gather(st, base, 160, nitems, 4, lane, v);
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int k = 0; k < 8; ++k) s[q][k] = v[q][k];
        warp_gather(st, base + 128, 160, nitems, 1, lane, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[4][k] = v[0][k];
    }
    if (kDense)
        dense_permute(s);
    else
        hades_permute(s, 0x1fu P252_TAB_PASS);
    {
        uint32_t v[4][8];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int k = 0; k < 8; ++k) v[q][k] = s[q][k];
        warp_scatter(st, base, 160, nitems, 4, lane, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[0][k] = s[4][k];
        warp_scatter(st, base + 128, 160, nitems, 1, lane, v);
    }
}

// *counter += the number of active lanes of the warp with `hit`, one atomic per warp that has any
__device__ __forceinline__ void warp_count(unsigned long long* counter, bool hit) {
    const unsigned act = __activemask();
    const unsigned b = __ballot_sync(act, hit);
    if (b && (threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicAdd(counter, (unsigned long long)__popc(b));
}

// the same where every lane of the warp is still running: lane 0 adds
__device__ __forceinline__ void warp_count_full(unsigned long long* counter, bool hit) {
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if (b && (threadIdx.x & 31) == 0) atomicAdd(counter, (unsigned long long)__popc(b));
}

// ---- encrypt / decrypt (dusk_safe::encrypt / decrypt with Domain::Encryption) -------------------
// pattern [Absorb(2), Absorb(1), Squeeze(L), Absorb(L), Squeeze(1)]; 2*ceil(L/4) permutations.
template <bool kDecrypt>
__global__ void __launch_bounds__(kThreads, kMinBlocks) k_crypt(FrArg tag, const uint8_t* __restrict__ src, size_t n, uint32_t L,
                                                    const uint8_t* __restrict__ secret_uv,
                                                    const uint8_t* __restrict__ nonce, uint8_t* dst,
                                                    uint8_t* __restrict__ ok, unsigned long long* __restrict__ n_failed) {
    P252_STAGE_TABLES
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    // encrypt: src = message (n x L), dst = cipher (n x (L+1)); decrypt: the other way round
    const size_t src_len = kDecrypt ? (size_t)L + 1 : L, dst_len = kDecrypt ? L : (size_t)L + 1;
    const uint8_t* srci = src + i * src_len * 32;
    uint8_t* dsti = dst + i * dst_len * 32;
    const uint8_t* msgi = kDecrypt ? dsti : srci;        // the plaintext, wherever it lives

    uint32_t s[5][8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[0][k] = tag.l[k], s[4][k] = 0;
    load_fr(s[1], secret_uv + i * 64);                   // Absorb(2): u, v added to zero
    load_fr(s[2], secret_uv + i * 64 + 32);
    load_fr(s[3], nonce + i * 32);                       // Absorb(1)
    const uint32_t nk = (L + 3) / 4;
    bool good = true;
#pragma unroll 1
    for (uint32_t step = 0; step < 2 * nk; ++step) {
        hades_permute(s, (step + 1 == 2 * nk) ? 0x2u : 0x1fu P252_TAB_PASS);   // last: only the Squeeze(1) lane is read
        if (step < nk) {
            // Squeeze chunk `step` of the keystream and emit cipher (or recovered message)
            const uint32_t left = L - 4 * step;
            const int nscal = left < 4 ? (int)left : 4;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t x[8], y[8];
                    load_fr(x, srci + (size_t)(4 * step + q) * 32);
                    if (kDecrypt)
                        fr_sub_mod(y, x, s[1 + q]);      // Encryption::subtract
                    else
                        fr_add_mod(y, x, s[1 + q]);      // Safe::add
                    store_fr(dsti + (size_t)(4 * step + q) * 32, y);
                }
            }
        }
        if (step + 1 >= nk && step + 1 < 2 * nk) {
            // Absorb(L) chunk c of the plaintext: chunk 0 right after the last squeeze (no
            // permutation in between), chunk c > 0 after one more permutation each
            const uint32_t c = step + 1 - nk;
            const uint32_t left = L - 4 * c;
            const int nscal = left < 4 ? (int)left : 4;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t x[8], t[8];
                    if (kDecrypt)
                        load_fr_rw(x, msgi + (size_t)(4 * c + q) * 32);
                    else
                        load_fr(x, msgi + (size_t)(4 * c + q) * 32);
                    fr_add_mod(t, s[1 + q], x);
#pragma unroll
                    for (int k = 0; k < 8; ++k) s[1 + q][k] = t[k];
                }
            }
        }
        if (step + 1 == 2 * nk) {
            // Squeeze(1): authentication element
            if (kDecrypt) {
                uint32_t x[8];
                load_fr(x, srci + (size_t)L * 32);
#pragma unroll
                for (int k = 0; k < 8; ++k) good = good && (x[k] == s[1][k]);   // Encryption::is_equal
            } else {
                store_fr(dsti + (size_t)L * 32, s[1]);
            }
        }
    }
    if (kDecrypt) {
        ok[i] = good ? 1 : 0;
        if (!good) {                                      // Error::DecryptionFailed: release nothing
            const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t k = 0; k < L; ++k) store_fr(dsti + (size_t)k * 32, zero);
        }
        if (n_failed) warp_count(n_failed, !good);
    }
}

// ---- Merkle openings (consumer: poseidon-merkle `Opening`, AGENTS.md:62-66) -------------------
// A tree is stored as `leaves` + `nodes` (levels 1..depth bottom-up, root last).  Level l >= 1 starts at slot
// lv.off[l] of `nodes` and holds lv.m[l] occupied nodes; lv.m[0] is the number of occupied leaves.  The dense layout of
// p252_merkle_build is the case m[l] = n_leaves / arity^l, off[l] = sum_{q<l} m[q] - n_leaves; a fixed-height tree
// (p252_mtree) has padded levels.  The opening of leaf i holds, for every level l = 0..depth-1 (0 = leaf level), the
// whole sibling group of the path node: the `arity` items at positions [g*arity, (g+1)*arity) of level l, with
// g = i / arity^(l+1); the path node itself sits at offset (i / arity^l) % arity inside its group.  Slots at or beyond
// m[l] are written as zero (the empty-slot rule, src/hash.rs:24-26).
// k_merkle_open: pure gather, one thread per (opening, level).  kPresence (p252_smtree): the leaf must also be present
// (present[idx] != 0), otherwise the opening is all zero.
template <bool kPresence>
__global__ void __launch_bounds__(256) k_merkle_open(const uint8_t* __restrict__ leaves, const uint8_t* __restrict__ nodes,
                                                     const uint64_t* __restrict__ leaf_idx, size_t n, uint32_t log2_arity,
                                                     uint32_t depth, OpenLevels lv, uint8_t* __restrict__ paths,
                                                     const uint8_t* __restrict__ present) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * depth) return;
    const size_t item = t / depth;
    const uint32_t level = (uint32_t)(t % depth);
    const uint32_t arity = 1u << log2_arity;
    const uint64_t idx = leaf_idx[item];
    uint4* dst = reinterpret_cast<uint4*>(paths + ((size_t)item * depth + level) * arity * 32);
    if (idx >= lv.m[0] || (kPresence && !present[idx])) { // HOST buffers are rejected on the host; a device index outside
        for (uint32_t q = 0; q < arity * 2; ++q)          // the prefix gets an all-zero opening (it cannot verify)
            dst[q] = make_uint4(0, 0, 0, 0);
        return;
    }
    const uint64_t group = idx >> (log2_arity * (level + 1));
    const uint8_t* src = (level == 0 ? leaves : nodes + lv.off[level] * 32) + group * arity * 32;
    for (uint32_t q = 0; q < arity * 2; ++q)
        dst[q] = (group * arity + q / 2 < lv.m[level]) ? ldg128(src + q * 16) : make_uint4(0, 0, 0, 0);
}

// ---- fixed-height trees: batched leaf updates that rehash only the touched paths (p252_mtree_update) ----------------
// The dirty set of a level is a sorted array of distinct node indices whose length lives on the device (*cnt); the
// host sizes every launch by an upper bound and threads at or past *cnt do nothing.
//
// k_mtree_keys: one thread per batch item.  Overwrites carry their leaf index (an index >= n_old gets the sentinel key
// n_new, sorted last and skipped, and is counted into *rejected); append j gets key n_old + j.  pos = batch position.
__global__ void __launch_bounds__(256) k_mtree_keys(const uint64_t* __restrict__ idx, uint32_t n_upd, uint64_t n_old,
                                                    uint32_t total, uint64_t* __restrict__ keys, uint32_t* __restrict__ pos,
                                                    unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    uint64_t key;
    bool bad = false;
    if (i < n_upd) {
        key = idx[i];
        bad = key >= n_old;
        if (bad) key = n_old + (total - n_upd);           // sentinel = n_new
    } else {
        key = n_old + (i - n_upd);
    }
    keys[i] = key;
    pos[i] = i;
    if (rejected) warp_count(rejected, bad);
}

// k_mtree_leaf_write: over the keys sorted stably by leaf index, the last item of every run of equal keys (the last
// write in batch order) stores its value into leaves[key].  Also emits the level-1 candidates: flag[i] = 1 for the
// first key of every run of equal parents key / arity, parent[i] = key / arity.
__global__ void __launch_bounds__(256) k_mtree_leaf_write(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ pos,
                                                          uint32_t total, uint64_t sentinel, uint32_t log2_arity,
                                                          const uint8_t* __restrict__ values, uint32_t n_upd,
                                                          const uint8_t* __restrict__ append, uint8_t* __restrict__ leaves,
                                                          uint8_t* __restrict__ flag, uint64_t* __restrict__ parent) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint64_t key = keys[i];
    const bool valid = key != sentinel;
    if (valid && (i + 1 == total || keys[i + 1] != key)) {
        const uint32_t p = pos[i];
        const uint8_t* src = p < n_upd ? values + (size_t)p * 32 : append + (size_t)(p - n_upd) * 32;
        uint32_t v[8];
        load_fr(v, src);
        store_fr(leaves + key * 32, v);
    }
    const uint64_t par = key >> log2_arity;
    flag[i] = valid && (i == 0 || (keys[i - 1] >> log2_arity) != par);
    parent[i] = par;
}

// k_mtree_parents: the same candidates one level further up, from a compacted dirty set d[0..*cnt).
__global__ void __launch_bounds__(256) k_mtree_parents(const uint64_t* __restrict__ d, const int* __restrict__ cnt,
                                                       uint32_t bound, uint32_t log2_arity, uint8_t* __restrict__ flag,
                                                       uint64_t* __restrict__ parent) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= bound) return;
    const bool valid = (int)i < *cnt;
    const uint64_t par = valid ? d[i] >> log2_arity : 0;
    flag[i] = valid && (i == 0 || (d[i - 1] >> log2_arity) != par);
    parent[i] = par;
}

// k_mtree_digest: the Merkle case of k_sponge_digest with an index indirection -- warp item k hashes group d[k] of the
// level below (the arity children at [d[k]*arity, d[k]*arity + arity)) into slot d[k] of its level.  Groups are whole
// aligned 32*arity-byte segments, so the warp tile still moves complete segments (4 x 128 B per LDG.128 for arity 4).
// 4 resident blocks per SM (128 registers): a dirty set is rarely more than one wave, and at kMinBlocks' 96 registers
// the permutation spills.
// kSparse (p252_smtree): presence bytes ride along -- below_present / level_present are indexed like below / level.  A
// group whose arity presence bytes are all zero is empty: its node stores value 0 and presence 0; any other node stores
// its digest and presence 1.  A warp whose groups are all empty skips the permutation.  Each node's value and presence
// byte are written only by the lane that owns the node.
__device__ __forceinline__ bool group_present(const uint8_t* p, uint32_t arity) {
    // per-level slot counts are multiples of the arity: a group's presence bytes are one aligned 16- or 32-bit word
    return arity == 4 ? *reinterpret_cast<const uint32_t*>(p) != 0u : *reinterpret_cast<const uint16_t*>(p) != 0u;
}

template <int kLog2Arity, bool kSparse>
__global__ void __launch_bounds__(kThreads, 4) k_mtree_digest(FrArg tag, const uint8_t* __restrict__ below,
                                                                       uint8_t* __restrict__ level, const uint64_t* __restrict__ d,
                                                                       const int* __restrict__ cnt,
                                                                       const uint8_t* __restrict__ below_present,
                                                                       uint8_t* __restrict__ level_present) {
    constexpr int kArity = 1 << kLog2Arity;
    __shared__ uint4 stage[kWarps][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const size_t n = (size_t)*cnt;
    const size_t item0 = ((size_t)blockIdx.x * kWarps + warp) * 32;
    if (item0 >= n) return;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    uint4(*st)[8] = stage[warp];
    const uint64_t mine = d[item0 + (lane < nitems ? lane : 0)];
    bool any = true;
    if (kSparse) any = group_present(below_present + mine * kArity, kArity);
    const int part = lane & 7;
#pragma unroll
    for (int r = 0; r < 8; ++r) {                          // warp_gather with a per-item base address
        const int item = r * 4 + (lane >> 3);
        const uint64_t g = __shfl_sync(0xffffffffu, mine, item);
        uint4 x = make_uint4(0, 0, 0, 0);
        if (item < nitems && (part >> 1) < kArity) x = ldg128(below + g * (kArity * 32) + part * 16);
        st[item][part ^ (item & 7)] = x;
    }
    __syncwarp();
    uint32_t s[5][8];
    tile_row(st, lane, s + 1);
#pragma unroll
    for (int q = 0; q < 4; ++q) {                          // absorb into the zero rate lanes, as k_sponge_digest does
        uint32_t t[8];
        const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        fr_add_mod(t, zero, s[1 + q]);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[1 + q][k] = (q < kArity) ? t[k] : 0u;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s[0][k] = tag.l[k];
    if (kSparse) {
        if (__any_sync(0xffffffffu, any && lane < nitems)) hades_permute(s, 0x2u P252_TAB_PASS);
        if (lane < nitems) {
#pragma unroll
            for (int k = 0; k < 8; ++k) s[1][k] = any ? s[1][k] : 0u;
            store_fr(level + mine * 32, s[1]);
            level_present[mine] = any ? 1 : 0;
        }
        return;
    }
    hades_permute(s, 0x2u P252_TAB_PASS);                  // a Merkle digest reads lane 1 only
    if (lane < nitems) store_fr(level + mine * 32, s[1]);
}

// the same for small dirty sets: five threads per item (hades_permute_coop), as k_sponge_digest_coop
template <bool kSparse>
__global__ void __launch_bounds__(kThreads) k_mtree_digest_coop(FrArg tag, const uint8_t* __restrict__ below, uint32_t arity,
                                                                uint8_t* __restrict__ level, const uint64_t* __restrict__ d,
                                                                const int* __restrict__ cnt,
                                                                const uint8_t* __restrict__ below_present,
                                                                uint8_t* __restrict__ level_present) {
    const size_t n = (size_t)*cnt;
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);
    const uint64_t g = live ? d[ls.item] : 0;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = (ls.li == 0) ? tag.l[k] : 0u;
    if (live && ls.li >= 1 && (uint32_t)ls.li <= arity) {
        uint32_t v[8], t[8];
        load_fr(v, below + (g * arity + (uint32_t)ls.li - 1) * 32);
        fr_add_mod(t, s, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] = t[k];
    }
    hades_permute_coop(s, ls.li, ls.g0, crow);                    // collective: every thread of the warp takes part
    if (kSparse) {
        if (live && ls.li == 1) {
            const bool any = group_present(below_present + g * arity, arity);
#pragma unroll
            for (int k = 0; k < 8; ++k) s[k] = any ? s[k] : 0u;
            store_fr(level + g * 32, s);
            level_present[g] = any ? 1 : 0;
        }
        return;
    }
    if (live && ls.li == 1) store_fr(level + g * 32, s);
}

// ---- sparse fixed-height trees: inserts and removals at any position (p252_smtree) -----------------------------------
// The climb is the one of p252_mtree_update (k_mtree_parents, DeviceSelect::Flagged) with the kSparse digest; presence
// bytes are laid out like the scalars (leaves, then nodes).
//
// k_smtree_keys: one thread per batch item.  key = pos[i] for a valid item (pos < capacity, op 0 or 1), the sentinel
// `capacity` otherwise (sorted last, skipped, counted into *rejected with one atomic per warp); bpos[i] = i.
__global__ void __launch_bounds__(256) k_smtree_keys(const uint64_t* __restrict__ pos, const uint8_t* __restrict__ op,
                                                     uint32_t n, uint64_t capacity, uint64_t* __restrict__ keys,
                                                     uint32_t* __restrict__ bpos, unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t key = pos[i];
    const bool bad = key >= capacity || (op && op[i] > 1);
    keys[i] = bad ? capacity : key;
    bpos[i] = i;
    if (rejected) warp_count(rejected, bad);
}

// k_smtree_leaf_write: over the keys sorted stably by position, the last item of every run of equal keys (the last
// operation in batch order) applies its op: insert (op 0, or no op array) stores its value and presence 1, remove
// (op 1) stores zero and presence 0.  Emits the level-1 candidates as k_mtree_leaf_write does.
__global__ void __launch_bounds__(256) k_smtree_leaf_write(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ bpos,
                                                           uint32_t n, uint64_t sentinel, uint32_t log2_arity,
                                                           const uint8_t* __restrict__ op, const uint8_t* __restrict__ values,
                                                           uint8_t* __restrict__ leaves, uint8_t* __restrict__ present,
                                                           uint8_t* __restrict__ flag, uint64_t* __restrict__ parent) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t key = keys[i];
    const bool valid = key != sentinel;
    if (valid && (i + 1 == n || keys[i + 1] != key)) {
        const uint32_t p = bpos[i];
        const bool insert = !op || op[p] == 0;
        uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (insert) load_fr(v, values + (size_t)p * 32);
        store_fr(leaves + key * 32, v);
        present[key] = insert ? 1 : 0;
    }
    const uint64_t par = key >> log2_arity;
    flag[i] = valid && (i == 0 || (keys[i - 1] >> log2_arity) != par);
    parent[i] = par;
}

// k_smtree_seed (build): one thread per leaf group g.  Normalises the group's presence bytes (a slot is present iff its
// byte is non-zero and it lies below capacity), zeroes the value of every absent leaf, and makes the group a level-1
// candidate iff one of its leaves is present: flag[g], parent[g] = g.
__global__ void __launch_bounds__(256) k_smtree_seed(uint8_t* __restrict__ present, uint8_t* __restrict__ leaves, uint64_t groups,
                                                     uint64_t capacity, uint32_t log2_arity, uint8_t* __restrict__ flag,
                                                     uint64_t* __restrict__ parent) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    const uint32_t arity = 1u << log2_arity;
    bool any = false;
    for (uint32_t q = 0; q < arity; ++q) {
        const uint64_t j = g * arity + q;
        const bool p = j < capacity && present[j] != 0;
        present[j] = p ? 1 : 0;
        any = any || p;
        if (!p) {
            const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            store_fr(leaves + j * 32, zero);
        }
    }
    flag[g] = any;
    parent[g] = g;
}

// k_smtree_count: *out += number of non-zero bytes in present[0, n) (grid-stride, one atomic per warp)
__global__ void __launch_bounds__(256) k_smtree_count(const uint8_t* __restrict__ present, uint64_t n,
                                                      unsigned long long* __restrict__ out) {
    unsigned c = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        c += present[i] != 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// ---- compact sparse trees: sorted (index, value) lists per level (p252_ctree) -----------------------------------------
// A change list is (key, value, present) sorted by key with distinct keys: present 1 inserts or overwrites, 0 removes.
// Level l's merge takes its sorted list (keys / values, count on the device) and its change list to a new sorted list
// out of place; the dirty parents of level l + 1 (k_mtree_parents over the change list) are gathered from the new list and
// hashed by the presence-aware launch_mtree_digest.

// first index in a[0, n) whose key is >= k
__device__ __forceinline__ uint64_t ctree_lower_bound(const uint64_t* __restrict__ a, uint64_t n, uint64_t k) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (a[mid] < k)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// exclusive prefix sum at x of flags f[0, s) with scan e: x == s is the total
__device__ __forceinline__ uint64_t ctree_excl(const uint32_t* __restrict__ e, const uint32_t* __restrict__ f, uint64_t s,
                                               uint64_t x) {
    return x < s ? e[x] : (uint64_t)e[s - 1] + f[s - 1];
}

// k_ctree_keys: one thread per batch item.  keys[i] = pos[i]; bpos[i] = i, with bit 31 set for an invalid item (pos >
// max_pos, or op not 0/1), which is counted into *rejected.  No key value is free to act as a sentinel.
__global__ void __launch_bounds__(256) k_ctree_keys(const uint64_t* __restrict__ pos, const uint8_t* __restrict__ op, uint32_t n,
                                                    uint64_t max_pos, uint64_t* __restrict__ keys, uint32_t* __restrict__ bpos,
                                                    unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t key = pos[i];
    const bool bad = key > max_pos || (op && op[i] > 1);
    keys[i] = key;
    bpos[i] = i | (bad ? 0x80000000u : 0u);
    if (rejected) warp_count(rejected, bad);
}

// k_ctree_valid: flag[k] = the sorted item k is valid (bit 31 of its batch position clear)
__global__ void __launch_bounds__(256) k_ctree_valid(const uint32_t* __restrict__ bpos, uint32_t n, uint8_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = (bpos[i] >> 31) == 0;
}

// k_ctree_last: over the valid items sorted stably by position (count *cnt <= n), flag the last of every run of equal
// positions: the last operation in batch order
__global__ void __launch_bounds__(256) k_ctree_last(const uint64_t* __restrict__ keys, const int* __restrict__ cnt, uint32_t n,
                                                    uint8_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t c = (uint32_t)*cnt;
    flag[i] = i < c && (i + 1 == c || keys[i + 1] != keys[i]);
}

// k_ctree_leaf_changes: level 0's change list from the last operation per position: value and present = insert
__global__ void __launch_bounds__(256) k_ctree_leaf_changes(const uint32_t* __restrict__ bpos, const int* __restrict__ cnt,
                                                            uint32_t n, const uint8_t* __restrict__ op,
                                                            const uint8_t* __restrict__ values, uint8_t* __restrict__ cval,
                                                            uint8_t* __restrict__ cpres) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || i >= (uint32_t)*cnt) return;
    const uint32_t p = bpos[i];
    const bool insert = !op || op[p] == 0;
    uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (insert) load_fr(v, values + (size_t)p * 32);
    store_fr(cval + (size_t)i * 32, v);
    cpres[i] = insert ? 1 : 0;
}

// k_ctree_mark: kept[t] (t < s) = old entry t exists and no change has its key; ins[t] (t < nb) = change t inserts
__global__ void __launch_bounds__(256) k_ctree_mark(const uint64_t* __restrict__ lkeys, const uint64_t* __restrict__ lcount,
                                                    uint64_t s, const uint64_t* __restrict__ ckeys, const int* __restrict__ ccnt,
                                                    uint32_t nb, const uint8_t* __restrict__ cpres, uint32_t* __restrict__ kept,
                                                    uint32_t* __restrict__ ins) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t cn = (uint64_t)*ccnt;
    if (t < s) {
        bool k = t < *lcount;
        if (k) {
            const uint64_t key = lkeys[t];
            const uint64_t j = ctree_lower_bound(ckeys, cn, key);
            k = j == cn || ckeys[j] != key;
        }
        kept[t] = k;
    }
    if (t < nb) ins[t] = t < cn && cpres[t];
}

// k_ctree_scatter: the merge.  A kept old entry t goes to K(t) + I(changes below its key), an inserting change t to
// I(t) + K(old entries below its key) (K / I: exclusive scans of kept / ins).  Writes at or past s are dropped: only a
// level-0 overflow produces them, and then nothing is committed.
__global__ void __launch_bounds__(256) k_ctree_scatter(const uint64_t* __restrict__ lkeys, const uint8_t* __restrict__ lvals,
                                                       const uint64_t* __restrict__ lcount, uint64_t s,
                                                       const uint64_t* __restrict__ ckeys, const uint8_t* __restrict__ cvals,
                                                       const int* __restrict__ ccnt, uint32_t nb, const uint32_t* __restrict__ kept,
                                                       const uint32_t* __restrict__ K, const uint32_t* __restrict__ ins,
                                                       const uint32_t* __restrict__ I, uint64_t* __restrict__ okeys,
                                                       uint8_t* __restrict__ ovals) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t cn = (uint64_t)*ccnt;
    if (t < s && kept[t]) {
        const uint64_t key = lkeys[t];
        const uint64_t p = K[t] + (nb ? ctree_excl(I, ins, nb, ctree_lower_bound(ckeys, cn, key)) : 0);
        if (p < s) {
            uint32_t v[8];
            load_fr(v, lvals + t * 32);
            okeys[p] = key;
            store_fr(ovals + p * 32, v);
        }
    }
    if (t < nb && ins[t]) {
        const uint64_t key = ckeys[t];
        const uint64_t p = I[t] + ctree_excl(K, kept, s, ctree_lower_bound(lkeys, *lcount, key));
        if (p < s) {
            uint32_t v[8];
            load_fr(v, cvals + t * 32);
            okeys[p] = key;
            store_fr(ovals + p * 32, v);
        }
    }
}

// k_ctree_count (one thread): st = {old count, new count}.  Level 0 decides the commit flag: the new count fits the
// level's s slots; a refused batch reports every item as rejected.
__global__ void k_ctree_count(const uint64_t* __restrict__ lcount, uint64_t s, uint32_t nb, const uint32_t* __restrict__ kept,
                              const uint32_t* __restrict__ K, const uint32_t* __restrict__ ins, const uint32_t* __restrict__ I,
                              bool level0, uint32_t n, uint64_t* __restrict__ st, uint32_t* __restrict__ ok,
                              unsigned long long* __restrict__ rejected) {
    const uint64_t c = ctree_excl(K, kept, s, s) + (nb ? ctree_excl(I, ins, nb, nb) : 0);
    st[0] = *lcount;
    st[1] = c;
    if (level0) {
        *ok = c <= s;
        if (c > s && rejected) *rejected = n;
    }
}

// k_ctree_commit: if *ok, level := the merged list; slots past the new count that held entries are zeroed (every slot
// past the old count is already zero)
__global__ void __launch_bounds__(256) k_ctree_commit(const uint64_t* __restrict__ okeys, const uint8_t* __restrict__ ovals,
                                                      uint64_t s, const uint64_t* __restrict__ st, const uint32_t* __restrict__ ok,
                                                      uint64_t* __restrict__ lkeys, uint8_t* __restrict__ lvals,
                                                      uint64_t* __restrict__ lcount) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= s || !*ok) return;
    const uint64_t old = st[0], c = st[1];
    if (t == 0) *lcount = c;
    uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (t < c) {
        load_fr(v, ovals + t * 32);
        lkeys[t] = okeys[t];
        store_fr(lvals + t * 32, v);
    } else if (t < old) {
        lkeys[t] = 0;
        store_fr(lvals + t * 32, v);
    }
}

// k_ctree_gather: one thread per dirty parent g: its arity children in the merged level (binary search for g * arity,
// then at most arity consecutive entries) as a dense group, absent slots 0, and their presence bytes
__global__ void __launch_bounds__(256) k_ctree_gather(const uint64_t* __restrict__ okeys, const uint8_t* __restrict__ ovals,
                                                      const uint64_t* __restrict__ st, uint64_t s, const uint64_t* __restrict__ pkeys,
                                                      const int* __restrict__ pcnt, uint32_t nb, uint32_t log2_arity,
                                                      uint8_t* __restrict__ groups, uint8_t* __restrict__ gpres) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nb || t >= (uint32_t)*pcnt) return;
    const uint32_t arity = 1u << log2_arity;
    const uint64_t c = st[1] < s ? st[1] : s;
    const uint64_t base = pkeys[t] << log2_arity;
    uint64_t p = ctree_lower_bound(okeys, c, base);
    for (uint32_t q = 0; q < arity; ++q) {
        uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const bool here = p < c && okeys[p] == base + q;
        if (here) load_fr(v, ovals + (p++) * 32);
        store_fr(groups + ((size_t)t * arity + q) * 32, v);
        gpres[(size_t)t * arity + q] = here ? 1 : 0;
    }
}

__global__ void __launch_bounds__(256) k_ctree_iota(uint64_t* __restrict__ d, uint32_t n) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) d[t] = t;
}

// k_ctree_open: one thread per (opening, level) as k_merkle_open.  The leaf must be present in level 0 (binary search),
// otherwise the opening is all zero; the sibling group of level l is found by a binary search for its first index.
__global__ void __launch_bounds__(256) k_ctree_open(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ vals,
                                                    const uint64_t* __restrict__ count, const uint64_t* __restrict__ pos, size_t n,
                                                    uint32_t log2_arity, uint32_t depth, OpenLevels lv, uint8_t* __restrict__ paths) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * depth) return;
    const size_t item = t / depth;
    const uint32_t level = (uint32_t)(t - item * depth);
    const uint32_t arity = 1u << log2_arity;
    const uint64_t idx = pos[item];
    uint8_t* dst = paths + ((size_t)item * depth + level) * arity * 32;
    const uint64_t c0 = count[0];
    const uint64_t j0 = ctree_lower_bound(keys, c0, idx);
    const bool present = j0 < c0 && keys[j0] == idx;
    const uint64_t* lk = keys + lv.off[level];
    const uint8_t* lvv = vals + lv.off[level] * 32;
    const uint64_t c = present ? count[level] : 0;
    const uint64_t base = (idx >> (log2_arity * level)) >> log2_arity << log2_arity;
    uint64_t p = ctree_lower_bound(lk, c, base);
    for (uint32_t q = 0; q < arity; ++q) {
        uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (p < c && lk[p] == base + q) load_fr(v, lvv + (p++) * 32);
        store_fr(dst + q * 32, v);
    }
}

// k_merkle_verify: one thread per opening, `depth` chained Merkle digests (Hash::digest(Domain::MerkleA, group),
// src/hash.rs:22-31,191-195) with the membership check of every level fused in:
//   cur = leaf;  for l: require group[l][pos_l] == cur;  cur = digest(group[l]);   finally require cur == root.
// The sibling groups are read with the same warp-cooperative 128-bit tile as k_sponge_digest.
template <int kLog2Arity>
__global__ void __launch_bounds__(kThreads, kMinBlocks) k_merkle_verify(FrArg tag, FrArg root, const uint8_t* __restrict__ leaf_items,
                                                                        const uint64_t* __restrict__ leaf_idx,
                                                                        const uint8_t* __restrict__ paths, size_t n, uint32_t depth,
                                                                        uint8_t* __restrict__ ok,
                                                                        unsigned long long* __restrict__ n_failed) {
    constexpr int kArity = 1 << kLog2Arity;
    __shared__ uint4 stage[kWarps][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const size_t item0 = ((size_t)blockIdx.x * kWarps + warp) * 32;
    if (item0 >= n) return;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    const bool live = lane < nitems;
    uint4(*st)[8] = stage[warp];
    const size_t me = item0 + (live ? lane : 0);

    uint32_t cur[8];
    load_fr(cur, leaf_items + me * 32);
    uint64_t idx = leaf_idx[me];
    bool good = true;
    const size_t stride = (size_t)depth * kArity * 32;
    const uint8_t* base = paths + item0 * stride;
#pragma unroll 1
    for (uint32_t level = 0; level < depth; ++level) {
        uint32_t v[4][8];
        warp_gather(st, base + (size_t)level * kArity * 32, stride, nitems, kArity, lane, v);
        const uint32_t pos = (uint32_t)idx & (kArity - 1);
        idx >>= kLog2Arity;
        uint32_t diff = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            uint32_t sel = v[0][k];
#pragma unroll
            for (int q = 1; q < kArity; ++q) sel = (pos == (uint32_t)q) ? v[q][k] : sel;
            diff |= sel ^ cur[k];
        }
        good = good && (diff == 0);
        uint32_t s[5][8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            s[0][k] = tag.l[k];
#pragma unroll
            for (int q = 0; q < 4; ++q) s[1 + q][k] = (q < kArity) ? v[q][k] : 0u;
        }
        hades_permute(s, 0x2u P252_TAB_PASS);          // a Merkle digest reads lane 1 only
#pragma unroll
        for (int k = 0; k < 8; ++k) cur[k] = s[1][k];
    }
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) diff |= cur[k] ^ root.l[k];
    good = good && (diff == 0) && (idx == 0);             // idx != 0: leaf index beyond arity^depth
    if (live) ok[me] = good ? 1 : 0;
    if (n_failed) warp_count_full(n_failed, live && !good);
}

// ---- variable-length digest batches (p252_hash_batch_varlen) ------------------------------------------------------
// Item i is the input range [offsets[i] - base, offsets[i+1] - base) of `in` (n_scalars scalars); base lets a staged
// chunk keep the caller's offsets.  tags[len] is the tag of Hash::digest over `len` inputs (tags[0] = 0, unused).
//
// k_varlen_keys: one thread per item.  key = len for a valid item, 0 for an invalid one (counted into *rejected, one
// atomic per warp); value = i.  Valid: offsets[i] - base <= offsets[i+1] - base <= n_scalars, 1 <= len <= max_len and,
// for a Merkle domain (fixed_len != 0), len == fixed_len.  Every later read of `in` is bounded by this check.
// kCrypt (p252_encrypt_batch_varlen = 1, p252_decrypt_batch_varlen = 2; fixed_len unused): with a0 = offsets[0] - base
// and an = offsets[n] - base, valid iff a0 <= a <= b <= an <= n_scalars and 1 <= len <= max_len (encrypt) or
// 2 <= len <= max_len + 1 plus a - a0 >= i and an - b >= n - 1 - i (decrypt: the message range [a - a0 - i,
// b - a0 - i - 1) lies inside an output of an - a0 - n scalars).  key = the message length (len, or len - 1 for decrypt).
template <int kCrypt>
__device__ __forceinline__ bool crypt_item_ok(const uint64_t* __restrict__ offsets, uint32_t n, uint64_t base, uint64_t n_scalars,
                                              uint32_t max_len, uint32_t i, uint64_t a, uint64_t b) {
    constexpr uint64_t kMin = kCrypt == 2 ? 2u : 1u;              // a cipher carries one authentication scalar more
    const uint64_t a0 = offsets[0] - base, an = offsets[n] - base, len = b - a;
    bool ok = a0 <= a && a <= b && b <= an && an <= n_scalars && len >= kMin && len <= (uint64_t)max_len + kMin - 1;
    if (kCrypt == 2) ok = ok && a - a0 >= i && an - b >= (uint64_t)(n - 1 - i);
    return ok;
}

template <int kCrypt>
__global__ void __launch_bounds__(256) k_varlen_keys(const uint64_t* __restrict__ offsets, uint32_t n, uint64_t base,
                                                     uint64_t n_scalars, uint32_t max_len, uint32_t fixed_len,
                                                     uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                     unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t a = offsets[i] - base, b = offsets[i + 1] - base;
    const uint64_t len = b - a;
    const bool ok = kCrypt == 0
                        ? a <= b && b <= n_scalars && len >= 1 && len <= max_len && (fixed_len == 0 || len == fixed_len)
                        : crypt_item_ok<kCrypt>(offsets, n, base, n_scalars, max_len, i, a, b);
    keys[i] = ok ? (uint32_t)(len - (kCrypt == 2 ? 1 : 0)) : 0u;
    vals[i] = i;
    if (rejected) warp_count(rejected, !ok);
}

// The loop of the variable-length digest kernels, one lane per item, shared by k_sponge_digest_varlen (one out_len and a
// tag table indexed by length) and k_sponge_digest_mixed (kMixed: a tag, out_len, output base and truncation per lane).
// tag: the lane's tag row; src / dst: its input and output rows; len == 0: a rejected item (out_len zero rows).  The loop
// runs to the warp's largest step count; a lane past its own last step neither absorbs nor permutes.  kMixed && trunc:
// every squeezed scalar is stored as k_sponge_digest<true> stores it.  kMixed keeps out_len and trunc in one word, the
// last squeeze chunk's padding 4 nout - out_len | trunc << 2: a per-lane out_len takes a register the kernel parameter
// of k_sponge_digest_varlen does not, and a second one for trunc spills under the 128-register bound.
template <bool kMixed>
__device__ __forceinline__ void sponge_varlen_lane(uint4 (*st)[8], int lane, bool live, const uint8_t* tag, const uint8_t* src,
                                                   uint8_t* dst, uint32_t len, uint32_t out_len, bool trunc) {
    const uint32_t nin = (len + 3) / 4, nout = (out_len + 3) / 4;
    const uint32_t steps = len ? nin + nout : 0u;
    const uint32_t wsteps = __reduce_max_sync(0xffffffffu, steps);
    const uint32_t tail = kMixed ? (4 * nout - out_len) | (trunc ? 4u : 0u) : 0u;
    uint32_t s[5][8];
    load_fr(s[0], tag);
#pragma unroll
    for (int q = 1; q < 5; ++q)
#pragma unroll
        for (int w = 0; w < 8; ++w) s[q][w] = 0;
    if (live && len == 0)                                  // rejected: a zero row
        for (uint32_t q = 0; q < out_len; ++q) store_fr(dst + (size_t)q * 32, s[1]);
    const int part = lane & 7;
#pragma unroll 1
    for (uint32_t step = 0; step < wsteps; ++step) {
        if (step > 0 && step < steps) {
            uint32_t need = 0x1fu;
            if (step + 1 == steps) need = kMixed ? ((1u << (4 - (tail & 3))) - 1u) << 1 : last_squeeze_lanes(out_len);
            hades_permute(s, need P252_TAB_PASS);
        }
        const uint32_t left = step < nin ? len - 4 * step : 0u;
        const int nscal = left < 4 ? (int)left : 4;
        if (__any_sync(0xffffffffu, nscal > 0)) {
            const uint8_t* mine = src + (size_t)step * 128;
#pragma unroll
            for (int r = 0; r < 8; ++r) {                  // warp_gather with a per-item base address and width
                const int item = r * 4 + (lane >> 3);
                const uint8_t* g = reinterpret_cast<const uint8_t*>(
                    __shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(mine), item));
                const int ns = __shfl_sync(0xffffffffu, nscal, item);
                uint4 x = make_uint4(0, 0, 0, 0);
                if ((part >> 1) < ns) x = ldg128(g + part * 16);
                st[item][part ^ (item & 7)] = x;
            }
            __syncwarp();
            uint32_t v[4][8];
            tile_row(st, lane, v);
            __syncwarp();
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t t[8];
                    fr_add_mod(t, s[1 + q], v[q]);
#pragma unroll
                    for (int w = 0; w < 8; ++w) s[1 + q][w] = t[w];
                }
            }
        }
        if (step >= nin && step < steps) {
            const uint32_t c = step - nin;
            const uint32_t oleft = kMixed ? 4 * (steps - step) - (tail & 3) : out_len - 4 * c;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if ((uint32_t)q < oleft) {
                    if (kMixed && (tail & 4)) {
                        uint32_t v[8];
                        fr_to_canonical(v, s[1 + q]);
                        v[7] &= 0x03ffffffu;               // TRUNCATION_MASK, src/hash.rs:167-172
                        store_fr(dst + (size_t)(4 * c + q) * 32, v);
                    } else {
                        store_fr(dst + (size_t)(4 * c + q) * 32, s[1 + q]);
                    }
                }
            }
        }
    }
}

// k_sponge_digest_varlen: k_sponge_digest over the items sorted by length.  Warp item k is item i = perm[k] with
// len = lens[k]; every lane carries its own tag, step count and last-chunk width, input chunks go through the warp tile
// with a per-item base address (shuffled, as in k_mtree_digest), outputs are stored per item.  Rejected items (len 0,
// sorted to the front) write zero rows.  Warps take the sorted segments from the end, so the longest items start first.
// 4 resident blocks per SM (128 registers): the per-lane sponge bookkeeping does not fit kMinBlocks' 96 without spills.
__global__ void __launch_bounds__(kThreads, 4) k_sponge_digest_varlen(const uint8_t* __restrict__ tags,
                                                                      const uint8_t* __restrict__ in, uint64_t base,
                                                                      const uint64_t* __restrict__ offsets,
                                                                      const uint32_t* __restrict__ lens,
                                                                      const uint32_t* __restrict__ perm, uint32_t n,
                                                                      uint8_t* __restrict__ out, uint32_t out_len) {
    __shared__ uint4 stage[kWarps][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t nseg = (n + 31) / 32;
    const uint32_t wg = blockIdx.x * kWarps + warp;
    if (wg >= nseg) return;
    const uint32_t item0 = (nseg - 1 - wg) * 32;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    const bool live = lane < nitems;
    const uint32_t k = item0 + (live ? lane : 0);
    const uint32_t len = live ? lens[k] : 0u;
    const uint32_t i = perm[k];
    const uint8_t* src = in + (len ? (offsets[i] - base) * 32 : 0);
    uint8_t* dst = out + (size_t)i * out_len * 32;
    sponge_varlen_lane<false>(stage[warp], lane, live, tags + (size_t)len * 32, src, dst, len, out_len, false);
}

// k_sponge_digest_mixed (p252_hash_batch_mixed): the same over the order of k_mixed_keys and the sort (by step count).
// Warp item k is item i = perm[k]; desc[i] = (len, out_len | truncated << 31), (0, 0) for a rejected item (its zero rows
// were written by k_mixed_keys), so a lane of a rejected item only idles; tags + 32 i is its tag, row out_offsets[i] -
// obase of `out` its first output row.
__global__ void __launch_bounds__(kThreads, 4) k_sponge_digest_mixed(const uint8_t* __restrict__ tags,
                                                                     const uint2* __restrict__ desc,
                                                                     const uint8_t* __restrict__ in, uint64_t base,
                                                                     const uint64_t* __restrict__ offsets, uint64_t obase,
                                                                     const uint64_t* __restrict__ out_offsets,
                                                                     const uint32_t* __restrict__ perm, uint32_t n,
                                                                     uint8_t* __restrict__ out) {
    __shared__ uint4 stage[kWarps][32][8];
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t nseg = (n + 31) / 32;
    const uint32_t wg = blockIdx.x * kWarps + warp;
    if (wg >= nseg) return;
    const uint32_t item0 = (nseg - 1 - wg) * 32;
    const int nitems = (n - item0 < 32) ? (int)(n - item0) : 32;
    const bool live = lane < nitems;
    const uint32_t i = perm[item0 + (live ? lane : 0)];
    const uint2 d = live ? desc[i] : make_uint2(0, 0);
    const uint32_t len = d.x, out_len = d.y & 0x7fffffffu;
    const uint8_t* src = in + (len ? (offsets[i] - base) * 32 : 0);
    uint8_t* dst = out + (len ? (out_offsets[i] - obase) * 32 : 0);
    sponge_varlen_lane<true>(stage[warp], lane, false, tags + (size_t)i * 32, src, dst, len, out_len, (d.y >> 31) != 0);
}

// The lane-split loop of the variable-length digest kernels (five threads per item, hades_permute_coop), shared as
// sponge_varlen_lane is.  Every thread runs the warp's largest step count (the permutation's shuffles span the warp); a
// group past its own last step only idles.
template <bool kMixed>
__device__ __forceinline__ void sponge_varlen_coop(const LaneSplit& ls, bool live, const double (&crow)[5], const uint8_t* tag,
                                                   const uint8_t* src, uint8_t* dst, uint32_t len, uint32_t out_len, bool trunc) {
    const uint32_t nin = (len + 3) / 4, nout = (out_len + 3) / 4;
    const uint32_t steps = len ? nin + nout : 0u;
    const uint32_t wsteps = __reduce_max_sync(0xffffffffu, steps);
    uint32_t s[8];
    if (ls.li == 0) {
        load_fr(s, tag);
    } else {
#pragma unroll
        for (int w = 0; w < 8; ++w) s[w] = 0u;
        if (live && len == 0)                                    // rejected: a zero row
            for (uint32_t q = (uint32_t)ls.li - 1; q < out_len; q += 4) store_fr(dst + (size_t)q * 32, s);
    }
#pragma unroll 1
    for (uint32_t step = 0; step < wsteps; ++step) {
        if (step > 0) hades_permute_coop(s, ls.li, ls.g0, crow);
        if (step < nin) {
            const uint32_t q = 4 * step + (uint32_t)ls.li - 1;   // li == 0 wraps to a huge value -> no absorb
            if (ls.li >= 1 && q < len) {
                uint32_t v[8], t[8];
                load_fr(v, src + (size_t)q * 32);
                fr_add_mod(t, s, v);
#pragma unroll
                for (int w = 0; w < 8; ++w) s[w] = t[w];
            }
        } else if (step < steps) {
            const uint32_t q = 4 * (step - nin) + (uint32_t)ls.li - 1;
            if (ls.li >= 1 && q < out_len) {
                if (kMixed && trunc) {
                    uint32_t v[8];
                    fr_to_canonical(v, s);
                    v[7] &= 0x03ffffffu;                         // TRUNCATION_MASK, src/hash.rs:167-172
                    store_fr(dst + (size_t)q * 32, v);
                } else {
                    store_fr(dst + (size_t)q * 32, s);
                }
            }
        }
    }
}

// the same for small batches: five threads per item (hades_permute_coop), as k_sponge_digest_coop
__global__ void __launch_bounds__(kThreads) k_sponge_digest_varlen_coop(const uint8_t* __restrict__ tags,
                                                                        const uint8_t* __restrict__ in, uint64_t base,
                                                                        const uint64_t* __restrict__ offsets,
                                                                        const uint32_t* __restrict__ lens,
                                                                        const uint32_t* __restrict__ perm, uint32_t n,
                                                                        uint8_t* __restrict__ out, uint32_t out_len) {
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);
    const uint32_t len = live ? lens[ls.item] : 0u;
    const uint32_t i = live ? perm[ls.item] : 0u;
    const uint8_t* src = in + (len ? (offsets[i] - base) * 32 : 0);
    uint8_t* dst = out + (size_t)i * out_len * 32;
    sponge_varlen_coop<false>(ls, live, crow, tags + (size_t)len * 32, src, dst, len, out_len, false);
}

// k_sponge_digest_mixed for small batches: five threads per item, as k_sponge_digest_varlen_coop
__global__ void __launch_bounds__(kThreads) k_sponge_digest_mixed_coop(const uint8_t* __restrict__ tags,
                                                                       const uint2* __restrict__ desc,
                                                                       const uint8_t* __restrict__ in, uint64_t base,
                                                                       const uint64_t* __restrict__ offsets, uint64_t obase,
                                                                       const uint64_t* __restrict__ out_offsets,
                                                                       const uint32_t* __restrict__ perm, uint32_t n,
                                                                       uint8_t* __restrict__ out) {
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);
    const uint32_t i = live ? perm[ls.item] : 0u;
    const uint2 d = live ? desc[i] : make_uint2(0, 0);
    const uint32_t len = d.x, out_len = d.y & 0x7fffffffu;
    const uint8_t* src = in + (len ? (offsets[i] - base) * 32 : 0);
    uint8_t* dst = out + (len ? (out_offsets[i] - obase) * 32 : 0);
    sponge_varlen_coop<true>(ls, false, crow, tags + (size_t)i * 32, src, dst, len, out_len, (d.y >> 31) != 0);
}

// ---- variable-length encrypt / decrypt batches (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen) ---------------
// Item i reads src[offsets[i] - base, offsets[i+1] - base) and writes its output from dst[offsets[i] - offsets[0] + i]
// (encrypt: L + 1 cipher scalars) or dst[offsets[i] - offsets[0] - i] (decrypt: L message scalars), i.e. the input CSR
// with every item one scalar longer / shorter, packed from 0.  tags[L] is the tag of p252_encryption_tag(L) (tags[0] = 0,
// unused); secret_uv / nonce / ok are indexed by i.  The items come sorted by message length L (lens; 0 = rejected by
// k_varlen_keys<1|2>, which bounds every address below) with their indices (perm).
//
// k_crypt_varlen: k_crypt over the sorted order, one thread per item.  Every lane carries its own tag, step count
// 2*ceil(L/4), last-chunk widths and base addresses; the loop runs to the warp's largest step count and a lane past its
// own last step neither permutes nor touches memory.  A rejected item writes nothing (decrypt: ok = 0).  Warps take the
// sorted segments from the end, so the longest items start first.  4 resident blocks per SM (128 registers): at
// kMinBlocks' 96 the per-lane bookkeeping spills.
template <bool kDecrypt>
__global__ void __launch_bounds__(kThreads, 4) k_crypt_varlen(const uint8_t* __restrict__ tags, const uint8_t* __restrict__ src,
                                                              uint64_t base, const uint64_t* __restrict__ offsets,
                                                              const uint32_t* __restrict__ lens, const uint32_t* __restrict__ perm,
                                                              uint32_t n, const uint8_t* __restrict__ secret_uv,
                                                              const uint8_t* __restrict__ nonce, uint8_t* dst,
                                                              uint8_t* __restrict__ ok, unsigned long long* __restrict__ n_failed) {
    P252_STAGE_TABLES
    const int lane = threadIdx.x & 31;
    const uint32_t nseg = (n + 31) / 32;
    const uint32_t wg = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (wg >= nseg) return;
    const uint32_t k = (nseg - 1 - wg) * 32 + lane;
    const bool live = k < n;
    const uint32_t L = live ? lens[k] : 0u;
    const uint32_t i = live ? perm[k] : 0u;
    const uint64_t a = L ? offsets[i] : 0;
    const uint64_t o = L ? (kDecrypt ? a - offsets[0] - i : a - offsets[0] + i) : 0;
    const uint8_t* srci = src + (L ? (a - base) * 32 : 0);
    uint8_t* dsti = dst + o * 32;
    const uint8_t* msgi = kDecrypt ? dsti : srci;        // the plaintext, wherever it lives

    uint32_t s[5][8];
    load_fr(s[0], tags + (size_t)L * 32);
#pragma unroll
    for (int w = 0; w < 8; ++w) s[1][w] = s[2][w] = s[3][w] = s[4][w] = 0;
    if (L) {
        load_fr(s[1], secret_uv + (size_t)i * 64);       // Absorb(2): u, v added to zero
        load_fr(s[2], secret_uv + (size_t)i * 64 + 32);
        load_fr(s[3], nonce + (size_t)i * 32);           // Absorb(1)
    }
    const uint32_t nk = (L + 3) / 4, steps = 2 * nk;
    const uint32_t wsteps = __reduce_max_sync(0xffffffffu, steps);
    bool good = true;
#pragma unroll 1
    for (uint32_t step = 0; step < wsteps; ++step) {
        if (step >= steps) continue;
        hades_permute(s, (step + 1 == steps) ? 0x2u : 0x1fu P252_TAB_PASS);   // last: only the Squeeze(1) lane is read
        if (step < nk) {
            // Squeeze chunk `step` of the keystream and emit cipher (or recovered message)
            const uint32_t left = L - 4 * step;
            const int nscal = left < 4 ? (int)left : 4;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t x[8], y[8];
                    load_fr(x, srci + (size_t)(4 * step + q) * 32);
                    if (kDecrypt)
                        fr_sub_mod(y, x, s[1 + q]);      // Encryption::subtract
                    else
                        fr_add_mod(y, x, s[1 + q]);      // Safe::add
                    store_fr(dsti + (size_t)(4 * step + q) * 32, y);
                }
            }
        }
        if (step + 1 >= nk && step + 1 < steps) {
            // Absorb(L) chunk c of the plaintext: chunk 0 right after the last squeeze, chunk c > 0 one permutation later each
            const uint32_t c = step + 1 - nk;
            const uint32_t left = L - 4 * c;
            const int nscal = left < 4 ? (int)left : 4;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < nscal) {
                    uint32_t x[8], t[8];
                    if (kDecrypt)
                        load_fr_rw(x, msgi + (size_t)(4 * c + q) * 32);
                    else
                        load_fr(x, msgi + (size_t)(4 * c + q) * 32);
                    fr_add_mod(t, s[1 + q], x);
#pragma unroll
                    for (int w = 0; w < 8; ++w) s[1 + q][w] = t[w];
                }
            }
        }
        if (step + 1 == steps) {
            // Squeeze(1): authentication element
            if (kDecrypt) {
                uint32_t x[8];
                load_fr(x, srci + (size_t)L * 32);
#pragma unroll
                for (int w = 0; w < 8; ++w) good = good && (x[w] == s[1][w]);   // Encryption::is_equal
            } else {
                store_fr(dsti + (size_t)L * 32, s[1]);
            }
        }
    }
    if (kDecrypt) {
        if (live) ok[i] = (L && good) ? 1 : 0;
        if (L && !good) {                                 // Error::DecryptionFailed: release nothing
            const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t q = 0; q < L; ++q) store_fr(dsti + (size_t)q * 32, zero);
        }
        // rejected items are not failures (k_varlen_keys counted them)
        if (n_failed) warp_count_full(n_failed, L && !good);
    }
}

// the same for small batches: five threads per item (hades_permute_coop), as k_sponge_digest_varlen_coop.  Thread li of
// a group owns state lane li: lane 0 the tag, lanes 1..3 u, v, nonce; rate thread li adds / subtracts, stores and absorbs
// message scalar 4*c + li - 1 of chunk c, and thread 1 holds the Squeeze(1) lane.  Every thread runs the warp's largest
// step count (the permutation's shuffles span the warp); a group past its own last step only idles.  Decrypt: thread 1's
// authentication result is shuffled to its group before any thread zeroes its message scalars.
template <bool kDecrypt>
__global__ void __launch_bounds__(kThreads) k_crypt_varlen_coop(const uint8_t* __restrict__ tags, const uint8_t* __restrict__ src,
                                                                uint64_t base, const uint64_t* __restrict__ offsets,
                                                                const uint32_t* __restrict__ lens,
                                                                const uint32_t* __restrict__ perm, uint32_t n,
                                                                const uint8_t* __restrict__ secret_uv,
                                                                const uint8_t* __restrict__ nonce, uint8_t* dst,
                                                                uint8_t* __restrict__ ok, unsigned long long* __restrict__ n_failed) {
    const LaneSplit ls;
    if (ls.idle(n)) return;
    const bool live = ls.live(n);
    double crow[5];
    ls.mds_row(crow);
    const uint32_t L = live ? lens[ls.item] : 0u;
    const uint32_t i = live ? perm[ls.item] : 0u;
    const uint64_t a = L ? offsets[i] : 0;
    const uint64_t o = L ? (kDecrypt ? a - offsets[0] - i : a - offsets[0] + i) : 0;
    const uint8_t* srci = src + (L ? (a - base) * 32 : 0);
    uint8_t* dsti = dst + o * 32;
    const uint8_t* msgi = kDecrypt ? dsti : srci;
    uint32_t s[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) s[w] = 0u;
    if (ls.li == 0)
        load_fr(s, tags + (size_t)L * 32);
    else if (L && ls.li <= 2)
        load_fr(s, secret_uv + (size_t)i * 64 + (size_t)(ls.li - 1) * 32);
    else if (L && ls.li == 3)
        load_fr(s, nonce + (size_t)i * 32);
    const uint32_t nk = (L + 3) / 4, steps = 2 * nk;
    const uint32_t wsteps = __reduce_max_sync(0xffffffffu, steps);
    bool good = true;
#pragma unroll 1
    for (uint32_t step = 0; step < wsteps; ++step) {
        hades_permute_coop(s, ls.li, ls.g0, crow);
        const uint32_t q = 4 * step + (uint32_t)ls.li - 1;       // li == 0 wraps to a huge value -> no memory access
        if (step < nk && ls.li >= 1 && q < L) {                  // squeeze chunk `step`: emit cipher / message scalar q
            uint32_t x[8], y[8];
            load_fr(x, srci + (size_t)q * 32);
            if (kDecrypt)
                fr_sub_mod(y, x, s);
            else
                fr_add_mod(y, x, s);
            store_fr(dsti + (size_t)q * 32, y);
        }
        if (step + 1 >= nk && step + 1 < steps) {                // absorb plaintext chunk c (this thread's own stores)
            const uint32_t qa = 4 * (step + 1 - nk) + (uint32_t)ls.li - 1;
            if (ls.li >= 1 && qa < L) {
                uint32_t x[8], t[8];
                if (kDecrypt)
                    load_fr_rw(x, msgi + (size_t)qa * 32);
                else
                    load_fr(x, msgi + (size_t)qa * 32);
                fr_add_mod(t, s, x);
#pragma unroll
                for (int w = 0; w < 8; ++w) s[w] = t[w];
            }
        }
        if (step + 1 == steps && ls.li == 1) {                   // Squeeze(1): authentication element
            if (kDecrypt) {
                uint32_t x[8];
                load_fr(x, srci + (size_t)L * 32);
#pragma unroll
                for (int w = 0; w < 8; ++w) good = good && (x[w] == s[w]);
            } else {
                store_fr(dsti + (size_t)L * 32, s);
            }
        }
    }
    if (kDecrypt) {
        good = __shfl_sync(0xffffffffu, good, ls.g0 + 1);        // the group's verdict, before anyone zeroes
        if (live && ls.li == 0) ok[i] = (L && good) ? 1 : 0;
        if (L && !good && ls.li >= 1) {
            const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t q = (uint32_t)ls.li - 1; q < L; q += 4) store_fr(dsti + (size_t)q * 32, zero);
        }
        if (n_failed) warp_count_full(n_failed, ls.li == 0 && L && !good);
    }
}

// ---- host-callable launchers -------------------------------------------------------------------
static inline FrArg to_arg(const uint64_t tag[4]) {
    FrArg a;
    for (int k = 0; k < 4; ++k) {
        a.l[2 * k] = (uint32_t)tag[k];
        a.l[2 * k + 1] = (uint32_t)(tag[k] >> 32);
    }
    return a;
}

// A launcher's untyped buffer (void* or const void*) becomes the kernel's typed pointer parameter; every other argument
// is passed as it is, so a const buffer still needs a visible const_cast to reach a non-const parameter.
template <class P, class A>
static inline P kernel_arg(A a) { return a; }
template <class P>
static inline P kernel_arg(void* a) { return static_cast<P>(a); }
template <class P>
static inline P kernel_arg(const void* a) { return static_cast<P>(a); }

// Launches kernel k with `grid` blocks of `threads` threads on stream st and returns the launch's status.  An empty
// grid (an empty batch) launches nothing and returns cudaSuccess.
template <class... P, class... A>
static cudaError_t launch_grid(void (*k)(P...), unsigned grid, unsigned threads, cudaStream_t st, A... a) {
    if (grid == 0) return cudaSuccess;
    k<<<grid, threads, 0, st>>>(kernel_arg<P>(a)...);
    return cudaGetLastError();
}

// The same for n items, one per thread: ceil(n / threads) blocks
template <class... P, class... A>
static cudaError_t launch(void (*k)(P...), size_t n, unsigned threads, cudaStream_t st, A... a) {
    return launch_grid(k, (unsigned)((n + threads - 1) / threads), threads, st, a...);
}

// lane-split kernels: kCoopItemsPerWarp items per warp
static inline unsigned coop_grid(size_t n) {
    return (unsigned)(((n + kCoopItemsPerWarp - 1) / kCoopItemsPerWarp + kWarps - 1) / kWarps);
}
static inline uint32_t log2_arity(int arity) { return arity == 4 ? 2u : 1u; }
// digest batches from this size on (>= 7 waves of 256-thread blocks) take the 256 x 2 launch shape
#ifndef P252_WIDE_SHAPE_MIN
#define P252_WIDE_SHAPE_MIN (1u << 19)
#endif
constexpr size_t kWideShapeMinItems = P252_WIDE_SHAPE_MIN;

// Default for p252_set_small_batch_max: batches up to this many items take the lane-split kernel (latency-bound
// regime): one lane-split warp (6 items) per SM sub-partition, i.e. 3168 items on a 132-SM H100.  The environment
// variable P252_COOP_MAX overrides it (0 disables the lane-split path).
size_t coop_max_items(int sm_count) {
    const char* e = getenv("P252_COOP_MAX");
    return e ? (size_t)strtoull(e, nullptr, 10) : (size_t)sm_count * 4 * kCoopItemsPerWarp;
}

cudaError_t launch_permute(void* states, size_t n, bool dense, size_t coop_max, cudaStream_t st) {
    if (!dense && n <= coop_max) return launch_grid(k_permute_coop, coop_grid(n), kThreads, st, states, n);
    if (dense) return launch(k_permute<true>, n, kThreads, st, states, n);
    if (n >= kWideShapeMinItems) return launch(k_permute<false, 256, 2>, n, 256, st, states, n);
    return launch(k_permute<false>, n, kThreads, st, states, n);
}

cudaError_t launch_digest(const uint64_t tag[4], const void* in, size_t n, uint32_t in_len, void* out,
                          uint32_t out_len, bool truncate, size_t coop_max, cudaStream_t st) {
    const FrArg t = to_arg(tag);
    if (!truncate && n <= coop_max)
        return launch_grid(k_sponge_digest_coop, coop_grid(n), kThreads, st, t, in, n, in_len, out, out_len);
    if (truncate) return launch(k_sponge_digest<true>, n, kThreads, st, t, in, n, in_len, out, out_len);
    if (n >= kWideShapeMinItems) return launch(k_sponge_digest<false, 256, 2>, n, 256, st, t, in, n, in_len, out, out_len);
    return launch(k_sponge_digest<false>, n, kThreads, st, t, in, n, in_len, out, out_len);
}

// ---- wire format: canonical 32-byte little-endian <-> BlsScalar.0 (Montgomery limbs) ---------------------
// BlsScalar::from_bytes / to_bytes (used at src/hades.rs:94-105,131 and
// src/hades/round_constants.rs:64-68).  Elementwise, 32 B in + 32 B out per scalar: the one HBM-bound kernel.
template <bool kFromBytes>
__global__ void __launch_bounds__(256) k_convert(const uint8_t* __restrict__ in, size_t n, uint8_t* __restrict__ out,
                                                 uint8_t* __restrict__ ok) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[8], r[8];
    load_fr(x, in + i * 32);
    if (kFromBytes) {
        const bool valid = fr_is_canonical(x);               // from_bytes rejects values >= p
        fr_from_canonical(r, x);
        if (!valid) {
#pragma unroll
            for (int k = 0; k < 8; ++k) r[k] = 0;
        }
        if (ok) ok[i] = valid ? 1 : 0;
    } else {
        fr_to_canonical(r, x);
    }
    store_fr(out + i * 32, r);
}

cudaError_t launch_convert(const void* in, size_t n, void* out, uint8_t* ok, bool from_bytes, cudaStream_t st) {
    if (from_bytes) return launch(k_convert<true>, n, 256, st, in, n, out, ok);
    return launch(k_convert<false>, n, 256, st, in, n, out, nullptr);
}

cudaError_t launch_encrypt(const uint64_t tag[4], const void* msg, size_t n, uint32_t L, const void* secret_uv,
                           const void* nonce, void* cipher, cudaStream_t st) {
    return launch(k_crypt<false>, n, kThreads, st, to_arg(tag), msg, n, L, secret_uv, nonce, cipher, nullptr, nullptr);
}

cudaError_t launch_decrypt(const uint64_t tag[4], const void* cipher, size_t n, uint32_t L, const void* secret_uv,
                           const void* nonce, void* msg, uint8_t* ok, unsigned long long* n_failed, cudaStream_t st) {
    return launch(k_crypt<true>, n, kThreads, st, to_arg(tag), cipher, n, L, secret_uv, nonce, msg, ok, n_failed);
}

// ---- JubJub operands: point rows, masks and the projective comparison -----------------------------------------------
// Every JubJub kernel runs the same instructions for every item (DESIGN.md §4): an invalid operand is replaced by the
// identity or by zero, never skipped.  None of these helpers branches on or indexes by an operand's value; a mask m is
// all ones or all zeros.

// Loads the point row at p into (u, v) and returns whether it is a curve point with u, v < p.  Substitutes nothing.
__device__ __forceinline__ bool load_curve_point(uint32_t (&u)[8], uint32_t (&v)[8], const uint8_t* p) {
    load_fr(u, p);
    load_fr(v, p + 32);
    return fr_is_canonical(u) & fr_is_canonical(v) & jj::on_curve(u, v);
}

// Loads the point row at p into (u, v) and returns whether u, v < p (no curve check).  A pair with a coordinate >= p is
// replaced so that it enters no product: by the identity (0, 1) if kIdentity, by (0, 0) otherwise.
template <bool kIdentity>
__device__ __forceinline__ bool load_canonical_point(uint32_t (&u)[8], uint32_t (&v)[8], const uint8_t* p) {
    load_fr(u, p);
    load_fr(v, p + 32);
    uint32_t one[8];
    jj::set_one(one);
    const bool canon = fr_is_canonical(u) & fr_is_canonical(v);
    const uint32_t mc = 0u - (uint32_t)canon;
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] &= mc, v[k] = (v[k] & mc) | (kIdentity ? one[k] & ~mc : 0u);
    return canon;
}

// (u, v) = m ? (u, v) : the identity (0, 1)
__device__ __forceinline__ void mask_point(uint32_t (&u)[8], uint32_t (&v)[8], uint32_t m) {
    uint32_t one[8];
    jj::set_one(one);
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] &= m, v[k] = (v[k] & m) | (one[k] & ~m);
}

// (u, v) &= m, then stores (u, v) as the 64-byte point row at p: a zeroed row where m is zero
__device__ __forceinline__ void store_masked_point(uint8_t* p, uint32_t (&u)[8], uint32_t (&v)[8], uint32_t m) {
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] &= m, v[k] &= m;
    store_fr(p, u);
    store_fr(p + 32, v);
}

// Whether the affine (u, v) is the point t, compared projectively (u Z == X and v Z == Y): no inversion
__device__ __forceinline__ bool equals_affine(const uint32_t (&u)[8], const uint32_t (&v)[8], const jj::Ext& t) {
    uint32_t x[8], y[8];
    jj::fmul(x, u, t.Z);
    jj::fmul(y, v, t.Z);
    return jj::feq(x, t.X) & jj::feq(y, t.Y);
}

// ---- JubJub key exchange (dhke(secret, public) = [s] public, JubJubAffine out) -------------------------------------
// One thread per item, 2819 products (jubjub_device.cuh).  Item i reads secret[sb ? 0 : i] (canonical 4 x u64) and
// pub[pb ? 0 : i] ((u, v), Montgomery); valid iff s < r_J, u, v < p and (u, v) on the curve.  An invalid item runs the
// same schedule on (0, identity), so the instruction stream is the same for every item, and writes (0, 0), ok = 0.
__global__ void __launch_bounds__(kThreads, 3) k_dhke(const uint8_t* __restrict__ secret, bool sb, const uint8_t* __restrict__ pub,
                                                   bool pb, size_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ ok,
                                                   unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8], u[8], v[8];
    load_fr(s, secret + (sb ? 0 : i) * 32);
    load_fr(u, pub + (pb ? 0 : i) * 64);
    load_fr(v, pub + (pb ? 0 : i) * 64 + 32);
    const bool valid = jj::below_order(s) & fr_is_canonical(u) & fr_is_canonical(v) & jj::on_curve(u, v);
    const uint32_t m = 0u - (uint32_t)valid;
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] &= m;
    mask_point(u, v, m);
    uint32_t ou[8], ov[8];
    jj::scalar_mul(ou, ov, s, u, v);
    store_masked_point(out + i * 64, ou, ov, m);
    ok[i] = valid ? 1 : 0;
    if (n_invalid) warp_count(n_invalid, !valid);
}

// After a fused crypt: every item whose key exchange was invalid (valid[i] == 0) gets ok[i] = 0 and a zeroed output row
// of `row` scalars.  count (may be null): encrypt adds the invalid items; decrypt adds those k_crypt did not already
// count as authentication failures, so that each failed item is counted once.
__global__ void __launch_bounds__(256) k_dhke_fix(bool decrypt, const uint8_t* __restrict__ valid, size_t n, uint8_t* out,
                                                  uint32_t row, uint8_t* ok, unsigned long long* __restrict__ count) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool bad = valid[i] == 0;
    bool hit = bad;
    if (decrypt) hit = bad && ok[i] != 0;
    if (bad) {
        ok[i] = 0;
        const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (uint32_t k = 0; k < row; ++k) store_fr(out + (i * row + k) * 32, zero);
    } else if (!decrypt) {
        ok[i] = 1;
    }
    if (count) warp_count(count, hit);
}

cudaError_t launch_dhke(const void* secret, bool secret_bcast, const void* pub, bool pub_bcast, size_t n, void* shared_uv,
                        uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_dhke, n, kThreads, st, secret, secret_bcast, pub, pub_bcast, n, shared_uv, ok, n_invalid);
}

cudaError_t launch_dhke_fix(bool decrypt, const uint8_t* valid, size_t n, void* out, uint32_t row, uint8_t* ok,
                            unsigned long long* count, cudaStream_t st) {
    return launch(k_dhke_fix, n, 256, st, decrypt, valid, n, out, row, ok, count);
}

// ---- fixed-base JubJub scalar multiplication (out = [s] B for one base B of the whole batch) -------------------------
static_assert(kFixedBaseTableBytes == jj::kFbTableWords * sizeof(uint4), "fixed-base table size of kernels.h");
struct FixedBase {               // the base (u, v), Montgomery, passed by value: the table build reads no host memory
    uint32_t uv[16];
};

// One thread per table entry (w, j): 512 threads, entry e = 8 w + j - 1 at table + 6 e (jubjub_device.cuh).
__global__ void __launch_bounds__(128) k_fixed_base_table(FixedBase b, uint4* __restrict__ table) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= jj::kFbWindows * jj::kFbEntries) return;
    uint32_t u[8], v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] = b.uv[k], v[k] = b.uv[8 + k];
    jj::fixed_base_entry(table + e * jj::kFbEntryWords, u, v, e / jj::kFbEntries, e % jj::kFbEntries + 1);
}

// One thread per item, 866 products.  Item i reads secret[i] (canonical 4 x u64); valid iff s < r_J.  An invalid item runs
// the same schedule on s = 0 and writes (0, 0), ok = 0.  Every lane of a warp reads the same table address at the same
// time (the window and entry counters are public), so the read-only path serves each load as one broadcast.
__global__ void __launch_bounds__(kThreads, 3) k_fixed_base(const uint8_t* __restrict__ secret, size_t n,
                                                         const uint4* __restrict__ table, uint8_t* __restrict__ out,
                                                         uint8_t* __restrict__ ok, unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    load_fr(s, secret + i * 32);
    const bool valid = jj::below_order(s);
    const uint32_t m = 0u - (uint32_t)valid;
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] &= m;
    uint32_t ou[8], ov[8];
    jj::fixed_base_mul<true>(ou, ov, s, table);
    store_masked_point(out + i * 64, ou, ov, m);
    ok[i] = valid ? 1 : 0;
    if (n_invalid) warp_count(n_invalid, !valid);
}

cudaError_t launch_fixed_base_table(const uint64_t base_uv[8], void* table, cudaStream_t st) {
    FixedBase b;
    for (int k = 0; k < 8; ++k) b.uv[2 * k] = (uint32_t)base_uv[k], b.uv[2 * k + 1] = (uint32_t)(base_uv[k] >> 32);
    return launch(k_fixed_base_table, jj::kFbWindows * jj::kFbEntries, 128, st, b, table);
}

cudaError_t launch_fixed_base(const void* secret, size_t n, const void* table, void* out_uv, uint8_t* ok,
                              unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_fixed_base, n, kThreads, st, secret, n, table, out_uv, ok, n_invalid);
}

// ---- stealth addresses: note_pk = [h] G + B, h = hash([r] A) = hash([a] R) (jubjub_device.cuh) ------------------------
struct NielsArg {                // the receiver's B in Niels form (v - u, v + u, 2d u v), Montgomery, passed by value
    uint32_t w[24];
};

// *counter += the lanes of the warp with `hit`: one atomic per warp whatever the flags, so that not even the count's
// bookkeeping branches on an item's result
__device__ __forceinline__ void warp_count_every(unsigned long long* counter, bool hit) {
    const unsigned act = __activemask();
    const unsigned b = __ballot_sync(act, hit);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicAdd(counter, (unsigned long long)__popc(b));
}

// One thread per item.  h[i]: the truncated digest of the item's shared point (raw limbs < 2^250); valid[i]: the validity
// k_dhke gave that point.  Every item runs the same schedule: invalid operands are replaced by the identity or zero.
//   kOwns (the receiver, 456 products): pk = the note keys (read); flag[i] = owned = valid[i], both note_pk coordinates
//     < p and note_pk == [h] G + nb, compared projectively.  cnt_a += owned, cnt_b += invalid.
//   derive (the sender, 879 products): B_uv[bb ? 0 : i] is B (read); pk = the note keys (written); flag[i] = ok = valid[i]
//     and B a curve point with u, v < p.  An item with ok = 0 gets a zeroed note_pk row and a zeroed R row (R as written
//     by k_fixed_base).  cnt_a += invalid.
template <bool kOwns>
__global__ void __launch_bounds__(kThreads, 3) k_stealth(const uint8_t* __restrict__ h, size_t n, const uint4* __restrict__ table,
                                                      NielsArg nb, const uint8_t* __restrict__ B_uv, bool bb,
                                                      const uint8_t* __restrict__ valid, uint8_t* pk, uint8_t* R_uv,
                                                      uint8_t* __restrict__ flag, unsigned long long* __restrict__ cnt_a,
                                                      unsigned long long* __restrict__ cnt_b) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    // The point operand is loaded twice (derive: its check runs before [h] G, its Niels form after) so that during the
    // 64 windows of [h] G nothing but the scalar and a flag is live.  Coordinates >= p enter no product: they are
    // replaced first (derive: by the identity (0, 1)).
    uint32_t u[8], v[8];
    const uint8_t* pt = kOwns ? pk + i * 64 : B_uv + (bb ? 0 : i) * 64;
    bool good = valid[i] != 0;
    if (!kOwns) {
        const bool canon = load_canonical_point<true>(u, v, pt);
        good &= canon & jj::on_curve(u, v);
    }
    jj::Ext t, r;
    {
        uint32_t s[8];
        load_fr(s, h + i * 32);
        jj::fixed_base_ext<true, true>(t, s, table);
    }
    const bool canon = load_canonical_point<!kOwns>(u, v, pt);
    jj::Niels q;
    if (kOwns) {
#pragma unroll
        for (int k = 0; k < 8; ++k) q.ymx[k] = nb.w[k], q.ypx[k] = nb.w[8 + k], q.kt[k] = nb.w[16 + k];
        good &= canon;
    } else {
        mask_point(u, v, 0u - (uint32_t)good);   // an item that is not valid adds the identity: B is on the curve
        jj::to_niels(q, u, v);
    }
    jj::madd<false>(r, t, q);
    if (kOwns) {
        const bool owned = good & equals_affine(u, v, r);
        flag[i] = owned ? 1 : 0;
        if (cnt_a) warp_count_every(cnt_a, owned);
        if (cnt_b) warp_count_every(cnt_b, !good);
    } else {
        uint32_t zi[8], ou[8], ov[8];
        jj::inverse(zi, r.Z);
        jj::fmul(ou, r.X, zi);
        jj::fmul(ov, r.Y, zi);
        const uint32_t m = 0u - (uint32_t)good;
        uint32_t ru[8], rv[8];
        load_fr_rw(ru, R_uv + i * 64);
        load_fr_rw(rv, R_uv + i * 64 + 32);
        store_masked_point(pk + i * 64, ou, ov, m);
        store_masked_point(R_uv + i * 64, ru, rv, m);
        flag[i] = good ? 1 : 0;
        if (cnt_a) warp_count_every(cnt_a, !good);
    }
}

cudaError_t launch_stealth_owns(const void* h, size_t n, const void* table, const uint64_t b_niels[12], const void* note_pk,
                                const uint8_t* valid, uint8_t* owned, unsigned long long* n_owned,
                                unsigned long long* n_invalid, cudaStream_t st) {
    NielsArg nb;
    for (int k = 0; k < 12; ++k) nb.w[2 * k] = (uint32_t)b_niels[k], nb.w[2 * k + 1] = (uint32_t)(b_niels[k] >> 32);
    return launch(k_stealth<true>, n, kThreads, st, h, n, table, nb, nullptr, false, valid, const_cast<void*>(note_pk), nullptr,
                  owned, n_owned, n_invalid);
}

cudaError_t launch_stealth_derive(const void* h, size_t n, const void* table, const void* B_uv, bool B_bcast,
                                  const uint8_t* valid, void* R_uv, void* note_pk, uint8_t* ok, unsigned long long* n_invalid,
                                  cudaStream_t st) {
    return launch(k_stealth<false>, n, kThreads, st, h, n, table, NielsArg{}, B_uv, B_bcast, valid, note_pk, R_uv, ok, n_invalid,
                  nullptr);
}

// ---- note nullifiers: the digest rows [pk'.u, pk'.v, pos] of pk' = [(h + b) mod r_J] G' (jubjub_device.cuh) -------------
// One thread per item, kProductsPerNullifierKey products, after k_dhke (valid[i]: a < r_J and R a curve point) and the
// truncated digest (h[i] < 2^250 < r_J).  b[bb ? 0 : i] (canonical 4 x u64) must be < r_J: valid[i] &= b < r_J, and an
// out-of-range b enters the sum as 0.  rows[i] = [pk'.u, pk'.v, Montgomery(pos[i])] (96 bytes) for every item; the caller
// zeroes the outputs of invalid ones after the digest (launch_dhke_fix).  a, b and note_sk are secret: every item runs the
// same schedule, the validity is a mask, and the table reads are masked selects, as in k_fixed_base.
__global__ void __launch_bounds__(kThreads, 3) k_nullifier_key(const uint8_t* __restrict__ h, const uint8_t* __restrict__ b,
                                                            bool bb, const uint64_t* __restrict__ pos, size_t n,
                                                            const uint4* __restrict__ table, uint8_t* __restrict__ rows,
                                                            uint8_t* valid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8], t[8];
    load_fr(s, h + i * 32);
    load_fr(t, b + (bb ? 0 : i) * 32);
    const bool in_range = jj::below_order(t);
    const uint32_t m = 0u - (uint32_t)in_range;
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] &= m;
    uint32_t sk[8];
    jj::order_add(sk, s, t);
    uint32_t ou[8], ov[8];
    jj::fixed_base_mul<true>(ou, ov, sk, table);
    uint32_t c[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pm[8];
    const uint64_t p = pos[i];
    c[0] = (uint32_t)p, c[1] = (uint32_t)(p >> 32);
    fr_from_canonical(pm, c);
    store_fr(rows + i * 96, ou);
    store_fr(rows + i * 96 + 32, ov);
    store_fr(rows + i * 96 + 64, pm);
    valid[i] = (valid[i] != 0) & in_range ? 1 : 0;
}

cudaError_t launch_nullifier_key(const void* h, const void* b, bool b_bcast, const uint64_t* pos, size_t n, const void* table,
                                 void* rows, uint8_t* valid, cudaStream_t st) {
    return launch(k_nullifier_key, n, kThreads, st, h, b, b_bcast, pos, n, table, rows, valid);
}

// ---- Schnorr signatures: u = r - c sk mod r_J; [u] G + [c] PK == R, c = challenge(R, m) (jubjub_device.cuh) -----------
// The digest's input rows [R.u, R.v, m]: a value >= p is written as 0, and flag[i] = (and_flag ? flag[i] : 1) and all three
// values < p.  Sign: flag is ok (r < r_J from k_fixed_base), R as k_fixed_base wrote it; verify: flag is the item's
// validity, R the caller's.  Public data only.
__global__ void __launch_bounds__(256) k_schnorr_pack(const uint8_t* R_uv, const uint8_t* __restrict__ msg, size_t n,
                                                      uint8_t* __restrict__ rows, uint8_t* flag, bool and_flag) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[3][8];
    load_fr_rw(x[0], R_uv + i * 64);
    load_fr_rw(x[1], R_uv + i * 64 + 32);
    load_fr(x[2], msg + i * 32);
    bool good = !and_flag || flag[i] != 0;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const bool canon = fr_is_canonical(x[q]);
        const uint32_t m = 0u - (uint32_t)canon;
#pragma unroll
        for (int k = 0; k < 8; ++k) x[q][k] &= m;
        good &= canon;
        store_fr(rows + i * 96 + q * 32, x[q]);
    }
    flag[i] = good ? 1 : 0;
}

// Sign, one thread per item, after k_fixed_base (R rows, ok = r < r_J), k_schnorr_pack (ok &= m < p) and the truncated
// digest (c[i] < 2^250): ok[i] = ok[i] and sk < r_J; u[i] = (r - c sk) mod r_J (kOrderProductsPerSchnorrSign Montgomery
// products modulo r_J).  An item with ok = 0 runs the same code on r = sk = 0 and gets zeroed u and R rows; *n_invalid
// += invalid items.  sk and r are secret: every validity is a mask, and no branch or address depends on them.
__global__ void __launch_bounds__(kThreads, 3) k_schnorr_sign(const uint8_t* __restrict__ sk, bool sb, const uint8_t* __restrict__ r,
                                                           const uint8_t* __restrict__ c, size_t n, uint8_t* __restrict__ u_out,
                                                           uint8_t* R_uv, uint8_t* ok, unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8], k[8], e[8];
    load_fr(s, sk + (sb ? 0 : i) * 32);
    load_fr(k, r + i * 32);
    load_fr(e, c + i * 32);
    const bool good = (ok[i] != 0) & jj::below_order(s);
    const uint32_t m = 0u - (uint32_t)good;
#pragma unroll
    for (int q = 0; q < 8; ++q) s[q] &= m, k[q] &= m;
    uint32_t x[8], u[8];
    jj::order_mul(x, e, s);
    jj::order_sub(u, k, x);
    uint32_t ru[8], rv[8];
    load_fr_rw(ru, R_uv + i * 64);
    load_fr_rw(rv, R_uv + i * 64 + 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) u[q] &= m;
    store_fr(u_out + i * 32, u);
    store_masked_point(R_uv + i * 64, ru, rv, m);
    ok[i] = good ? 1 : 0;
    if (n_invalid) warp_count_every(n_invalid, !good);
}

// The single-key check [c] PK + [u] G == R of item i (PK = pk[pb ? 0 : i]), compared projectively
// (kProductsPerSchnorrVerify products), with public operands only: the variable-base walk of [c] PK reads one table entry per window at the digit's address
// (jj::scalar_mul_ext<true, ...>); k_dhke keeps the masked reads.  PK, then u, then R are loaded, each just before its
// use, so that across each walk little else is live.  good &= PK a curve point with u, v < p and u < r_J; an invalid
// operand is replaced by the identity or zero, so every item runs the same code.  Returns good and the equation.
__device__ __forceinline__ bool schnorr_check(const uint8_t* __restrict__ pk, bool pb, const uint8_t* __restrict__ u,
                                              const uint8_t* __restrict__ R_uv, const uint8_t* __restrict__ c, size_t i,
                                              const uint4* __restrict__ table, bool& good) {
    jj::Ext acc;
    {
        uint32_t x[8], y[8], one[8], e[8];
        load_fr(x, pk + (pb ? 0 : i) * 64);
        load_fr(y, pk + (pb ? 0 : i) * 64 + 32);
        const bool canon = fr_is_canonical(x) & fr_is_canonical(y);
        jj::set_one(one);
        const uint32_t mc = 0u - (uint32_t)canon;      // coordinates >= p enter no product
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] &= mc, y[k] = (y[k] & mc) | (one[k] & ~mc);
        const bool on = canon & jj::on_curve(x, y);
        good &= on;
        mask_point(x, y, 0u - (uint32_t)on);           // an off-curve PK is replaced by the identity
        load_fr(e, c + i * 32);
        jj::scalar_mul_ext<true, true>(acc, e, x, y);
    }
    jj::Ext t;
    {
        uint32_t s[8];
        load_fr(s, u + i * 32);
        const bool in_range = jj::below_order(s);
        good &= in_range;
        const uint32_t m = 0u - (uint32_t)in_range;
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] &= m;
        jj::fixed_base_from<true, false>(t, acc, s, table);
    }
    uint32_t ru[8], rv[8];
    load_fr(ru, R_uv + i * 64);
    load_fr(rv, R_uv + i * 64 + 32);
    const uint32_t m = 0u - (uint32_t)good;             // an invalid item's R may be >= p: it enters no product
#pragma unroll
    for (int k = 0; k < 8; ++k) ru[k] &= m, rv[k] &= m;
    return good & equals_affine(ru, rv, t);
}

// Verify, one thread per item, after k_schnorr_pack (valid[i]: R and m canonical) and the truncated digest (c[i]):
// verified[i] = valid[i], u < r_J, PK = pk[pb ? 0 : i] a curve point with u, v < p, and [c] PK + [u] G == R
// (schnorr_check).  cnt_ok += verified items, cnt_bad += invalid ones.
__global__ void __launch_bounds__(kThreads, 3) k_schnorr_verify(const uint8_t* __restrict__ pk, bool pb, const uint8_t* __restrict__ u,
                                                             const uint8_t* __restrict__ R_uv, const uint8_t* __restrict__ c,
                                                             const uint8_t* __restrict__ valid, size_t n,
                                                             const uint4* __restrict__ table, uint8_t* __restrict__ verified,
                                                             unsigned long long* __restrict__ cnt_ok,
                                                             unsigned long long* __restrict__ cnt_bad) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    bool good = valid[i] != 0;
    const bool ok = schnorr_check(pk, pb, u, R_uv, c, i, table, good);
    verified[i] = ok ? 1 : 0;
    if (cnt_ok) warp_count_every(cnt_ok, ok);
    if (cnt_bad) warp_count_every(cnt_bad, !good);
}

cudaError_t launch_schnorr_pack(const void* R_uv, const void* msg, size_t n, void* rows, uint8_t* flag, bool and_flag,
                                cudaStream_t st) {
    return launch(k_schnorr_pack, n, 256, st, R_uv, msg, n, rows, flag, and_flag);
}

cudaError_t launch_schnorr_sign(const void* sk, bool sk_bcast, const void* r, const void* c, size_t n, void* u_out, void* R_uv,
                                uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_schnorr_sign, n, kThreads, st, sk, sk_bcast, r, c, n, u_out, R_uv, ok, n_invalid);
}

cudaError_t launch_schnorr_verify(const void* pk, bool pk_bcast, const void* u, const void* R_uv, const void* c,
                                  const uint8_t* valid, size_t n, const void* table, uint8_t* verified,
                                  unsigned long long* n_verified, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_schnorr_verify, n, kThreads, st, pk, pk_bcast, u, R_uv, c, valid, n, table, verified, n_verified, n_invalid);
}

// ---- double-key Schnorr signatures over G and G': c = challenge2(R, R', m) (jubjub_device.cuh) -------------------------
// The digest's input rows [R.u, R.v, R'.u, R'.v, m] (160 bytes): a value >= p is written as 0, and flag[i] =
// (and_flag ? flag[i] : 1) and all five values < p.  Sign: flag is ok (r < r_J from k_fixed_base), R and R' as k_fixed_base
// wrote them; verify: flag is the item's validity, R and R' the caller's.  Public data only.
__global__ void __launch_bounds__(256) k_schnorr_pack_double(const uint8_t* R_uv, const uint8_t* Rp_uv,
                                                             const uint8_t* __restrict__ msg, size_t n,
                                                             uint8_t* __restrict__ rows, uint8_t* flag, bool and_flag) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[5][8];
    load_fr_rw(x[0], R_uv + i * 64);
    load_fr_rw(x[1], R_uv + i * 64 + 32);
    load_fr_rw(x[2], Rp_uv + i * 64);
    load_fr_rw(x[3], Rp_uv + i * 64 + 32);
    load_fr(x[4], msg + i * 32);
    bool good = !and_flag || flag[i] != 0;
#pragma unroll
    for (int q = 0; q < 5; ++q) {
        const bool canon = fr_is_canonical(x[q]);
        const uint32_t m = 0u - (uint32_t)canon;
#pragma unroll
        for (int k = 0; k < 8; ++k) x[q][k] &= m;
        good &= canon;
        store_fr(rows + i * 160 + q * 32, x[q]);
    }
    flag[i] = good ? 1 : 0;
}

// Sign, one thread per item, after k_fixed_base twice (R and R' rows, ok = r < r_J), k_schnorr_pack_double (ok &= m < p)
// and the truncated digest (c[i] < 2^250).  Plain: sk = key[kb ? 0 : i], ok[i] &= sk < r_J.  Note: key is b, h[i] the
// truncated digest of [a] R_note and valid[i] its validity from k_dhke; sk = (h + b) mod r_J with an out-of-range b entering
// as 0, ok[i] &= valid[i] and b < r_J, and pk'[i] = [sk] G' (table: the fixed-base table of G', kProductsPerFixedBase
// products).  u[i] = (r - c sk) mod r_J (kOrderProductsPerSchnorrSign products modulo r_J).  An item with ok = 0 runs the
// same code on r = sk = 0 and gets zeroed u, R, R' (and pk') rows; *n_invalid += invalid items.  The keys, r and note_sk
// are secret: every validity is a mask, the table reads are masked selects, and no branch or address depends on them.
template <bool Note>
__global__ void __launch_bounds__(kThreads, 3) k_schnorr_sign_double(const uint8_t* __restrict__ key, bool kb,
                                                                  const uint8_t* __restrict__ h,
                                                                  const uint8_t* __restrict__ valid,
                                                                  const uint8_t* __restrict__ r, const uint8_t* __restrict__ c,
                                                                  size_t n, const uint4* __restrict__ table,
                                                                  uint8_t* __restrict__ u_out, uint8_t* R_uv, uint8_t* Rp_uv,
                                                                  uint8_t* __restrict__ pkp_uv, uint8_t* ok,
                                                                  unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    load_fr(s, key + (kb ? 0 : i) * 32);
    bool good = (ok[i] != 0) & jj::below_order(s);
    if (Note) {
        good &= valid[i] != 0;
        uint32_t t[8];
        const uint32_t mb = 0u - (uint32_t)jj::below_order(s);
#pragma unroll
        for (int q = 0; q < 8; ++q) t[q] = s[q] & mb;
        load_fr(s, h + i * 32);
        jj::order_add(s, s, t);
    }
    const uint32_t m = 0u - (uint32_t)good;
    uint32_t k[8], e[8];
    load_fr(k, r + i * 32);
    load_fr(e, c + i * 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) s[q] &= m, k[q] &= m;
    if (Note) {
        uint32_t pu[8], pv[8];
        jj::fixed_base_mul<true>(pu, pv, s, table);
        store_masked_point(pkp_uv + i * 64, pu, pv, m);
    }
    uint32_t x[8], u[8];
    jj::order_mul(x, e, s);
    jj::order_sub(u, k, x);
#pragma unroll
    for (int q = 0; q < 8; ++q) u[q] &= m;
    store_fr(u_out + i * 32, u);
    uint8_t* const pts[2] = {R_uv + i * 64, Rp_uv + i * 64};
#pragma unroll
    for (int w = 0; w < 2; ++w) {
        uint8_t* P = pts[w];
        uint32_t pu[8], pv[8];
        load_fr_rw(pu, P);
        load_fr_rw(pv, P + 32);
        store_masked_point(P, pu, pv, m);
    }
    ok[i] = good ? 1 : 0;
    if (n_invalid) warp_count_every(n_invalid, !good);
}

// Verify, one thread per item, after k_schnorr_pack_double (valid[i]: R, R' and m canonical) and the truncated digest
// (c[i]): verified[i] = valid[i], u < r_J, PK and PK' curve points with coordinates < p, [c] PK + [u] G == R (table) and
// [c] PK' + [u] G' == R' (table_p): schnorr_check twice, kProductsPerSchnorrVerifyDouble products.  cnt_ok += verified
// items, cnt_bad += invalid ones (once each, whichever side made them invalid).
__global__ void __launch_bounds__(kThreads, 3) k_schnorr_verify_double(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ pkp,
                                                                    bool pb, const uint8_t* __restrict__ u,
                                                                    const uint8_t* __restrict__ R_uv,
                                                                    const uint8_t* __restrict__ Rp_uv,
                                                                    const uint8_t* __restrict__ c,
                                                                    const uint8_t* __restrict__ valid, size_t n,
                                                                    const uint4* __restrict__ table,
                                                                    const uint4* __restrict__ table_p,
                                                                    uint8_t* __restrict__ verified,
                                                                    unsigned long long* __restrict__ cnt_ok,
                                                                    unsigned long long* __restrict__ cnt_bad) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    bool good = valid[i] != 0, ok = true;
    // one copy of the check's code for both sides: the kernel's SASS stays the size of k_schnorr_verify's
#pragma unroll 1
    for (int side = 0; side < 2; ++side)
        ok &= schnorr_check(side ? pkp : pk, pb, u, side ? Rp_uv : R_uv, c, i, side ? table_p : table, good);
    verified[i] = ok ? 1 : 0;
    if (cnt_ok) warp_count_every(cnt_ok, ok);
    if (cnt_bad) warp_count_every(cnt_bad, !good);
}

cudaError_t launch_schnorr_pack_double(const void* R_uv, const void* Rp_uv, const void* msg, size_t n, void* rows,
                                       uint8_t* flag, bool and_flag, cudaStream_t st) {
    return launch(k_schnorr_pack_double, n, 256, st, R_uv, Rp_uv, msg, n, rows, flag, and_flag);
}

cudaError_t launch_schnorr_sign_double(const void* sk, bool sk_bcast, const void* r, const void* c, size_t n, void* u_out,
                                       void* R_uv, void* Rp_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_schnorr_sign_double<false>, n, kThreads, st, sk, sk_bcast, nullptr, nullptr, r, c, n, nullptr, u_out, R_uv,
                  Rp_uv, nullptr, ok, n_invalid);
}

cudaError_t launch_note_sign_double(const void* b, bool b_bcast, const void* h, const uint8_t* valid, const void* r,
                                    const void* c, size_t n, const void* table_p, void* u_out, void* R_uv, void* Rp_uv,
                                    void* pkp_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_schnorr_sign_double<true>, n, kThreads, st, b, b_bcast, h, valid, r, c, n, table_p, u_out, R_uv, Rp_uv,
                  pkp_uv, ok, n_invalid);
}

cudaError_t launch_schnorr_verify_double(const void* pk, const void* pkp, bool pk_bcast, const void* u, const void* R_uv,
                                         const void* Rp_uv, const void* c, const uint8_t* valid, size_t n, const void* table,
                                         const void* table_p, uint8_t* verified, unsigned long long* n_verified,
                                         unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_schnorr_verify_double, n, kThreads, st, pk, pkp, pk_bcast, u, R_uv, Rp_uv, c, valid, n, table, table_p,
                  verified, n_verified, n_invalid);
}

// ---- note values: C = [v] G + [blinder] G' (jubjub_device.cuh) ---------------------------------------------------------
// One thread per item.  table / table_p: the fixed-base tables of G and G'.  [blinder] G' walks the whole table of G' with
// T, then the walk of G continues from it over kValueWindows windows (v is a u64).  v, blinder and the plaintext rows are
// secret: every validity is a mask, an out-of-range operand enters the walk as 0, and the table reads are masked selects.
//   kValueCommit (kProductsPerValueCommit): value[i], blinder[i] (canonical 4 x u64) in; ok[i] = blinder < r_J; the
//     affine C into commitment, zeroed for an invalid item; *count += invalid items.
//   kValueCreate (kProductsPerNoteCreateValue): as commit, but C is written unmasked (the caller zeroes the rows of invalid
//     items once every check is in), rows[i] = [Fr(v), Fr(blinder)] (64 bytes, Montgomery: the message to encrypt), and
//     valid[i] &= blinder < r_J.
//   kValueOpen (kProductsPerNoteOpenValue): rows[i] the decrypted [m0, m1] (Montgomery), ok[i] their authentication,
//     valid[i] the key exchange's validity; opened = ok and valid, m0 < 2^64, m1 < r_J, C's coordinates < p and
//     [m0] G + [m1] G' == C (projective).  value[i] = m0 and blinder[i] = m1 if opened, zeros otherwise; ok[i] = opened;
//     *count += items not opened.
enum ValueMode { kValueCommit, kValueCreate, kValueOpen };

template <int kMode>
__global__ void __launch_bounds__(kThreads, 3) k_value_commit(uint64_t* value, uint8_t* blinder, size_t n,
                                                           const uint4* __restrict__ table, const uint4* __restrict__ table_p,
                                                           uint8_t* commitment, uint8_t* rows, uint8_t* valid, uint8_t* ok,
                                                           unsigned long long* __restrict__ count) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[8];
    bool good;
    if (kMode == kValueOpen) {
        uint32_t m[8];
        load_fr_rw(m, rows + i * 64);
        fr_to_canonical(v, m);
        load_fr_rw(m, rows + i * 64 + 32);
        fr_to_canonical(b, m);
        const bool small = (v[2] | v[3] | v[4] | v[5] | v[6] | v[7]) == 0;
        const bool in_range = jj::below_order(b);
        const uint32_t ms = 0u - (uint32_t)small, mb = 0u - (uint32_t)in_range;
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] &= ms, b[k] &= mb;
        good = (ok[i] != 0) & (valid[i] != 0) & small & in_range;
    } else {
        const uint64_t x = value[i];
        v[0] = (uint32_t)x, v[1] = (uint32_t)(x >> 32);
        load_fr(b, blinder + i * 32);
        good = jj::below_order(b);
        const uint32_t mb = 0u - (uint32_t)good;
#pragma unroll
        for (int k = 0; k < 8; ++k) b[k] &= mb;
    }
    jj::Ext t;
    {
        jj::Ext acc;
        jj::fixed_base_ext<true, true>(acc, b, table_p);
        jj::fixed_base_from<true, false, jj::kValueWindows>(t, acc, v, table);
    }
    if (kMode == kValueOpen) {
        uint32_t cu[8], cv[8];
        const bool canon = load_canonical_point<false>(cu, cv, commitment + i * 64);
        const bool opened = good & canon & equals_affine(cu, cv, t);
        const uint32_t mo = 0u - (uint32_t)opened;
#pragma unroll
        for (int k = 0; k < 8; ++k) b[k] &= mo;
        value[i] = ((uint64_t)v[1] << 32 | v[0]) & ((uint64_t)mo << 32 | mo);
        store_fr(blinder + i * 32, b);
        ok[i] = opened ? 1 : 0;
        if (count) warp_count_every(count, !opened);
    } else {
        uint32_t zi[8], ou[8], ov[8];
        jj::inverse(zi, t.Z);
        jj::fmul(ou, t.X, zi);
        jj::fmul(ov, t.Y, zi);
        store_masked_point(commitment + i * 64, ou, ov, kMode == kValueCommit ? 0u - (uint32_t)good : ~0u);
        if (kMode == kValueCommit) {
            ok[i] = good ? 1 : 0;
            if (count) warp_count_every(count, !good);
        } else {
            uint32_t fv[8], fb[8];
            fr_from_canonical(fv, v);
            fr_from_canonical(fb, b);
            store_fr(rows + i * 64, fv);
            store_fr(rows + i * 64 + 32, fb);
            valid[i] = (valid[i] != 0) & good ? 1 : 0;
        }
    }
}

cudaError_t launch_value_commit(const uint64_t* value, const void* blinder, size_t n, const void* table, const void* table_p,
                                void* commitment, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_value_commit<kValueCommit>, n, kThreads, st, const_cast<uint64_t*>(value), const_cast<void*>(blinder), n,
                  table, table_p, commitment, nullptr, nullptr, ok, n_invalid);
}

cudaError_t launch_note_value(const uint64_t* value, const void* blinder, size_t n, const void* table, const void* table_p,
                              void* commitment, void* rows, uint8_t* valid, cudaStream_t st) {
    return launch(k_value_commit<kValueCreate>, n, kThreads, st, const_cast<uint64_t*>(value), const_cast<void*>(blinder), n,
                  table, table_p, commitment, rows, valid, nullptr, nullptr);
}

cudaError_t launch_note_open_value(const void* rows, const uint8_t* valid, const void* commitment, size_t n, const void* table,
                                   const void* table_p, uint64_t* value, void* blinder, uint8_t* ok,
                                   unsigned long long* n_failed, cudaStream_t st) {
    return launch(k_value_commit<kValueOpen>, n, kThreads, st, value, blinder, n, table, table_p, const_cast<void*>(commitment),
                  const_cast<void*>(rows), const_cast<uint8_t*>(valid), ok, n_failed);
}

// ---- wallet scans: owner, nullifier, checked opening and per-key totals (jubjub_device.cuh) -----------------------------
// k keys (a_j, b_j) and a chunk of n notes; a pair is (note i, key j), at index i k + j.  The key index of a pair is part of
// the schedule (public), like the note index; what no address may depend on is which key owns a note (k_wallet_select).
// keys (kProductsPerWalletKey per key): nb[j] = the Niels form of B_j = [b_j] G (96 bytes), kvalid[j] = a_j, b_j < r_J; a
//   bad key derives B from b = 0.  Thread 0 zeroes the chunk's owned count; *n_bad += bad keys.
__global__ void __launch_bounds__(kThreads, 3) k_wallet_keys(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                                          uint32_t k, const uint4* __restrict__ table, uint8_t* __restrict__ nb,
                                                          uint8_t* __restrict__ kvalid, unsigned long long* __restrict__ n_owned,
                                                          unsigned long long* __restrict__ n_bad) {
    const uint32_t j = blockIdx.x * kThreads + threadIdx.x;
    if (j == 0) *n_owned = 0;
    if (j >= k) return;
    uint32_t s[8], t[8];
    load_fr(s, a + (size_t)j * 32);
    load_fr(t, b + (size_t)j * 32);
    const bool good = jj::below_order(s) & jj::below_order(t);
    const uint32_t m = 0u - (uint32_t)good;
#pragma unroll
    for (int q = 0; q < 8; ++q) t[q] &= m;
    uint32_t u[8], v[8];
    jj::fixed_base_mul<true>(u, v, t, table);
    jj::Niels q;
    jj::to_niels(q, u, v);
    store_fr(nb + (size_t)j * 96, q.ymx);
    store_fr(nb + (size_t)j * 96 + 32, q.ypx);
    store_fr(nb + (size_t)j * 96 + 64, q.kt);
    kvalid[j] = good ? 1 : 0;
    if (n_bad) warp_count_every(n_bad, !good);
}

// dhke (k_dhke's schedule, kProductsPerDhke per pair): out[p] = [a_j] R_i as (u, v), ok[p] = key j good and R_i a curve
// point with u, v < p.  An invalid pair runs the same schedule on (0, identity) and writes (0, 0).
__global__ void __launch_bounds__(kThreads, 3) k_wallet_dhke(const uint8_t* __restrict__ a, const uint8_t* __restrict__ kvalid,
                                                          uint32_t k, const uint8_t* __restrict__ R, size_t n_pairs,
                                                          uint8_t* __restrict__ out, uint8_t* __restrict__ ok) {
    const size_t p = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (p >= n_pairs) return;
    const size_t i = p / k, j = p - i * k;
    uint32_t s[8], u[8], v[8];
    load_fr(s, a + j * 32);
    load_fr(u, R + i * 64);
    load_fr(v, R + i * 64 + 32);
    const bool valid = (kvalid[j] != 0) & fr_is_canonical(u) & fr_is_canonical(v) & jj::on_curve(u, v);
    const uint32_t m = 0u - (uint32_t)valid;
#pragma unroll
    for (int q = 0; q < 8; ++q) s[q] &= m;
    mask_point(u, v, m);
    uint32_t ou[8], ov[8];
    jj::scalar_mul(ou, ov, s, u, v);
    store_masked_point(out + p * 64, ou, ov, m);
    ok[p] = valid ? 1 : 0;
}

// match (k_stealth<true>'s check, kProductsPerStealthOwns per pair): matched[p] = valid[p], both note_pk_i coordinates < p
// and note_pk_i == [h[p]] G + B_j, with B_j's Niels form read from nb; compared projectively.
__global__ void __launch_bounds__(kThreads, 3) k_wallet_match(const uint8_t* __restrict__ h, size_t n_pairs, uint32_t k,
                                                           const uint4* __restrict__ table, const uint8_t* __restrict__ nb,
                                                           const uint8_t* __restrict__ note_pk, const uint8_t* __restrict__ valid,
                                                           uint8_t* __restrict__ matched) {
    const size_t p = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (p >= n_pairs) return;
    const size_t i = p / k, j = p - i * k;
    jj::Ext t, r;
    {
        uint32_t s[8];
        load_fr(s, h + p * 32);
        jj::fixed_base_ext<true, true>(t, s, table);
    }
    uint32_t u[8], v[8];
    const bool canon = load_canonical_point<false>(u, v, note_pk + i * 64);
    jj::Niels q;
    load_fr(q.ymx, nb + j * 96);
    load_fr(q.ypx, nb + j * 96 + 32);
    load_fr(q.kt, nb + j * 96 + 64);
    jj::madd<false>(r, t, q);
    matched[p] = (valid[p] != 0) & canon & equals_affine(u, v, r) ? 1 : 0;
}

// select (per note, kProductsPerWalletSelect): owner[i] = the smallest j with matched[i k + j], -1 if none; the note's
// nullifier, value, blinder and opened rows zeroed; *n_invalid += notes whose R is not a curve point with u, v < p or whose
// note_pk has a coordinate >= p.  S, h and b of the owner's pair are read by masked selects over all k pairs and key
// rows.  An owned note then takes the next dense row (warp-aggregated atomic on *n_owned): meta = (i, owner), S, h, b,
// pos, nonce, cipher, C, dvalid = 1.  Ownership is the only thing that steers the schedule, and the call returns it.
struct WalletDense {
    uint2* meta;
    uint8_t *S, *h, *b;
    uint64_t* pos;
    uint8_t *nonce, *cipher, *C, *valid;
};

__device__ __forceinline__ void copy_row(uint8_t* dst, const uint8_t* src, int words16) {
    for (int q = 0; q < words16; ++q) reinterpret_cast<uint4*>(dst)[q] = __ldg(reinterpret_cast<const uint4*>(src) + q);
}

__global__ void __launch_bounds__(kThreads) k_wallet_select(uint32_t k, const uint8_t* __restrict__ matched,
                                                            const uint8_t* __restrict__ S, const uint8_t* __restrict__ h,
                                                            const uint8_t* __restrict__ b, const uint8_t* __restrict__ R,
                                                            const uint8_t* __restrict__ note_pk, const uint64_t* __restrict__ pos,
                                                            const uint8_t* __restrict__ nonce, const uint8_t* __restrict__ cipher,
                                                            const uint8_t* __restrict__ C, size_t n, int32_t* __restrict__ owner,
                                                            uint8_t* __restrict__ nullifier, uint64_t* __restrict__ value,
                                                            uint8_t* __restrict__ blinder, uint8_t* __restrict__ opened,
                                                            WalletDense dn, unsigned long long* __restrict__ n_owned,
                                                            unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    int32_t own = -1;
#pragma unroll 1
    for (int32_t j = (int32_t)k - 1; j >= 0; --j) own = matched[i * k + j] ? j : own;
    {
        uint32_t u[8], v[8];
        bool good = load_curve_point(u, v, R + i * 64);
        good &= load_canonical_point<false>(u, v, note_pk + i * 64);
        if (n_invalid) warp_count_every(n_invalid, !good);
    }
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    owner[i] = own;
    store_fr(nullifier + i * 32, zero);
    store_fr(blinder + i * 32, zero);
    value[i] = 0;
    opened[i] = 0;
    uint32_t su[8], sv[8], hs[8], bs[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) su[q] = 0, sv[q] = 0, hs[q] = 0, bs[q] = 0;
#pragma unroll 1
    for (uint32_t j = 0; j < k; ++j) {            // j is the public loop counter: the same addresses for every owner
        const uint32_t m = 0u - (uint32_t)((int32_t)j == own);
        uint32_t x[8];
        load_fr(x, S + (i * k + j) * 64);
#pragma unroll
        for (int q = 0; q < 8; ++q) su[q] |= x[q] & m;
        load_fr(x, S + (i * k + j) * 64 + 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) sv[q] |= x[q] & m;
        load_fr(x, h + (i * k + j) * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) hs[q] |= x[q] & m;
        load_fr(x, b + (size_t)j * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) bs[q] |= x[q] & m;
    }
    const bool is_owned = own >= 0;
    const unsigned act = __activemask();
    const unsigned bal = __ballot_sync(act, is_owned);
    const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
    unsigned long long base = 0;
    if (lane == leader && bal) base = atomicAdd(n_owned, (unsigned long long)__popc(bal));
    base = __shfl_sync(act, base, leader);
    if (!is_owned) return;
    const size_t r = base + __popc(bal & ((1u << lane) - 1u));
    dn.meta[r] = make_uint2((uint32_t)i, (uint32_t)own);
    store_fr(dn.S + r * 64, su);
    store_fr(dn.S + r * 64 + 32, sv);
    store_fr(dn.h + r * 32, hs);
    store_fr(dn.b + r * 32, bs);
    dn.pos[r] = pos[i];
    copy_row(dn.nonce + r * 32, nonce + i * 32, 2);
    copy_row(dn.cipher + r * 96, cipher + i * 96, 6);
    copy_row(dn.C + r * 64, C + i * 64, 4);
    dn.valid[r] = 1;
}

// scatter (per owned note): dense row r back to note meta[r].x -- nullifier, value, blinder, opened -- and key meta[r].y's
// totals: value_lo / value_hi (a 128-bit sum: the add that wraps the low word carries one into the high word), n_owned,
// n_opened.  value is zero for a note that did not open.
__global__ void __launch_bounds__(256) k_wallet_scatter(const uint2* __restrict__ meta, const uint8_t* __restrict__ dnul,
                                                        const uint64_t* __restrict__ dvalue, const uint8_t* __restrict__ dblinder,
                                                        const uint8_t* __restrict__ dok, size_t n_own, uint8_t* __restrict__ nullifier,
                                                        uint64_t* __restrict__ value, uint8_t* __restrict__ blinder,
                                                        uint8_t* __restrict__ opened, unsigned long long* __restrict__ totals) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_own) return;
    const uint2 mt = meta[r];
    const size_t i = mt.x;
    copy_row(nullifier + i * 32, dnul + r * 32, 2);
    copy_row(blinder + i * 32, dblinder + r * 32, 2);
    const uint64_t v = dvalue[r];
    const bool op = dok[r] != 0;
    value[i] = v;
    opened[i] = op ? 1 : 0;
    unsigned long long* t = totals + (size_t)mt.y * 4;
    const unsigned long long old = atomicAdd(t, (unsigned long long)v);
    if (old + v < old) atomicAdd(t + 1, 1ull);
    atomicAdd(t + 2, 1ull);
    if (op) atomicAdd(t + 3, 1ull);
}

cudaError_t launch_wallet_keys(const void* a, const void* b, uint32_t k, const void* table, void* nb, uint8_t* kvalid,
                               unsigned long long* n_owned, unsigned long long* n_bad, cudaStream_t st) {
    return launch(k_wallet_keys, k, kThreads, st, a, b, k, table, nb, kvalid, n_owned, n_bad);
}

cudaError_t launch_wallet_dhke(const void* a, const uint8_t* kvalid, uint32_t k, const void* R_uv, size_t n_pairs, void* shared_uv,
                               uint8_t* valid, cudaStream_t st) {
    return launch(k_wallet_dhke, n_pairs, kThreads, st, a, kvalid, k, R_uv, n_pairs, shared_uv, valid);
}

cudaError_t launch_wallet_match(const void* h, size_t n_pairs, uint32_t k, const void* table, const void* nb, const void* note_pk,
                                const uint8_t* valid, uint8_t* matched, cudaStream_t st) {
    return launch(k_wallet_match, n_pairs, kThreads, st, h, n_pairs, k, table, nb, note_pk, valid, matched);
}

cudaError_t launch_wallet_select(uint32_t k, const uint8_t* matched, const void* S, const void* h, const void* b,
                                 const void* R_uv, const void* note_pk, const uint64_t* pos, const void* nonce,
                                 const void* cipher, const void* C, size_t n, int32_t* owner, void* nullifier, uint64_t* value,
                                 void* blinder, uint8_t* opened, const WalletRows& dense, unsigned long long* n_owned,
                                 unsigned long long* n_invalid, cudaStream_t st) {
    WalletDense dn{static_cast<uint2*>(dense.meta), static_cast<uint8_t*>(dense.S), static_cast<uint8_t*>(dense.h),
                   static_cast<uint8_t*>(dense.b), dense.pos, static_cast<uint8_t*>(dense.nonce),
                   static_cast<uint8_t*>(dense.cipher), static_cast<uint8_t*>(dense.C), dense.valid};
    return launch(k_wallet_select, n, kThreads, st, k, matched, S, h, b, R_uv, note_pk, pos, nonce, cipher, C, n, owner, nullifier,
                  value, blinder, opened, dn, n_owned, n_invalid);
}

cudaError_t launch_wallet_scatter(const void* meta, const void* nul, const uint64_t* value_rows, const void* blinder_rows,
                                  const uint8_t* ok, size_t n_own, void* nullifier, uint64_t* value, void* blinder,
                                  uint8_t* opened, unsigned long long* totals, cudaStream_t st) {
    return launch(k_wallet_scatter, n_own, 256, st, meta, nul, value_rows, blinder_rows, ok, n_own, nullifier, value, blinder,
                  opened, totals);
}

// ---- JubJub ElGamal: (c1, c2) = ([r] G, M + [r] PK), M = c2 - [sk] c1 (jubjub_device.cuh) -----------------------------
// One thread per item, jj::elgamal_enc_products<kPairs>() products.  Item i reads PK = pk[pb ? 0 : i], and for each pair
// j < kPairs the message M_j = (j ? m1 : m0)[mb ? 0 : i] and r_j = r[kPairs i + j] (canonical 4 x u64); points are (u, v)
// Montgomery pairs.  c1_j goes to c1 + i stride + 128 j, c2_j to c2 + i stride + 128 j: the generic call has kPairs = 1,
// c1 and c2 two arrays of 64-byte rows; the sender call has kPairs = 2 and rows of 256 bytes [c1_A, c2_A, c1_B, c2_B]
// with c2 = c1 + 64.  valid iff every r_j < r_J and PK and every M_j are curve points with u, v < p; an invalid item runs
// the same schedule on r = 0 and identities, writes zeroed rows and ok = 0, and is counted once.  r and M are secret:
// the table reads of both walks are masked selects, and the points are parked in thread-local memory (never in the
// caller's buffers) until the shared inversion.
template <int kPairs>
__global__ void __launch_bounds__(kThreads, 3) k_elgamal_enc(const uint8_t* __restrict__ pk, bool pb,
                                                          const uint8_t* __restrict__ m0, const uint8_t* __restrict__ m1,
                                                          bool mb, const uint8_t* __restrict__ r, size_t n,
                                                          const uint4* __restrict__ table, uint8_t* c1, uint8_t* c2,
                                                          uint32_t stride, uint8_t* __restrict__ ok,
                                                          unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const uint8_t* mi0 = m0 + (mb ? 0 : i) * 64;
    const uint8_t* mi1 = kPairs == 2 ? m1 + (mb ? 0 : i) * 64 : mi0;
    const uint8_t* ri = r + i * kPairs * 32;
    uint32_t u[8], v[8], s[8];
    bool valid = load_curve_point(u, v, pk + (pb ? 0 : i) * 64);
#pragma unroll
    for (int j = 0; j < kPairs; ++j) {
        uint32_t mu[8], mv[8];
        valid &= load_curve_point(mu, mv, j ? mi1 : mi0);
        load_fr(s, ri + j * 32);
        valid &= jj::below_order(s);
    }
    const uint32_t m = 0u - (uint32_t)valid;
    mask_point(u, v, m);
    jj::Entry tab[16];
    jj::Cached c;
    {
        jj::Ext acc;
        jj::var_table(tab, acc, c, u, v);
    }
    jj::Proj out[2 * kPairs];   // c1_j at 2 j, c2_j at 2 j + 1
#pragma unroll 1
    for (int j = 0; j < kPairs; ++j) {
        load_fr(s, ri + j * 32);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] &= m;
        jj::Ext acc, t;
        jj::var_walk<false, true>(acc, c, tab, s);
        {
            uint32_t mu[8], mv[8];
            const uint8_t* mj = j ? mi1 : mi0;
            load_fr(mu, mj);
            load_fr(mv, mj + 32);
            mask_point(mu, mv, m);
            jj::Niels q;
            jj::to_niels(q, mu, mv);
            jj::madd<false>(t, acc, q);
        }
        jj::park(out[2 * j + 1], t);
        jj::fixed_base_ext<true, false>(t, s, table);
        jj::park(out[2 * j], t);
    }
    jj::batch_affine(out);
#pragma unroll
    for (int j = 0; j < 2 * kPairs; ++j)
        store_masked_point(((j & 1) ? c2 : c1) + i * stride + (j >> 1) * 128, out[j].X, out[j].Y, m);
    ok[i] = valid ? 1 : 0;
    if (n_invalid) warp_count_every(n_invalid, !valid);
}

// One thread per item.  The ciphertext (c1_j, c2_j), j < kPairs, is read at c1 + i stride + 128 j and c2 + i stride + 128 j
// (layouts as for k_elgamal_enc); M_j = c2_j - [s] c1_j = c2_j + [s] (-c1_j) goes to out_j + 64 i.
//   generic (jj::kProductsPerElGamalDec): s = key[kb ? 0 : i] = sk; valid iff sk < r_J and c1, c2 curve points with
//     u, v < p; ok[i] = valid.
//   note (jj::kProductsPerSenderDec), after k_dhke (valid[i]: a < r_J, R a curve point) and the truncated digest (h[i]):
//     s = note_sk = (h + b) mod r_J with b = key[kb ? 0 : i]; valid iff valid[i], b < r_J and all four ciphertext points
//     curve points with u, v < p; ok[i] = valid and owned, owned iff both coordinates of note_pk[i] < p and
//     [note_sk] G == note_pk[i] (table: G's fixed-base table; projective comparison, no inversion).
// An item with ok = 0 gets zeroed rows and is counted once into *count.  Every item runs the same schedule: an invalid
// one on s = 0 and identities, and a note that is not owned is decrypted all the same and its rows zeroed.  The keys,
// h, note_sk and the plaintexts are secret: the table reads are masked selects.  The generic form fits in 128 registers
// without spilling, so it keeps k_dhke's four blocks per SM; the note form needs more and runs three.
template <bool kNote>
__global__ void __launch_bounds__(kThreads, kNote ? 3 : 4) k_elgamal_dec(const uint8_t* __restrict__ key, bool kb,
                                                          const uint8_t* __restrict__ h, const uint8_t* __restrict__ valid,
                                                          const uint8_t* __restrict__ note_pk, const uint8_t* __restrict__ c1,
                                                          const uint8_t* __restrict__ c2, uint32_t stride, size_t n,
                                                          const uint4* __restrict__ table, uint8_t* out0, uint8_t* out1,
                                                          uint8_t* __restrict__ ok, unsigned long long* __restrict__ count) {
    constexpr int kPairs = kNote ? 2 : 1;
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8], u[8], v[8];
    load_fr(s, key + (kb ? 0 : i) * 32);
    bool good = jj::below_order(s);
    if (kNote) {
        const uint32_t mb = 0u - (uint32_t)good;
        uint32_t hh[8], t[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] &= mb;
        load_fr(hh, h + i * 32);
        jj::order_add(t, hh, s);
        jj::fcopy(s, t);
        good &= valid[i] != 0;
    }
#pragma unroll 1
    for (int j = 0; j < kPairs; ++j) {
        good &= load_curve_point(u, v, c1 + i * stride + j * 128);
        good &= load_curve_point(u, v, c2 + i * stride + j * 128);
    }
    const uint32_t m = 0u - (uint32_t)good;
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] &= m;
    jj::Proj out[kPairs];
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll 1
    for (int j = 0; j < kPairs; ++j) {
        jj::Entry tab[16];
        jj::Cached c;
        jj::Ext acc, t;
        load_fr(u, c1 + i * stride + j * 128);
        load_fr(v, c1 + i * stride + j * 128 + 32);
        mask_point(u, v, m);
        fr_sub_mod(u, zero, u);                     // -c1 = (-u, v)
        jj::var_table(tab, acc, c, u, v);
        jj::var_walk<false, true>(acc, c, tab, s);
        load_fr(u, c2 + i * stride + j * 128);
        load_fr(v, c2 + i * stride + j * 128 + 32);
        mask_point(u, v, m);
        jj::Niels q;
        jj::to_niels(q, u, v);
        jj::madd<false>(t, acc, q);
        jj::park(out[j], t);
    }
    bool opened = good;
    if (kNote) {
        jj::Ext t;
        jj::fixed_base_ext<true, false>(t, s, table);
        const bool canon = load_canonical_point<false>(u, v, note_pk + i * 64);
        uint32_t x[8], y[8];
        jj::fmul(x, u, t.Z);
        jj::fmul(y, v, t.Z);
        opened = good & canon & jj::feq(x, t.X) & jj::feq(y, t.Y);
    }
    jj::batch_affine(out);
    const uint32_t mo = 0u - (uint32_t)opened;
#pragma unroll
    for (int j = 0; j < kPairs; ++j) store_masked_point((j ? out1 : out0) + i * 64, out[j].X, out[j].Y, mo);
    ok[i] = opened ? 1 : 0;
    if (count) warp_count_every(count, !opened);
}

cudaError_t launch_elgamal_encrypt(const void* pk, bool pk_bcast, const void* msg, bool msg_bcast, const void* r, size_t n,
                                   const void* table, void* c1_uv, void* c2_uv, uint8_t* ok, unsigned long long* n_invalid,
                                   cudaStream_t st) {
    return launch(k_elgamal_enc<1>, n, kThreads, st, pk, pk_bcast, msg, nullptr, msg_bcast, r, n, table, c1_uv, c2_uv, 64, ok,
                  n_invalid);
}

cudaError_t launch_note_sender_encrypt(const void* note_pk, const void* A_uv, const void* B_uv, bool sender_bcast,
                                       const void* blinder, size_t n, const void* table, void* enc, uint8_t* ok,
                                       unsigned long long* n_invalid, cudaStream_t st) {
    uint8_t* e = static_cast<uint8_t*>(enc);
    return launch(k_elgamal_enc<2>, n, kThreads, st, note_pk, false, A_uv, B_uv, sender_bcast, blinder, n, table, e, e + 64, 256,
                  ok, n_invalid);
}

cudaError_t launch_elgamal_decrypt(const void* sk, bool sk_bcast, const void* c1_uv, const void* c2_uv, size_t n,
                                   void* msg_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_elgamal_dec<false>, n, kThreads, st, sk, sk_bcast, nullptr, nullptr, nullptr, c1_uv, c2_uv, 64, n, nullptr,
                  msg_uv, nullptr, ok, n_invalid);
}

cudaError_t launch_note_sender_decrypt(const void* h, const void* b, bool b_bcast, const uint8_t* valid, const void* note_pk,
                                       const void* enc, size_t n, const void* table, void* A_uv, void* B_uv, uint8_t* ok,
                                       unsigned long long* n_failed, cudaStream_t st) {
    const uint8_t* e = static_cast<const uint8_t*>(enc);
    return launch(k_elgamal_dec<true>, n, kThreads, st, b, b_bcast, h, valid, note_pk, e, e + 64, 256, n, table, A_uv, B_uv, ok,
                  n_failed);
}

// ---- point compression: JubJubAffine::from_bytes / to_bytes (jubjub_device.cuh) ---------------------------------------
// One thread per point.  Public data only.
// from_bytes (kProductsPerDecompress products): bytes[i] -> (u, v) Montgomery; ok[i] = v < p and u^2 a square.  An
// invalid item writes (0, 0), which is not a curve point.
__global__ void __launch_bounds__(kThreads, 3) k_points_from_bytes(const uint8_t* __restrict__ bytes, size_t n,
                                                                uint8_t* __restrict__ uv, uint8_t* __restrict__ ok,
                                                                unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t b[8], u[8], v[8];
    load_fr(b, bytes + i * 32);
    const bool good = jj::decompress(u, v, b);
    store_masked_point(uv + i * 64, u, v, 0u - (uint32_t)good);
    ok[i] = good ? 1 : 0;
    if (n_invalid) warp_count_every(n_invalid, !good);
}

// to_bytes (kProductsPerCompress products): (u, v) Montgomery -> bytes[i]; ok[i] = u, v < p and (u, v) on the curve.  An
// invalid item writes 32 bytes of 0xff: v = 2^255 - 1 >= p, which from_bytes rejects (zero bytes would decode).
__global__ void __launch_bounds__(kThreads, 3) k_points_to_bytes(const uint8_t* __restrict__ uv, size_t n,
                                                              uint8_t* __restrict__ bytes, uint8_t* __restrict__ ok,
                                                              unsigned long long* __restrict__ n_invalid) {
    const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    uint32_t u[8], v[8], b[8];
    const bool canon = load_canonical_point<false>(u, v, uv + i * 64);
    const bool good = canon & jj::on_curve(u, v);
    jj::compress(b, u, v);
    const uint32_t m = 0u - (uint32_t)good;
#pragma unroll
    for (int k = 0; k < 8; ++k) b[k] |= ~m;
    store_fr(bytes + i * 32, b);
    ok[i] = good ? 1 : 0;
    if (n_invalid) warp_count_every(n_invalid, !good);
}

cudaError_t launch_points_from_bytes(const void* bytes, size_t n, void* uv, uint8_t* ok, unsigned long long* n_invalid,
                                     cudaStream_t st) {
    return launch(k_points_from_bytes, n, kThreads, st, bytes, n, uv, ok, n_invalid);
}

cudaError_t launch_points_to_bytes(const void* uv, size_t n, void* bytes, uint8_t* ok, unsigned long long* n_invalid,
                                   cudaStream_t st) {
    return launch(k_points_to_bytes, n, kThreads, st, uv, n, bytes, ok, n_invalid);
}

// ---- multi-scalar multiplication by buckets (jubjub_device.cuh): sum [s_i] P_i --------------------------------------
// Variable time: scalars are public; their digits index buckets and steer branches.  One chunk of m rows at a time:
// k_msm_prep (validity, Niels form, the (window, bucket) key of every digit) -> radix sort of the keys (capi.cu) ->
// k_msm_fill (buckets = identity) -> k_msm_bucket over the sorted digits, then over its carries until one piece is left
// -> k_msm_window (one window sum S_w per window).  k_msm_final adds the chunks' window sums per window and combines the
// windows.
constexpr int kMsmThreads = 128;
constexpr uint32_t kMsmEmpty = 1u << 31;   // a carry slot that holds nothing (its key only keeps the list sorted)

// One thread per row: row i is valid iff s < r_J, u, v < p and (u, v) on the curve (an invalid row is skipped: all its
// keys are the sentinel W B, behind every bucket).  Digit e != 0 of window w gets key w B + |e| - 1 and value i | sign << 31;
// keys and values are window-major (index w m + i).
__global__ void __launch_bounds__(kMsmThreads) k_msm_prep(const uint8_t* __restrict__ sc, const uint8_t* __restrict__ pts,
                                                          uint32_t m, int c, uint4* __restrict__ niels,
                                                          uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                          unsigned long long* __restrict__ n_invalid) {
    const uint32_t i = blockIdx.x * kMsmThreads + threadIdx.x;
    if (i >= m) return;
    uint32_t s[8], u[8], v[8];
    load_fr(s, sc + (size_t)i * 32);
    const bool canon = load_canonical_point<true>(u, v, pts + (size_t)i * 64);
    const bool valid = canon & jj::below_order(s) & jj::on_curve(u, v);
    if (n_invalid) warp_count_every(n_invalid, !valid);
    jj::Niels q;
    jj::to_niels(q, u, v);
    const uint32_t* src[3] = {q.ymx, q.ypx, q.kt};
#pragma unroll
    for (int q3 = 0; q3 < 3; ++q3) {
        niels[(size_t)i * 6 + 2 * q3] = make_uint4(src[q3][0], src[q3][1], src[q3][2], src[q3][3]);
        niels[(size_t)i * 6 + 2 * q3 + 1] = make_uint4(src[q3][4], src[q3][5], src[q3][6], src[q3][7]);
    }
    const int W = jj::msm_windows(c);
    const uint32_t B = 1u << (c - 1), sentinel = (uint32_t)W * B;
    uint32_t carry = 0;
    for (int w = 0; w < W; ++w) {
        const int32_t e = jj::recode_window(s, carry, c, w == W - 1);
        const uint32_t mag = (uint32_t)(e < 0 ? -e : e);
        keys[(size_t)w * m + i] = (valid && mag) ? (uint32_t)w * B + mag - 1 : sentinel;
        vals[(size_t)w * m + i] = i | ((uint32_t)(e < 0) << 31);
    }
}

__global__ void __launch_bounds__(256) k_msm_fill(uint4* __restrict__ buckets, uint32_t nb) {
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= nb) return;
    jj::Ext p;
    jj::set_identity(p);
    jj::store_ext(buckets + (size_t)i * 8, p);
}

// One thread per piece of kMsmPiece consecutive entries of a key-sorted list: the sorted digits (kRows: values index the
// Niels rows, bit 31 the sign) or the carries of the previous pass (extended points, kMsmEmpty in the key marks an empty
// slot).  Each run of equal keys in the piece is summed; keys >= nb (the sentinel) are skipped.  A run that continues into
// the neighbouring piece on either side goes to the next list -- slot 2 t if it starts the piece, 2 t + 1 if it ends it --
// and every other run is a whole bucket, stored.  So no thread adds more than kMsmPiece points however the scalars fall,
// each pass shrinks the list by kMsmPiece / 2, and a list of one piece stores everything.
template <bool kRows>
__global__ void __launch_bounds__(kMsmThreads) k_msm_bucket(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                            const uint4* __restrict__ src, uint32_t N, uint32_t nb,
                                                            uint4* __restrict__ buckets, uint32_t* __restrict__ okeys,
                                                            uint4* __restrict__ opts) {
    const uint32_t t = blockIdx.x * kMsmThreads + threadIdx.x;
    const uint32_t lo = t * kMsmPiece;
    if (lo >= N) return;
    const uint32_t hi = min(N, lo + kMsmPiece);
    auto key_at = [&](uint32_t j) { return kRows ? keys[j] : keys[j] & ~kMsmEmpty; };
    const uint32_t none = 0xffffffffu;
    const uint32_t prevk = lo > 0 ? key_at(lo - 1) : none, nextk = hi < N ? key_at(hi) : none;
    bool head = false, tail = false;
    for (uint32_t i = lo; i < hi;) {
        const uint32_t k = key_at(i);
        jj::Ext acc, r;
        jj::set_identity(acc);
        bool any = false;
        uint32_t j = i;
        for (; j < hi && key_at(j) == k; ++j) {
            if (k >= nb) continue;
            if (kRows) {
                const uint32_t v = vals[j];
                const uint4* e = src + (size_t)(v & 0x7fffffffu) * 6;
                jj::Niels q;
                uint32_t* dst[3] = {q.ymx, q.ypx, q.kt};
#pragma unroll
                for (int q3 = 0; q3 < 3; ++q3) {
                    const uint4 a = __ldg(e + 2 * q3), b = __ldg(e + 2 * q3 + 1);
                    dst[q3][0] = a.x, dst[q3][1] = a.y, dst[q3][2] = a.z, dst[q3][3] = a.w;
                    dst[q3][4] = b.x, dst[q3][5] = b.y, dst[q3][6] = b.z, dst[q3][7] = b.w;
                }
                if (v >> 31) {                              // -(u, v) = (-u, v): swap v - u and v + u, negate 2d u v
                    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
                    for (int k2 = 0; k2 < 8; ++k2) {
                        const uint32_t x = q.ymx[k2];
                        q.ymx[k2] = q.ypx[k2];
                        q.ypx[k2] = x;
                    }
                    uint32_t nk[8];
                    fr_sub_mod(nk, zero, q.kt);
                    jj::fcopy(q.kt, nk);
                }
                jj::madd<true>(r, acc, q);
            } else {
                if (keys[j] & kMsmEmpty) continue;
                jj::Ext p;
                jj::load_ext(p, src + (size_t)j * 8);
                jj::add_ext(r, acc, p);
            }
            acc = r;
            any = true;
        }
        const bool first = i == lo;
        if ((first && prevk == k) || (j == hi && nextk == k)) {
            const uint32_t slot = 2 * t + (first ? 0 : 1);
            okeys[slot] = k | (any ? 0u : kMsmEmpty);
            if (any) jj::store_ext(opts + (size_t)slot * 8, acc);
            (first ? head : tail) = true;
        } else if (any) {
            jj::store_ext(buckets + (size_t)k * 8, acc);
        }
        i = j;
    }
    if (okeys && !head) okeys[2 * t] = key_at(lo) | kMsmEmpty;
    if (okeys && !tail) okeys[2 * t + 1] = key_at(hi - 1) | kMsmEmpty;
}

// One block per window, P = msm_window_parts(c) threads, each over L = B / P consecutive buckets (index lo + j holds
// |digit| = lo + j + 1): running sums from the top give r = sum B and t = sum (j + 1) B, so the part's share of
// S_w = sum |digit| B is t + [lo] r (the offset correction); the parts are added in shared memory.
__global__ void __launch_bounds__(kMsmThreads) k_msm_window(const uint4* __restrict__ buckets, int c, uint4* __restrict__ wsum) {
    __shared__ uint4 sh[kMsmThreads * 8];
    const int w = blockIdx.x, p = threadIdx.x, P = blockDim.x;
    const uint32_t B = 1u << (c - 1), L = B / P, lo = p * L;
    jj::Ext r, t, x;
    jj::set_identity(r);
    jj::set_identity(t);
    for (int j = (int)L - 1; j >= 0; --j) {
        jj::Ext b;
        jj::load_ext(b, buckets + ((size_t)w * B + lo + j) * 8);
        jj::add_ext(x, r, b);
        r = x;
        jj::add_ext(x, t, r);
        t = x;
    }
    jj::mul_small(x, r, lo);
    jj::add_ext(r, t, x);
    jj::store_ext(sh + p * 8, r);
    __syncthreads();
    for (int s = P / 2; s > 0; s >>= 1) {
        if (p < s) {
            jj::Ext a, b;
            jj::load_ext(a, sh + p * 8);
            jj::load_ext(b, sh + (p + s) * 8);
            jj::add_ext(x, a, b);
            jj::store_ext(sh + p * 8, x);
        }
        __syncthreads();
    }
    if (p == 0) {
#pragma unroll
        for (int q = 0; q < 8; ++q) wsum[(size_t)w * 8 + q] = sh[q];
    }
}

static_assert(kMsmThreads == kMsmItemsPerSum, "one (z u, z c) sum per block of k_msmv_prep");
static_assert(jj::kMsmMaxBits <= 13, "k_msm_window: at most 4096 buckets per window, 32 per thread of 128");

int msm_windows(int c) { return jj::msm_windows(c); }

// The window width for chunks of `rows` rows: the fewest products by the counts of jubjub_device.cuh, rows x W (c) digit
// additions (a digit is 0 with probability 2^-c only) against W (c) 2^(c-1) running-sum steps.
int msm_bits(size_t rows) {
    int best = jj::kMsmMinBits;
    double best_cost = 0;
    for (int c = jj::kMsmMinBits; c <= jj::kMsmMaxBits; ++c) {
        const double W = jj::msm_windows(c);
        const double cost = (double)rows * W * jj::kProductsPerMsmDigit + W * (double)(1 << (c - 1)) * jj::kProductsPerMsmBucket;
        if (c == jj::kMsmMinBits || cost < best_cost) best = c, best_cost = cost;
    }
    return best;
}

int msm_window_parts(int c) {
    const int B = 1 << (c - 1);
    return B >= 32 ? (B / 32 < kMsmThreads ? B / 32 : kMsmThreads) : 1;
}

// verify_all, one thread per item, after k_schnorr_pack (valid[i]: R and m canonical) and the truncated digest (c[i]).  The
// item is valid iff valid[i], u < r_J, z < r_J and PK = pk[pb ? 0 : i] is a curve point with u, v < p; an R off the curve
// is not invalid but fails the batch.  Either sets *bad.  Rows: pb: row i = (z, -R); otherwise rows 2 i = (z c mod r_J, PK)
// and 2 i + 1 = (z, -R).  An invalid item's (and an off-curve R's) rows are (0, identity).  The block's sums of z u (and,
// pb, of z c) modulo r_J go to zsum[blk0 + block] (64 bytes).
__global__ void __launch_bounds__(kMsmThreads) k_msmv_prep(const uint8_t* __restrict__ pk, bool pb, const uint8_t* __restrict__ u,
                                                           const uint8_t* __restrict__ R_uv, const uint8_t* __restrict__ c,
                                                           const uint8_t* __restrict__ z, const uint8_t* __restrict__ valid,
                                                           uint32_t n, uint8_t* __restrict__ rsc, uint8_t* __restrict__ rpt,
                                                           uint8_t* __restrict__ zsum, uint32_t blk0, uint32_t* __restrict__ bad,
                                                           unsigned long long* __restrict__ n_invalid) {
    __shared__ uint32_t sh[kMsmThreads][16];
    const uint32_t i = blockIdx.x * kMsmThreads + threadIdx.x;
    uint32_t zu[8] = {0, 0, 0, 0, 0, 0, 0, 0}, zc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (i < n) {
        uint32_t x[8], y[8], one[8], s[8], w[8], e[8];
        jj::set_one(one);
        load_fr(x, pk + (pb ? 0 : (size_t)i) * 64);
        load_fr(y, pk + (pb ? 0 : (size_t)i) * 64 + 32);
        const bool canon = fr_is_canonical(x) & fr_is_canonical(y);
        const uint32_t mc = 0u - (uint32_t)canon;
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] &= mc, y[k] = (y[k] & mc) | (one[k] & ~mc);
        load_fr(s, u + (size_t)i * 32);
        load_fr(w, z + (size_t)i * 32);
        load_fr(e, c + (size_t)i * 32);
        const bool good = (valid[i] != 0) & canon & jj::on_curve(x, y) & jj::below_order(s) & jj::below_order(w);
        uint32_t ru[8], rv[8];
        load_fr(ru, R_uv + (size_t)i * 64);
        load_fr(rv, R_uv + (size_t)i * 64 + 32);
        mask_point(ru, rv, 0u - (uint32_t)good);        // an invalid item's R may be >= p: it enters no product
        const bool r_on = jj::on_curve(ru, rv);
        if (!good || !r_on) *bad = 1u;
        if (n_invalid) warp_count_every(n_invalid, !good);
        const uint32_t mg = 0u - (uint32_t)(good & r_on);
        const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t nu[8];
        fr_sub_mod(nu, zero, ru);
#pragma unroll
        for (int k = 0; k < 8; ++k) w[k] &= mg, s[k] &= mg, x[k] &= mg, y[k] = (y[k] & mg) | (one[k] & ~mg),
                                    nu[k] &= mg, rv[k] = (rv[k] & mg) | (one[k] & ~mg);
        jj::order_mul(zc, w, e);                        // c < 2^250 < r_J
        jj::order_mul(zu, w, s);
        const size_t rr = pb ? i : 2 * (size_t)i + 1;   // the row of (z, -R)
        store_fr(rsc + rr * 32, w);
        store_fr(rpt + rr * 64, nu);
        store_fr(rpt + rr * 64 + 32, rv);
        if (!pb) {
            store_fr(rsc + (rr - 1) * 32, zc);
            store_fr(rpt + (rr - 1) * 64, x);
            store_fr(rpt + (rr - 1) * 64 + 32, y);
#pragma unroll
            for (int k = 0; k < 8; ++k) zc[k] = 0;
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) sh[threadIdx.x][k] = zu[k], sh[threadIdx.x][8 + k] = zc[k];
    __syncthreads();
    for (int h = kMsmThreads / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) {
            uint32_t a[8], b[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] = sh[threadIdx.x][k], b[k] = sh[threadIdx.x + h][k];
            jj::order_add(a, a, b);
#pragma unroll
            for (int k = 0; k < 8; ++k) sh[threadIdx.x][k] = a[k], a[k] = sh[threadIdx.x][8 + k], b[k] = sh[threadIdx.x + h][8 + k];
            jj::order_add(a, a, b);
#pragma unroll
            for (int k = 0; k < 8; ++k) sh[threadIdx.x][8 + k] = a[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t a[8], b[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = sh[0][k], b[k] = sh[0][8 + k];
        store_fr(zsum + (size_t)(blk0 + blockIdx.x) * 64, a);
        store_fr(zsum + (size_t)(blk0 + blockIdx.x) * 64 + 32, b);
    }
}

// One block of kMsmThreads threads.  Threads w < W add window w's sums of every chunk; with zsum (verify_all) the block
// first adds the nsum (z u, z c) pairs modulo r_J, then thread 64 computes [sum z u] G from the fixed-base table and thread
// 96 [sum z c] PK (pk: the one public key, or null).  Thread 0 combines the windows (c doublings each) and adds both:
//   MSM:        out_uv = the sum, affine (the identity (0, 1) for no chunks);
//   verify_all: *verified = [8] sum == identity (X == 0, Y == Z) and *bad == 0.
struct MsmFinal {
    const uint4* wsum;
    uint32_t nchunks;
    int c;
    uint8_t* out_uv;
    const uint8_t* zsum;
    uint32_t nsum;
    const uint4* table;
    const uint8_t* pk;
    const uint32_t* bad;
    unsigned long long* verified;
};

__global__ void __launch_bounds__(kMsmThreads) k_msm_final(MsmFinal a) {
    __shared__ uint4 sw[64 * 8], sg[8], sp[8];
    __shared__ uint32_t ss[kMsmThreads][16];
    const int W = jj::msm_windows(a.c), tid = threadIdx.x;
    if (a.zsum) {
        uint32_t x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (uint32_t k = tid; k < a.nsum; k += kMsmThreads) {
            uint32_t b[8];
            load_fr_rw(b, a.zsum + (size_t)k * 64);
            jj::order_add(x, x, b);
            load_fr_rw(b, a.zsum + (size_t)k * 64 + 32);
            jj::order_add(y, y, b);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) ss[tid][k] = x[k], ss[tid][8 + k] = y[k];
        __syncthreads();
        for (int h = kMsmThreads / 2; h > 0; h >>= 1) {
            if (tid < h) {
                uint32_t p[8], q[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) p[k] = ss[tid][k], q[k] = ss[tid + h][k];
                jj::order_add(p, p, q);
#pragma unroll
                for (int k = 0; k < 8; ++k) ss[tid][k] = p[k], p[k] = ss[tid][8 + k], q[k] = ss[tid + h][8 + k];
                jj::order_add(p, p, q);
#pragma unroll
                for (int k = 0; k < 8; ++k) ss[tid][8 + k] = p[k];
            }
            __syncthreads();
        }
    }
    if (tid < W) {
        jj::Ext s, x;
        jj::set_identity(s);
        for (uint32_t k = 0; k < a.nchunks; ++k) {
            jj::Ext p;
            jj::load_ext(p, a.wsum + ((size_t)k * W + tid) * 8);
            jj::add_ext(x, s, p);
            s = x;
        }
        jj::store_ext(sw + tid * 8, s);
    } else if (tid == 64 && a.zsum) {
        uint32_t s[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] = ss[0][k];
        jj::Ext t;
        jj::fixed_base_ext<true, true>(t, s, a.table);
        jj::store_ext(sg, t);
    } else if (tid == 96 && a.zsum) {
        jj::Ext t;
        if (a.pk) {
            uint32_t s[8], x[8], y[8], one[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) s[k] = ss[0][8 + k];
            load_canonical_point<true>(x, y, a.pk);
            jj::set_one(one);
            const uint32_t mc = 0u - (uint32_t)jj::on_curve(x, y);    // an off-curve PK made every item invalid: *bad is set
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] &= mc, y[k] = (y[k] & mc) | (one[k] & ~mc), s[k] &= mc;
            jj::scalar_mul_ext<true, true>(t, s, x, y);
        } else {
            jj::set_identity(t);
        }
        jj::store_ext(sp, t);
    }
    __syncthreads();
    if (tid != 0) return;
    jj::Ext acc, x;
    jj::load_ext(acc, sw + (W - 1) * 8);
    for (int w = W - 2; w >= 0; --w) {
        for (int d = 0; d < a.c; ++d) {
            jj::dbl<true>(x, acc);
            acc = x;
        }
        jj::Ext s;
        jj::load_ext(s, sw + w * 8);
        jj::add_ext(x, acc, s);
        acc = x;
    }
    if (!a.zsum) {
        uint32_t zi[8], ou[8], ov[8];
        jj::inverse(zi, acc.Z);
        jj::fmul(ou, acc.X, zi);
        jj::fmul(ov, acc.Y, zi);
        store_fr(a.out_uv, ou);
        store_fr(a.out_uv + 32, ov);
        return;
    }
    jj::Ext g;
    jj::load_ext(g, sg);
    jj::add_ext(x, acc, g);
    jj::load_ext(g, sp);
    jj::add_ext(acc, x, g);
    for (int d = 0; d < 3; ++d) {                        // the cofactor
        jj::dbl<true>(x, acc);
        acc = x;
    }
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const bool ok = jj::feq(acc.X, zero) & jj::feq(acc.Y, acc.Z) & (*a.bad == 0);
    *a.verified = ok ? 1ull : 0ull;
}

cudaError_t launch_msm_prep(const void* scalars, const void* points, uint32_t m, int c, void* niels, uint32_t* keys,
                            uint32_t* vals, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_msm_prep, m, kMsmThreads, st, scalars, points, m, c, niels, keys, vals, n_invalid);
}

cudaError_t launch_msm_fill(void* buckets, uint32_t nb, cudaStream_t st) {
    return launch(k_msm_fill, nb, 256, st, buckets, nb);
}

cudaError_t launch_msm_bucket(bool rows, const uint32_t* keys, const uint32_t* vals, const void* src, uint32_t N, uint32_t nb,
                              void* buckets, uint32_t* okeys, void* opts, cudaStream_t st) {
    const uint32_t pieces = (N + kMsmPiece - 1) / kMsmPiece;   // one thread per piece
    if (rows) return launch(k_msm_bucket<true>, pieces, kMsmThreads, st, keys, vals, src, N, nb, buckets, okeys, opts);
    return launch(k_msm_bucket<false>, pieces, kMsmThreads, st, keys, vals, src, N, nb, buckets, okeys, opts);
}

cudaError_t launch_msm_window(const void* buckets, int c, void* wsum, cudaStream_t st) {
    return launch_grid(k_msm_window, jj::msm_windows(c), msm_window_parts(c), st, buckets, c, wsum);
}

cudaError_t launch_msm_final(const void* wsum, uint32_t nchunks, int c, void* out_uv, const void* zsum, uint32_t nsum,
                             const void* table, const void* pk, const uint32_t* bad, unsigned long long* verified,
                             cudaStream_t st) {
    MsmFinal a{static_cast<const uint4*>(wsum), nchunks, c, static_cast<uint8_t*>(out_uv), static_cast<const uint8_t*>(zsum),
               nsum, static_cast<const uint4*>(table), static_cast<const uint8_t*>(pk), bad, verified};
    return launch_grid(k_msm_final, 1, kMsmThreads, st, a);
}

cudaError_t launch_msmv_prep(const void* pk, bool pk_bcast, const void* u, const void* R_uv, const void* c, const void* z,
                             const uint8_t* valid, uint32_t n, void* row_scalars, void* row_points, void* zsum, uint32_t blk0,
                             uint32_t* bad, unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_msmv_prep, n, kMsmThreads, st, pk, pk_bcast, u, R_uv, c, z, valid, n, row_scalars, row_points, zsum, blk0,
                  bad, n_invalid);
}

// ---- all-or-nothing verification of double-key signatures: one MSM over G and G' ---------------------------------------
// verify_double_all, one thread per item, after k_schnorr_pack_double (valid[i]: R, R' and m canonical) and the truncated
// digest (c[i]).  The item is valid iff valid[i], u, z, z' < r_J and PK, PK' = (pk, pkp)[pb ? 0 : i] are curve points with
// u, v < p; an R or R' off the curve is not invalid but fails the batch.  Either sets *bad.  Rows: pb: 2 i = (z, -R) and
// 2 i + 1 = (z', -R'); otherwise 4 i = (z c, PK), 4 i + 1 = (z' c, PK'), 4 i + 2 = (z, -R), 4 i + 3 = (z', -R').  An
// invalid item's (and an off-curve R's or R''s) rows are (0, identity).  The block's sums modulo r_J of z u, z' u and, pb,
// z c, z' c go to zsum[blk0 + block] (128 bytes, in that order).  The checks run first and the rows are written from a
// second load of each side, so only one side's operands are live at a time.
__global__ void __launch_bounds__(kMsmThreads) k_msmv_prep_double(const uint8_t* __restrict__ pk,
                                                                  const uint8_t* __restrict__ pkp, bool pb,
                                                                  const uint8_t* __restrict__ u,
                                                                  const uint8_t* __restrict__ R_uv,
                                                                  const uint8_t* __restrict__ Rp_uv,
                                                                  const uint8_t* __restrict__ c,
                                                                  const uint8_t* __restrict__ z,
                                                                  const uint8_t* __restrict__ zp,
                                                                  const uint8_t* __restrict__ valid, uint32_t n,
                                                                  uint8_t* __restrict__ rsc, uint8_t* __restrict__ rpt,
                                                                  uint8_t* __restrict__ zsum, uint32_t blk0,
                                                                  uint32_t* __restrict__ bad,
                                                                  unsigned long long* __restrict__ n_invalid) {
    __shared__ uint32_t sh[kMsmThreads][32];
    const uint32_t i = blockIdx.x * kMsmThreads + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 32; ++k) sh[threadIdx.x][k] = 0;
    if (i < n) {
        // side 0: (z, PK, R); side 1: (z', PK', R')
        auto key = [&](int side) { return (side ? pkp : pk) + (pb ? 0 : (size_t)i) * 64; };
        auto wt = [&](int side) { return (side ? zp : z) + (size_t)i * 32; };
        auto rr = [&](int side) { return (side ? Rp_uv : R_uv) + (size_t)i * 64; };
        uint32_t one[8], s[8], x[8], y[8], w[8];
        jj::set_one(one);
        load_fr(s, u + (size_t)i * 32);
        bool good = (valid[i] != 0) & jj::below_order(s);
#pragma unroll 1
        for (int side = 0; side < 2; ++side) {
            const bool canon = load_canonical_point<true>(x, y, key(side));
            load_fr(w, wt(side));
            good &= canon & jj::on_curve(x, y) & jj::below_order(w);
        }
        const uint32_t mv = 0u - (uint32_t)good;        // an invalid item's R and R' may be >= p: they enter no product
        bool r_on = true;
#pragma unroll 1
        for (int side = 0; side < 2; ++side) {
            load_fr(x, rr(side));
            load_fr(y, rr(side) + 32);
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] &= mv, y[k] = (y[k] & mv) | (one[k] & ~mv);
            r_on &= jj::on_curve(x, y);
        }
        if (!good || !r_on) *bad = 1u;
        if (n_invalid) warp_count_every(n_invalid, !good);
        const uint32_t mg = 0u - (uint32_t)(good & r_on);
        const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t e[8], t[8];
        load_fr(e, c + (size_t)i * 32);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] &= mg;
        const size_t per = pb ? 2 : 4, r0 = per * i + (pb ? 0 : 2);   // the row of (z, -R); (z', -R') follows it
#pragma unroll 1
        for (int side = 0; side < 2; ++side) {
            load_fr(w, wt(side));
#pragma unroll
            for (int k = 0; k < 8; ++k) w[k] &= mg;
            jj::order_mul(t, w, s);
#pragma unroll
            for (int k = 0; k < 8; ++k) sh[threadIdx.x][8 * side + k] = t[k];
            jj::order_mul(t, w, e);                     // c < 2^250 < r_J
            load_fr(x, rr(side));
            load_fr(y, rr(side) + 32);
            mask_point(x, y, mg);
            uint32_t nx[8];
            fr_sub_mod(nx, zero, x);
            store_fr(rsc + (r0 + side) * 32, w);
            store_fr(rpt + (r0 + side) * 64, nx);
            store_fr(rpt + (r0 + side) * 64 + 32, y);
            if (pb) {
#pragma unroll
                for (int k = 0; k < 8; ++k) sh[threadIdx.x][16 + 8 * side + k] = t[k];
            } else {
                load_fr(x, key(side));
                load_fr(y, key(side) + 32);
                mask_point(x, y, mg);
                store_fr(rsc + (per * i + side) * 32, t);
                store_fr(rpt + (per * i + side) * 64, x);
                store_fr(rpt + (per * i + side) * 64 + 32, y);
            }
        }
    }
    __syncthreads();
    for (int h = kMsmThreads / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) {
#pragma unroll 1
            for (int q = 0; q < 4; ++q) {
                uint32_t a[8], b[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) a[k] = sh[threadIdx.x][8 * q + k], b[k] = sh[threadIdx.x + h][8 * q + k];
                jj::order_add(a, a, b);
#pragma unroll
                for (int k = 0; k < 8; ++k) sh[threadIdx.x][8 * q + k] = a[k];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x < 4) {
        uint32_t a[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = sh[0][8 * threadIdx.x + k];
        store_fr(zsum + (size_t)(blk0 + blockIdx.x) * 128 + threadIdx.x * 32, a);
    }
}

// One block of kMsmFinalThreads threads, six warps.  Threads below kMsmThreads first add the nsum 4-tuples of zsum modulo
// r_J.  Then warps 0-1 add window w's sums of every chunk (thread w < W <= 64), and four walks run on warps of their own,
// so none waits for another: thread 64 [sum z u] G (table), thread 96 [sum z' u] G' (table_p), and, for one key pair (pk:
// PK then PK', 128 bytes; null for none), thread 128 [sum z c] PK and thread 160 [sum z' c] PK'.  Thread 0 combines the
// windows (c doublings each), adds the four points and writes *verified = [8] sum == identity (X == 0, Y == Z) and
// *bad == 0.
constexpr int kMsmFinalThreads = 192;
struct MsmFinalDouble {
    const uint4* wsum;
    uint32_t nchunks;
    int c;
    const uint8_t* zsum;
    uint32_t nsum;
    const uint4* table;
    const uint4* table_p;
    const uint8_t* pk;
    const uint32_t* bad;
    unsigned long long* verified;
};

__global__ void __launch_bounds__(kMsmFinalThreads) k_msmv_final_double(MsmFinalDouble a) {
    __shared__ uint4 sw[64 * 8], sq[4 * 8];
    __shared__ uint32_t ss[kMsmThreads][32];
    const int W = jj::msm_windows(a.c), tid = threadIdx.x;
    if (tid < kMsmThreads) {
#pragma unroll 1
        for (int q = 0; q < 4; ++q) {
            uint32_t x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t k = tid; k < a.nsum; k += kMsmThreads) {
                uint32_t b[8];
                load_fr_rw(b, a.zsum + (size_t)k * 128 + q * 32);
                jj::order_add(x, x, b);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) ss[tid][8 * q + k] = x[k];
        }
    }
    __syncthreads();
    for (int h = kMsmThreads / 2; h > 0; h >>= 1) {
        if (tid < h) {
#pragma unroll 1
            for (int q = 0; q < 4; ++q) {
                uint32_t p[8], r[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) p[k] = ss[tid][8 * q + k], r[k] = ss[tid + h][8 * q + k];
                jj::order_add(p, p, r);
#pragma unroll
                for (int k = 0; k < 8; ++k) ss[tid][8 * q + k] = p[k];
            }
        }
        __syncthreads();
    }
    if (tid < W) {
        jj::Ext s, x;
        jj::set_identity(s);
        for (uint32_t k = 0; k < a.nchunks; ++k) {
            jj::Ext p;
            jj::load_ext(p, a.wsum + ((size_t)k * W + tid) * 8);
            jj::add_ext(x, s, p);
            s = x;
        }
        jj::store_ext(sw + tid * 8, s);
    } else if (tid == 64 || tid == 96) {
        const int side = tid == 96;
        uint32_t s[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] = ss[0][8 * side + k];
        jj::Ext t;
        jj::fixed_base_ext<true, true>(t, s, side ? a.table_p : a.table);
        jj::store_ext(sq + side * 8, t);
    } else if (tid == 128 || tid == 160) {
        const int side = tid == 160;
        jj::Ext t;
        if (a.pk) {
            uint32_t s[8], x[8], y[8], one[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) s[k] = ss[0][16 + 8 * side + k];
            load_canonical_point<true>(x, y, a.pk + side * 64);
            jj::set_one(one);
            const uint32_t mc = 0u - (uint32_t)jj::on_curve(x, y);    // an off-curve key made every item invalid: *bad is set
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] &= mc, y[k] = (y[k] & mc) | (one[k] & ~mc), s[k] &= mc;
            jj::scalar_mul_ext<true, true>(t, s, x, y);
        } else {
            jj::set_identity(t);
        }
        jj::store_ext(sq + (2 + side) * 8, t);
    }
    __syncthreads();
    if (tid != 0) return;
    jj::Ext acc, x;
    jj::load_ext(acc, sw + (W - 1) * 8);
    for (int w = W - 2; w >= 0; --w) {
        for (int d = 0; d < a.c; ++d) {
            jj::dbl<true>(x, acc);
            acc = x;
        }
        jj::Ext s;
        jj::load_ext(s, sw + w * 8);
        jj::add_ext(x, acc, s);
        acc = x;
    }
#pragma unroll 1
    for (int q = 0; q < 4; ++q) {
        jj::Ext g;
        jj::load_ext(g, sq + q * 8);
        jj::add_ext(x, acc, g);
        acc = x;
    }
    for (int d = 0; d < 3; ++d) {                        // the cofactor
        jj::dbl<true>(x, acc);
        acc = x;
    }
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const bool ok = jj::feq(acc.X, zero) & jj::feq(acc.Y, acc.Z) & (*a.bad == 0);
    *a.verified = ok ? 1ull : 0ull;
}

cudaError_t launch_msmv_prep_double(const void* pk, const void* pkp, bool pk_bcast, const void* u, const void* R_uv,
                                    const void* Rp_uv, const void* c, const void* z, const void* zp, const uint8_t* valid,
                                    uint32_t n, void* row_scalars, void* row_points, void* zsum, uint32_t blk0, uint32_t* bad,
                                    unsigned long long* n_invalid, cudaStream_t st) {
    return launch(k_msmv_prep_double, n, kMsmThreads, st, pk, pkp, pk_bcast, u, R_uv, Rp_uv, c, z, zp, valid, n, row_scalars,
                  row_points, zsum, blk0, bad, n_invalid);
}

cudaError_t launch_msmv_final_double(const void* wsum, uint32_t nchunks, int c, const void* zsum, uint32_t nsum,
                                     const void* table, const void* table_p, const void* pk, const uint32_t* bad,
                                     unsigned long long* verified, cudaStream_t st) {
    MsmFinalDouble a{static_cast<const uint4*>(wsum), nchunks, c, static_cast<const uint8_t*>(zsum), nsum,
                     static_cast<const uint4*>(table), static_cast<const uint4*>(table_p), static_cast<const uint8_t*>(pk),
                     bad, verified};
    return launch_grid(k_msmv_final_double, 1, kMsmFinalThreads, st, a);
}

cudaError_t launch_merkle_open(const void* leaves, const void* nodes, const uint64_t* leaf_idx, size_t n, int arity,
                               uint32_t depth, const OpenLevels& lv, void* paths, cudaStream_t st, const uint8_t* present) {
    const uint32_t la = log2_arity(arity);
    if (present)
        return launch(k_merkle_open<true>, n * depth, 256, st, leaves, nodes, leaf_idx, n, la, depth, lv, paths, present);
    return launch(k_merkle_open<false>, n * depth, 256, st, leaves, nodes, leaf_idx, n, la, depth, lv, paths, nullptr);
}

cudaError_t launch_mtree_keys(const uint64_t* idx, uint32_t n_upd, uint64_t n_old, uint32_t total, uint64_t* keys,
                              uint32_t* pos, unsigned long long* rejected, cudaStream_t st) {
    return launch(k_mtree_keys, total, 256, st, idx, n_upd, n_old, total, keys, pos, rejected);
}

cudaError_t launch_mtree_leaf_write(const uint64_t* keys, const uint32_t* pos, uint32_t total, uint64_t sentinel, int arity,
                                    const void* values, uint32_t n_upd, const void* append, void* leaves, uint8_t* flag,
                                    uint64_t* parent, cudaStream_t st) {
    return launch(k_mtree_leaf_write, total, 256, st, keys, pos, total, sentinel, log2_arity(arity), values, n_upd, append, leaves,
                  flag, parent);
}

cudaError_t launch_mtree_parents(const uint64_t* d, const int* cnt, uint32_t bound, int arity, uint8_t* flag, uint64_t* parent,
                                 cudaStream_t st) {
    return launch(k_mtree_parents, bound, 256, st, d, cnt, bound, log2_arity(arity), flag, parent);
}

template <bool kSparse>
static cudaError_t mtree_digest(FrArg tag, const void* b, int arity, void* o, const uint64_t* d, const int* cnt, size_t bound,
                                size_t coop_max, cudaStream_t st, const uint8_t* bp, uint8_t* lp) {
    if (bound <= coop_max)
        return launch_grid(k_mtree_digest_coop<kSparse>, coop_grid(bound), kThreads, st, tag, b, (uint32_t)arity, o, d, cnt, bp, lp);
    if (arity == 4) return launch(k_mtree_digest<2, kSparse>, bound, kThreads, st, tag, b, o, d, cnt, bp, lp);
    return launch(k_mtree_digest<1, kSparse>, bound, kThreads, st, tag, b, o, d, cnt, bp, lp);
}

cudaError_t launch_mtree_digest(const uint64_t tag[4], const void* below, int arity, void* level, const uint64_t* d,
                                const int* cnt, size_t bound, size_t coop_max, cudaStream_t st, const uint8_t* below_present,
                                uint8_t* level_present) {
    if (below_present)
        return mtree_digest<true>(to_arg(tag), below, arity, level, d, cnt, bound, coop_max, st, below_present, level_present);
    return mtree_digest<false>(to_arg(tag), below, arity, level, d, cnt, bound, coop_max, st, nullptr, nullptr);
}

cudaError_t launch_smtree_keys(const uint64_t* pos, const uint8_t* op, uint32_t n, uint64_t capacity, uint64_t* keys,
                               uint32_t* bpos, unsigned long long* rejected, cudaStream_t st) {
    return launch(k_smtree_keys, n, 256, st, pos, op, n, capacity, keys, bpos, rejected);
}

cudaError_t launch_smtree_leaf_write(const uint64_t* keys, const uint32_t* bpos, uint32_t n, uint64_t sentinel, int arity,
                                     const uint8_t* op, const void* values, void* leaves, uint8_t* present, uint8_t* flag,
                                     uint64_t* parent, cudaStream_t st) {
    return launch(k_smtree_leaf_write, n, 256, st, keys, bpos, n, sentinel, log2_arity(arity), op, values, leaves, present, flag,
                  parent);
}

cudaError_t launch_smtree_seed(uint8_t* present, void* leaves, uint64_t groups, uint64_t capacity, int arity, uint8_t* flag,
                               uint64_t* parent, cudaStream_t st) {
    return launch(k_smtree_seed, groups, 256, st, present, leaves, groups, capacity, log2_arity(arity), flag, parent);
}

cudaError_t launch_smtree_count(const uint8_t* present, uint64_t n, unsigned long long* out, cudaStream_t st) {
    const unsigned grid = n < 4096 * 256 ? (unsigned)((n + 255) / 256) : 4096u;   // at most 4096 blocks: grid-stride
    return launch_grid(k_smtree_count, grid, 256, st, present, n, out);
}

cudaError_t launch_ctree_keys(const uint64_t* pos, const uint8_t* op, uint32_t n, uint64_t max_pos, uint64_t* keys, uint32_t* bpos,
                              unsigned long long* rejected, cudaStream_t st) {
    return launch(k_ctree_keys, n, 256, st, pos, op, n, max_pos, keys, bpos, rejected);
}

cudaError_t launch_ctree_valid(const uint32_t* bpos, uint32_t n, uint8_t* flag, cudaStream_t st) {
    return launch(k_ctree_valid, n, 256, st, bpos, n, flag);
}

cudaError_t launch_ctree_last(const uint64_t* keys, const int* cnt, uint32_t n, uint8_t* flag, cudaStream_t st) {
    return launch(k_ctree_last, n, 256, st, keys, cnt, n, flag);
}

cudaError_t launch_ctree_leaf_changes(const uint32_t* bpos, const int* cnt, uint32_t n, const uint8_t* op, const void* values,
                                      void* cval, uint8_t* cpres, cudaStream_t st) {
    return launch(k_ctree_leaf_changes, n, 256, st, bpos, cnt, n, op, values, cval, cpres);
}

cudaError_t launch_ctree_mark(const uint64_t* lkeys, const uint64_t* lcount, uint64_t s, const uint64_t* ckeys, const int* ccnt,
                              uint32_t nb, const uint8_t* cpres, uint32_t* kept, uint32_t* ins, cudaStream_t st) {
    return launch(k_ctree_mark, s > nb ? s : nb, 256, st, lkeys, lcount, s, ckeys, ccnt, nb, cpres, kept, ins);
}

cudaError_t launch_ctree_scatter(const uint64_t* lkeys, const void* lvals, const uint64_t* lcount, uint64_t s,
                                 const uint64_t* ckeys, const void* cvals, const int* ccnt, uint32_t nb, const uint32_t* kept,
                                 const uint32_t* K, const uint32_t* ins, const uint32_t* I, uint64_t* okeys, void* ovals,
                                 cudaStream_t st) {
    return launch(k_ctree_scatter, s > nb ? s : nb, 256, st, lkeys, lvals, lcount, s, ckeys, cvals, ccnt, nb, kept, K, ins, I,
                  okeys, ovals);
}

cudaError_t launch_ctree_count(const uint64_t* lcount, uint64_t s, uint32_t nb, const uint32_t* kept, const uint32_t* K,
                               const uint32_t* ins, const uint32_t* I, bool level0, uint32_t n, uint64_t* stats, uint32_t* ok,
                               unsigned long long* rejected, cudaStream_t st) {
    return launch_grid(k_ctree_count, 1, 1, st, lcount, s, nb, kept, K, ins, I, level0, n, stats, ok, rejected);
}

cudaError_t launch_ctree_commit(const uint64_t* okeys, const void* ovals, uint64_t s, const uint64_t* stats, const uint32_t* ok,
                                uint64_t* lkeys, void* lvals, uint64_t* lcount, cudaStream_t st) {
    return launch(k_ctree_commit, s, 256, st, okeys, ovals, s, stats, ok, lkeys, lvals, lcount);
}

cudaError_t launch_ctree_gather(const uint64_t* okeys, const void* ovals, const uint64_t* stats, uint64_t s, const uint64_t* pkeys,
                                const int* pcnt, uint32_t nb, int arity, void* groups, uint8_t* gpres, cudaStream_t st) {
    return launch(k_ctree_gather, nb, 256, st, okeys, ovals, stats, s, pkeys, pcnt, nb, log2_arity(arity), groups, gpres);
}

cudaError_t launch_ctree_iota(uint64_t* d, uint32_t n, cudaStream_t st) {
    return launch(k_ctree_iota, n, 256, st, d, n);
}

cudaError_t launch_ctree_open(const uint64_t* keys, const void* values, const uint64_t* count, const uint64_t* pos, size_t n,
                              int arity, uint32_t depth, const OpenLevels& lv, void* paths, cudaStream_t st) {
    return launch(k_ctree_open, n * depth, 256, st, keys, values, count, pos, n, log2_arity(arity), depth, lv, paths);
}

cudaError_t launch_merkle_verify(const uint64_t tag[4], const uint64_t root[4], const void* leaf_items,
                                 const uint64_t* leaf_idx, const void* paths, size_t n, int arity, uint32_t depth,
                                 uint8_t* ok, unsigned long long* n_failed, cudaStream_t st) {
    if (arity == 4)
        return launch(k_merkle_verify<2>, n, kThreads, st, to_arg(tag), to_arg(root), leaf_items, leaf_idx, paths, n, depth, ok,
                      n_failed);
    return launch(k_merkle_verify<1>, n, kThreads, st, to_arg(tag), to_arg(root), leaf_items, leaf_idx, paths, n, depth, ok,
                  n_failed);
}

cudaError_t launch_varlen_keys(const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_scalars, uint32_t max_len,
                               uint32_t fixed_len, uint32_t* keys, uint32_t* vals, unsigned long long* rejected, cudaStream_t st) {
    return launch(k_varlen_keys<0>, n, 256, st, offsets, n, base, n_scalars, max_len, fixed_len, keys, vals, rejected);
}

cudaError_t launch_crypt_varlen_keys(bool decrypt, const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_scalars,
                                     uint32_t max_len, uint32_t* keys, uint32_t* vals, unsigned long long* rejected,
                                     cudaStream_t st) {
    if (decrypt) return launch(k_varlen_keys<2>, n, 256, st, offsets, n, base, n_scalars, max_len, 0, keys, vals, rejected);
    return launch(k_varlen_keys<1>, n, 256, st, offsets, n, base, n_scalars, max_len, 0, keys, vals, rejected);
}

cudaError_t launch_crypt_varlen(bool decrypt, const void* tags, const void* src, uint64_t base, const uint64_t* offsets,
                                const uint32_t* lens, const uint32_t* perm, uint32_t n, const void* secret_uv, const void* nonce,
                                void* dst, uint8_t* ok, unsigned long long* n_failed, size_t coop_max, cudaStream_t st) {
    if (n <= coop_max) {
        if (decrypt)
            return launch_grid(k_crypt_varlen_coop<true>, coop_grid(n), kThreads, st, tags, src, base, offsets, lens, perm, n,
                               secret_uv, nonce, dst, ok, n_failed);
        return launch_grid(k_crypt_varlen_coop<false>, coop_grid(n), kThreads, st, tags, src, base, offsets, lens, perm, n,
                           secret_uv, nonce, dst, nullptr, nullptr);
    }
    if (decrypt)
        return launch(k_crypt_varlen<true>, n, kThreads, st, tags, src, base, offsets, lens, perm, n, secret_uv, nonce, dst, ok,
                      n_failed);
    return launch(k_crypt_varlen<false>, n, kThreads, st, tags, src, base, offsets, lens, perm, n, secret_uv, nonce, dst, nullptr,
                  nullptr);
}

cudaError_t launch_digest_varlen(const void* tags, const void* in, uint64_t base, const uint64_t* offsets, const uint32_t* lens,
                                 const uint32_t* perm, uint32_t n, void* out, uint32_t out_len, size_t coop_max, cudaStream_t st) {
    if (n <= coop_max)
        return launch_grid(k_sponge_digest_varlen_coop, coop_grid(n), kThreads, st, tags, in, base, offsets, lens, perm, n, out,
                           out_len);
    return launch(k_sponge_digest_varlen, n, kThreads, st, tags, in, base, offsets, lens, perm, n, out, out_len);
}

// ---- BlsScalar::hash_to_scalar on the device (p252_hash_to_scalar_batch, p252_scalars_from_bytes_wide) -------------
// BLAKE2b-512 (RFC 7693; host::Blake2b in host_field.h) of a byte string, then from_bytes_wide.  Public data only.

// BlsScalar::from_bytes_wide of the 64 little-endian bytes w: (lo + hi 2^256) mod p in Montgomery form, computed as
// host::from_bytes_wide does, lo R^2 + hi R^3 with two Montgomery products.  lo and hi are raw 256-bit values (up to
// 2^256 - 1, about 2.2 p).  montmul's contract is on the row operand alone (x + p <= 2^256, here R^2 or R^3 < p); the
// column operand may be any y < 2^256.  So lo and hi need no pre-reduction (no fr_condsub255): each product is
// (x y + m p) / 2^256 < (p 2^256 + 2^256 p) / 2^256 = 2p, and one conditional subtraction makes it canonical.
__device__ __forceinline__ void fr_from_bytes_wide(uint32_t (&r)[8], const uint64_t (&w)[8]) {
    const uint32_t r2[8] = {0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u,
                            0x0748d9d9u};   // R^2 mod p
    const uint32_t r3[8] = {0x439b73afu, 0xc62c1807u, 0x8cf06990u, 0x1b3e0d18u, 0xc7b5f418u, 0x73d13c71u, 0xc8db33e9u,
                            0x6e2a5bb9u};   // R^3 mod p
    uint32_t lo[8], hi[8], a[8], c[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        lo[2 * k] = (uint32_t)w[k], lo[2 * k + 1] = (uint32_t)(w[k] >> 32);
        hi[2 * k] = (uint32_t)w[4 + k], hi[2 * k + 1] = (uint32_t)(w[4 + k] >> 32);
    }
    montmul(a, r2, lo);        // lo R mod p, < 2p
    fr_condsub(a);
    montmul(c, r3, hi);        // hi 2^256 R mod p, < 2p
    fr_condsub(c);
    fr_add_mod(r, a, c);
}

// 64-bit rotations of the G function: 32 is a word swap, 24 and 16 are two funnel shifts, 63 (a rotation left by 1) two
// left funnel shifts
__device__ __forceinline__ uint64_t b2_rotr32(uint64_t x) { return (x << 32) | (x >> 32); }
template <int kN>
__device__ __forceinline__ uint64_t b2_rotr(uint64_t x) {   // 0 < kN < 32
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__funnelshift_r(hi, lo, kN) << 32) | __funnelshift_r(lo, hi, kN);
}
__device__ __forceinline__ uint64_t b2_rotr63(uint64_t x) {
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__funnelshift_l(lo, hi, 1) << 32) | __funnelshift_l(hi, lo, 1);
}

// The BLAKE2b compression F(h, m, t, last), fully unrolled: the SIGMA schedule is spelled out per round, so every
// message word is a compile-time register.  t is the byte counter's low word; its high word is 0, a message being
// shorter than 2^64 bytes.
__device__ __forceinline__ void blake2b_compress(uint64_t (&h)[8], const uint64_t (&m)[16], uint64_t t, bool last) {
    uint64_t v[16] = {h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7],
                      0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                      0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    v[12] ^= t;
    if (last) v[14] = ~v[14];
#define P252_B2G(a, b, c, d, x, y)              \
    v[a] = v[a] + v[b] + m[x];                  \
    v[d] = b2_rotr32(v[d] ^ v[a]);              \
    v[c] = v[c] + v[d];                         \
    v[b] = b2_rotr<24>(v[b] ^ v[c]);            \
    v[a] = v[a] + v[b] + m[y];                  \
    v[d] = b2_rotr<16>(v[d] ^ v[a]);            \
    v[c] = v[c] + v[d];                         \
    v[b] = b2_rotr63(v[b] ^ v[c]);
#define P252_B2ROUND(s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15) \
    P252_B2G(0, 4, 8, 12, s0, s1)                                                          \
    P252_B2G(1, 5, 9, 13, s2, s3)                                                          \
    P252_B2G(2, 6, 10, 14, s4, s5)                                                         \
    P252_B2G(3, 7, 11, 15, s6, s7)                                                         \
    P252_B2G(0, 5, 10, 15, s8, s9)                                                         \
    P252_B2G(1, 6, 11, 12, s10, s11)                                                       \
    P252_B2G(2, 7, 8, 13, s12, s13)                                                        \
    P252_B2G(3, 4, 9, 14, s14, s15)
    P252_B2ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    P252_B2ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
    P252_B2ROUND(11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4)
    P252_B2ROUND(7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8)
    P252_B2ROUND(9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13)
    P252_B2ROUND(2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9)
    P252_B2ROUND(12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11)
    P252_B2ROUND(13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10)
    P252_B2ROUND(6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5)
    P252_B2ROUND(10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0)
    P252_B2ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    P252_B2ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
#undef P252_B2ROUND
#undef P252_B2G
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
}

// The 16 bytes at the 16-byte aligned address p, those outside [lo, hi) read as zero: one LDG.128 when all 16 lie
// inside, otherwise byte loads of the inside ones only
__device__ __forceinline__ uint4 ldg128_within(uintptr_t p, uintptr_t lo, uintptr_t hi) {
    if (p >= lo && p + 16 <= hi) return ldg128(reinterpret_cast<const void*>(p));
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int b = 0; b < 16; ++b)
        if (p + b >= lo && p + b < hi) w[b >> 2] |= (uint32_t)*reinterpret_cast<const uint8_t*>(p + b) << (8 * (b & 3));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// One message block as 16 little-endian words: the r <= 128 bytes at src (any alignment), zero past them.  The aligned
// 16-byte loads that cover them never leave the caller's buffer [lo, hi) (ldg128_within); the block is then shifted
// down by src mod 16 bytes -- whole words by selects, the rest by funnel shifts -- so no array is indexed at run time.
__device__ __forceinline__ void b2_load_block(uint64_t (&m)[16], uintptr_t src, uint32_t r, uintptr_t lo, uintptr_t hi) {
    const uintptr_t a = src & ~(uintptr_t)15;
    const uint32_t off = (uint32_t)(src & 15);
    uint32_t w[36];
#pragma unroll
    for (int c = 0; c < 9; ++c) {
        const uint4 x = (uint32_t)(16 * c) < off + r ? ldg128_within(a + 16 * c, lo, hi) : make_uint4(0, 0, 0, 0);
        w[4 * c] = x.x, w[4 * c + 1] = x.y, w[4 * c + 2] = x.z, w[4 * c + 3] = x.w;
    }
    const bool q1 = (off & 4) != 0, q2 = (off & 8) != 0;
    const uint32_t sh = (off & 3) * 8;
    uint32_t y[35], z[33];
#pragma unroll
    for (int k = 0; k < 35; ++k) y[k] = q1 ? w[k + 1] : w[k];
#pragma unroll
    for (int k = 0; k < 33; ++k) z[k] = q2 ? y[k + 2] : y[k];
    uint32_t b[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) b[k] = __funnelshift_r(z[k], z[k + 1], sh);
    if (r < 128) {                                         // the last block of a message: zero past its end
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const uint32_t keep = r > 4u * k ? r - 4u * k : 0u;   // message bytes in word k
            b[k] = keep >= 4 ? b[k] : b[k] & ((1u << (8 * keep)) - 1u);
        }
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) m[k] = ((uint64_t)b[2 * k + 1] << 32) | b[2 * k];
}

// k_hash_to_scalar: one message per thread.  Item i is bytes[offsets[i] - base .. offsets[i+1] - base) of n_bytes; it
// is valid iff offsets[i] - base <= offsets[i+1] - base <= n_bytes and its length is <= max_len, and no byte outside
// [bytes, bytes + n_bytes) is read.  out[i] = hash_to_scalar (Montgomery), a zero row for an invalid item, which is
// counted into *rejected when that is given.  BLAKE2b as host::Blake2b: parameter block 0x01010040, the byte counter
// after each block, the last block flagged final even when it is full, the empty string one zero block with counter 0.
// kSorted: thread t hashes item perm[n - 1 - t] of the order k_hash_to_scalar_keys and the sort made (longest first,
// so that a warp runs messages of nearly equal block counts and the longest start first); otherwise item t.
template <bool kSorted>
__global__ void __launch_bounds__(256) k_hash_to_scalar(const uint8_t* __restrict__ bytes, uint64_t base, uint64_t n_bytes,
                                                        const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ perm,
                                                        uint32_t n, uint32_t max_len, uint8_t* __restrict__ out,
                                                        unsigned long long* __restrict__ rejected) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = kSorted ? perm[n - 1 - t] : t;
    const uint64_t a = offsets[i] - base, b = offsets[i + 1] - base, len = b - a;
    const bool ok = a <= b && b <= n_bytes && len <= max_len;
    if (rejected) warp_count(rejected, !ok);
    uint32_t r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (ok) {
        uint64_t h[8] = {0x6a09e667f3bcc908ull ^ 0x01010040ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull,
                         0xa54ff53a5f1d36f1ull, 0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull,
                         0x5be0cd19137e2179ull};
        const uintptr_t lo = reinterpret_cast<uintptr_t>(bytes), hi = lo + n_bytes, src = lo + a;
        const uint32_t L = (uint32_t)len, nblk = L ? (L + 127) / 128 : 1u;
#pragma unroll 1
        for (uint32_t j = 0; j < nblk; ++j) {
            const uint32_t left = L - 128 * j, take = left < 128 ? left : 128u;
            uint64_t m[16];
            b2_load_block(m, src + 128 * j, take, lo, hi);
            blake2b_compress(h, m, 128ull * j + take, j + 1 == nblk);
        }
        fr_from_bytes_wide(r, h);
    }
    store_fr(out + (size_t)i * 32, r);
}

// keys[i] = the block count max(1, ceil(len / 128)) of a valid item (as k_hash_to_scalar decides it), 0 for an invalid
// one (counted into *rejected); vals[i] = i
__global__ void __launch_bounds__(256) k_hash_to_scalar_keys(const uint64_t* __restrict__ offsets, uint32_t n, uint64_t base,
                                                             uint64_t n_bytes, uint32_t max_len, uint32_t* __restrict__ keys,
                                                             uint32_t* __restrict__ vals,
                                                             unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t a = offsets[i] - base, b = offsets[i + 1] - base, len = b - a;
    const bool ok = a <= b && b <= n_bytes && len <= max_len;
    keys[i] = ok ? (len ? (uint32_t)((len + 127) / 128) : 1u) : 0u;
    vals[i] = i;
    if (rejected) warp_count(rejected, !ok);
}

// rows of 64 bytes -> BlsScalar::from_bytes_wide, one thread per row
__global__ void __launch_bounds__(256) k_from_bytes_wide(const uint8_t* __restrict__ in, size_t n, uint8_t* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t w[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 x = ldg128(in + i * 64 + 16 * q);
        w[2 * q] = ((uint64_t)x.y << 32) | x.x;
        w[2 * q + 1] = ((uint64_t)x.w << 32) | x.z;
    }
    uint32_t r[8];
    fr_from_bytes_wide(r, w);
    store_fr(out + i * 32, r);
}

// ---- mixed digest batches (p252_hash_batch_mixed): per-item domain, input and output lengths, truncation --------------
// k_mixed_keys: one thread per item.  Item i is Hash::new(mode[i] & 3), update(in[offsets[i] - base .. offsets[i+1] - base))
// (n_scalars scalars), output_len(out_len), finalize() or (mode[i] & 0x80) finalize_truncated(), written to the rows
// [out_offsets[i] - obase, out_offsets[i+1] - obase) of `out` (n_out rows).  Valid: no mode bit outside 0x83, both ranges
// non-decreasing and inside their buffers, a Merkle domain with len == arity and out_len == 1, 1 <= len <= max_len and
// 1 <= out_len <= max_out_len -- the rules of p252_hash_tag.  Every later access of `in` and `out` is bounded by this.
// A valid item gets key = its step count ceil(len / 4) + ceil(out_len / 4), desc = (len, out_len | truncated << 31) and
// its tag: hash_to_scalar(BE32(0x80000000 | len) || BE32(out_len) || BE64(domain_sep)), one BLAKE2b block, derived here
// so that the sponge kernels keep their register budget.  An invalid item gets key 0, desc (0, 0), a zero tag and, when
// its output range is valid, zero rows; it is counted into *rejected.  vals[i] = i.
__global__ void __launch_bounds__(256) k_mixed_keys(const uint8_t* __restrict__ mode, const uint64_t* __restrict__ offsets,
                                                    uint64_t base, uint64_t n_scalars, const uint64_t* __restrict__ out_offsets,
                                                    uint64_t obase, uint64_t n_out, uint32_t n, uint32_t max_len,
                                                    uint32_t max_out_len, uint8_t* __restrict__ out, uint32_t* __restrict__ keys,
                                                    uint32_t* __restrict__ vals, uint8_t* __restrict__ tags,
                                                    uint2* __restrict__ desc, unsigned long long* __restrict__ rejected) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t m = mode[i], dom = m & 3u;
    const uint64_t a = offsets[i] - base, b = offsets[i + 1] - base, len = b - a;
    const uint64_t oa = out_offsets[i] - obase, ob = out_offsets[i + 1] - obase, olen = ob - oa;
    const bool out_ok = oa <= ob && ob <= n_out;
    const uint64_t arity = dom == 0 ? 4u : (dom == 1 ? 2u : 0u);   // P252_DOMAIN_MERKLE4, P252_DOMAIN_MERKLE2
    const bool ok = (m & ~0x83u) == 0 && a <= b && b <= n_scalars && out_ok && (arity == 0 || (len == arity && olen == 1)) &&
                    len >= 1 && olen >= 1 && len <= max_len && olen <= max_out_len;
    if (rejected) warp_count(rejected, !ok);
    uint32_t r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (ok) {
        // u64::from(Domain), src/hash.rs:43-55
        const uint64_t dsep = dom == 0 ? 0xfull : (dom == 1 ? 0x3ull : (dom == 2 ? 0x100000000ull : 0ull));
        const uint32_t w0 = 0x80000000u | (uint32_t)len, w1 = (uint32_t)olen;
        uint64_t msg[16] = {};
        msg[0] = ((uint64_t)__byte_perm(w1, 0, 0x0123) << 32) | __byte_perm(w0, 0, 0x0123);   // big-endian words
        msg[1] = ((uint64_t)__byte_perm((uint32_t)dsep, 0, 0x0123) << 32) | __byte_perm((uint32_t)(dsep >> 32), 0, 0x0123);
        uint64_t h[8] = {0x6a09e667f3bcc908ull ^ 0x01010040ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull,
                         0xa54ff53a5f1d36f1ull, 0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull,
                         0x5be0cd19137e2179ull};
        blake2b_compress(h, msg, 16, true);
        fr_from_bytes_wide(r, h);
    }
    store_fr(tags + (size_t)i * 32, r);
    keys[i] = ok ? (uint32_t)((len + 3) / 4 + (olen + 3) / 4) : 0u;
    vals[i] = i;
    desc[i] = ok ? make_uint2((uint32_t)len, (uint32_t)olen | (m & 0x80u) << 24) : make_uint2(0, 0);
    if (!ok && out_ok)                                     // rejected: zero rows
        for (uint64_t q = oa; q < ob; ++q) store_fr(out + q * 32, r);
}

cudaError_t launch_mixed_keys(const uint8_t* mode, const uint64_t* offsets, uint64_t base, uint64_t n_scalars,
                              const uint64_t* out_offsets, uint64_t obase, uint64_t n_out, uint32_t n, uint32_t max_len,
                              uint32_t max_out_len, void* out, uint32_t* keys, uint32_t* vals, void* tags, uint2* desc,
                              unsigned long long* rejected, cudaStream_t st) {
    return launch(k_mixed_keys, n, 256, st, mode, offsets, base, n_scalars, out_offsets, obase, n_out, n, max_len, max_out_len,
                  out, keys, vals, tags, desc, rejected);
}

cudaError_t launch_digest_mixed(const void* tags, const uint2* desc, const void* in, uint64_t base, const uint64_t* offsets,
                                uint64_t obase, const uint64_t* out_offsets, const uint32_t* perm, uint32_t n, void* out,
                                size_t coop_max, cudaStream_t st) {
    if (n <= coop_max)
        return launch_grid(k_sponge_digest_mixed_coop, coop_grid(n), kThreads, st, tags, desc, in, base, offsets, obase,
                           out_offsets, perm, n, out);
    return launch(k_sponge_digest_mixed, n, kThreads, st, tags, desc, in, base, offsets, obase, out_offsets, perm, n, out);
}

cudaError_t launch_hash_to_scalar(const void* bytes, uint64_t base, uint64_t n_bytes, const uint64_t* offsets,
                                  const uint32_t* perm, uint32_t n, uint32_t max_len, void* out, unsigned long long* rejected,
                                  cudaStream_t st) {
    if (perm) return launch(k_hash_to_scalar<true>, n, 256, st, bytes, base, n_bytes, offsets, perm, n, max_len, out, rejected);
    return launch(k_hash_to_scalar<false>, n, 256, st, bytes, base, n_bytes, offsets, nullptr, n, max_len, out, rejected);
}

cudaError_t launch_hash_to_scalar_keys(const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_bytes, uint32_t max_len,
                                       uint32_t* keys, uint32_t* vals, unsigned long long* rejected, cudaStream_t st) {
    return launch(k_hash_to_scalar_keys, n, 256, st, offsets, n, base, n_bytes, max_len, keys, vals, rejected);
}

cudaError_t launch_from_bytes_wide(const void* in, size_t n, void* out, cudaStream_t st) {
    return launch(k_from_bytes_wide, n, 256, st, in, n, out);
}

uint32_t wide_mul_per_permutation() { return (uint32_t)kWideMulPerPerm; }
uint32_t dfma_per_permutation() { return (uint32_t)kDfmaPerPerm; }

void kernel_launch_shape(int* threads_per_block, int* min_blocks_per_sm) {
    *threads_per_block = kThreads;
    *min_blocks_per_sm = kMinBlocks;
}

}  // namespace p252
