// Host-callable launchers of the sm_90a kernels (kernels.cu).  Internal to the library; the public
// boundary is include/poseidon252_b200.h.  All pointers are DEVICE pointers, 16-byte aligned;
// scalars are BlsScalar.0 (4 x u64 LE limbs, Montgomery form, < p).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace p252 {

cudaError_t launch_permute(void* states, size_t n, bool dense, size_t coop_max, cudaStream_t st);
// coop_max: batches of at most this many items run the lane-split (5 threads per state) kernel
cudaError_t launch_digest(const uint64_t tag[4], const void* in, size_t n, uint32_t in_len, void* out,
                          uint32_t out_len, bool truncate, size_t coop_max, cudaStream_t st);
cudaError_t launch_convert(const void* in, size_t n, void* out, uint8_t* ok, bool from_bytes, cudaStream_t st);
cudaError_t launch_encrypt(const uint64_t tag[4], const void* msg, size_t n, uint32_t L, const void* secret_uv,
                           const void* nonce, void* cipher, cudaStream_t st);
// n_failed (device pointer, may be null): incremented by the number of items whose authentication failed
cudaError_t launch_decrypt(const uint64_t tag[4], const void* cipher, size_t n, uint32_t L, const void* secret_uv,
                           const void* nonce, void* msg, uint8_t* ok, unsigned long long* n_failed, cudaStream_t st);
// Merkle openings over leaves + internal levels bottom-up (arity 2 or 4): level l >= 1 starts at slot off[l] of
// `nodes`; m[l] nodes of level l are occupied (m[0] = occupied leaves), slots at or beyond m[l] read as zero
constexpr int kMaxDepth = 64;
struct OpenLevels {
    uint64_t off[kMaxDepth];
    uint64_t m[kMaxDepth];
};
// present (optional, p252_smtree): leaf idx must also have present[idx] != 0, otherwise its opening is all zero
cudaError_t launch_merkle_open(const void* leaves, const void* nodes, const uint64_t* leaf_idx, size_t n, int arity,
                               uint32_t depth, const OpenLevels& lv, void* paths, cudaStream_t st,
                               const uint8_t* present = nullptr);
// Fixed-height tree updates (p252_mtree_update).  keys: overwrite i -> idx[i] (>= n_old: sentinel n_new, counted into
// *rejected), append j -> n_old + j; pos[i] = i
cudaError_t launch_mtree_keys(const uint64_t* idx, uint32_t n_upd, uint64_t n_old, uint32_t total, uint64_t* keys,
                              uint32_t* pos, unsigned long long* rejected, cudaStream_t st);
// over stably sorted (keys, pos): last write per key -> leaves[key]; level-1 candidates flag / parent = key / arity
cudaError_t launch_mtree_leaf_write(const uint64_t* keys, const uint32_t* pos, uint32_t total, uint64_t sentinel, int arity,
                                    const void* values, uint32_t n_upd, const void* append, void* leaves, uint8_t* flag,
                                    uint64_t* parent, cudaStream_t st);
// candidates of the next level from a sorted dirty set d[0..*cnt), cnt <= bound
cudaError_t launch_mtree_parents(const uint64_t* d, const int* cnt, uint32_t bound, int arity, uint8_t* flag, uint64_t* parent,
                                 cudaStream_t st);
// level[d[k]] = Hash::digest(Domain::Merkle{arity}, below[d[k]*arity .. +arity]) for k < *cnt <= bound; lane-split kernel
// when bound <= coop_max.  With presence bytes (p252_smtree / p252_ctree, indexed like below / level): an empty group
// stores value 0 / presence 0, any other its digest / presence 1
cudaError_t launch_mtree_digest(const uint64_t tag[4], const void* below, int arity, void* level, const uint64_t* d,
                                const int* cnt, size_t bound, size_t coop_max, cudaStream_t st,
                                const uint8_t* below_present = nullptr, uint8_t* level_present = nullptr);
// Sparse fixed-height trees (p252_smtree).  keys: pos[i] for a valid item (pos < capacity, op NULL or 0/1), else the
// sentinel `capacity` (counted into *rejected); bpos[i] = i
cudaError_t launch_smtree_keys(const uint64_t* pos, const uint8_t* op, uint32_t n, uint64_t capacity, uint64_t* keys,
                               uint32_t* bpos, unsigned long long* rejected, cudaStream_t st);
// over stably sorted (keys, bpos): the last op per key is applied (insert: value + presence 1, remove: zero + presence 0);
// level-1 candidates flag / parent = key / arity
cudaError_t launch_smtree_leaf_write(const uint64_t* keys, const uint32_t* bpos, uint32_t n, uint64_t sentinel, int arity,
                                     const uint8_t* op, const void* values, void* leaves, uint8_t* present, uint8_t* flag,
                                     uint64_t* parent, cudaStream_t st);
// build: normalise leaf presence (slots >= capacity absent), zero absent leaves, flag[g] = group g has a present leaf,
// parent[g] = g, for the `groups` leaf groups
cudaError_t launch_smtree_seed(uint8_t* present, void* leaves, uint64_t groups, uint64_t capacity, int arity, uint8_t* flag,
                               uint64_t* parent, cudaStream_t st);
// *out += non-zero bytes of present[0, n)
cudaError_t launch_smtree_count(const uint8_t* present, uint64_t n, unsigned long long* out, cudaStream_t st);
// Compact sparse trees (p252_ctree).  A change list is (keys, values, present) sorted by distinct key, count on the device;
// a level is (keys, values) sorted, count on the device, s slots.  keys: keys[i] = pos[i], bpos[i] = i | (invalid << 31)
// (invalid: pos > max_pos or op not NULL / 0 / 1, counted into *rejected)
cudaError_t launch_ctree_keys(const uint64_t* pos, const uint8_t* op, uint32_t n, uint64_t max_pos, uint64_t* keys, uint32_t* bpos,
                              unsigned long long* rejected, cudaStream_t st);
// flag[k] = bit 31 of bpos[k] is clear
cudaError_t launch_ctree_valid(const uint32_t* bpos, uint32_t n, uint8_t* flag, cudaStream_t st);
// flag[i] = i < *cnt and i is the last of its run of equal keys
cudaError_t launch_ctree_last(const uint64_t* keys, const int* cnt, uint32_t n, uint8_t* flag, cudaStream_t st);
// level 0's change values / presence from the batch positions of the last operation per position
cudaError_t launch_ctree_leaf_changes(const uint32_t* bpos, const int* cnt, uint32_t n, const uint8_t* op, const void* values,
                                      void* cval, uint8_t* cpres, cudaStream_t st);
// kept[t < s]: old entry t survives (present, no change with its key); ins[t < nb]: change t inserts
cudaError_t launch_ctree_mark(const uint64_t* lkeys, const uint64_t* lcount, uint64_t s, const uint64_t* ckeys, const int* ccnt,
                              uint32_t nb, const uint8_t* cpres, uint32_t* kept, uint32_t* ins, cudaStream_t st);
// merge into (okeys, ovals) with K / I the exclusive scans of kept / ins; writes at or past s are dropped
cudaError_t launch_ctree_scatter(const uint64_t* lkeys, const void* lvals, const uint64_t* lcount, uint64_t s,
                                 const uint64_t* ckeys, const void* cvals, const int* ccnt, uint32_t nb, const uint32_t* kept,
                                 const uint32_t* K, const uint32_t* ins, const uint32_t* I, uint64_t* okeys, void* ovals,
                                 cudaStream_t st);
// stats = {old count, new count}; level0: *ok = new count <= s, and a refusal sets *rejected = n
cudaError_t launch_ctree_count(const uint64_t* lcount, uint64_t s, uint32_t nb, const uint32_t* kept, const uint32_t* K,
                               const uint32_t* ins, const uint32_t* I, bool level0, uint32_t n, uint64_t* stats, uint32_t* ok,
                               unsigned long long* rejected, cudaStream_t st);
// if *ok: the level and its count become the merged list, vacated slots zeroed
cudaError_t launch_ctree_commit(const uint64_t* okeys, const void* ovals, uint64_t s, const uint64_t* stats, const uint32_t* ok,
                                uint64_t* lkeys, void* lvals, uint64_t* lcount, cudaStream_t st);
// dense groups (arity scalars, absent 0) and presence bytes of the dirty parents pkeys[0..*pcnt) from the merged level
cudaError_t launch_ctree_gather(const uint64_t* okeys, const void* ovals, const uint64_t* stats, uint64_t s, const uint64_t* pkeys,
                                const int* pcnt, uint32_t nb, int arity, void* groups, uint8_t* gpres, cudaStream_t st);
// d[t] = t
cudaError_t launch_ctree_iota(uint64_t* d, uint32_t n, cudaStream_t st);
// openings in the format of launch_merkle_open; lv.off[l] = first slot of level l; an absent leaf gets an all-zero opening
cudaError_t launch_ctree_open(const uint64_t* keys, const void* values, const uint64_t* count, const uint64_t* pos, size_t n,
                              int arity, uint32_t depth, const OpenLevels& lv, void* paths, cudaStream_t st);
cudaError_t launch_merkle_verify(const uint64_t tag[4], const uint64_t root[4], const void* leaf_items,
                                 const uint64_t* leaf_idx, const void* paths, size_t n, int arity, uint32_t depth,
                                 uint8_t* ok, unsigned long long* n_failed, cudaStream_t st);
// Variable-length digests (p252_hash_batch_varlen).  Item i = in[offsets[i] - base .. offsets[i+1] - base) of n_scalars.
// keys: len for a valid item (1 <= len <= max_len, len == fixed_len unless fixed_len == 0, range inside in), 0 for an
// invalid one (counted into *rejected); vals[i] = i
cudaError_t launch_varlen_keys(const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_scalars, uint32_t max_len,
                               uint32_t fixed_len, uint32_t* keys, uint32_t* vals, unsigned long long* rejected, cudaStream_t st);
// over the keys sorted ascending (lens) with their values (perm): out[perm[k]] = digest with tag tags[lens[k]] of item
// perm[k] (out_len scalars, a zero row for lens[k] == 0); lane-split kernel when n <= coop_max
cudaError_t launch_digest_varlen(const void* tags, const void* in, uint64_t base, const uint64_t* offsets, const uint32_t* lens,
                                 const uint32_t* perm, uint32_t n, void* out, uint32_t out_len, size_t coop_max, cudaStream_t st);
// Variable-length encrypt / decrypt (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen).  keys: the message length L
// of a valid item (a0 <= a <= b <= an <= n_scalars with a0 / an the first / last offset minus base; encrypt 1 <= b - a <=
// max_len, decrypt 2 <= b - a <= max_len + 1 and the message range inside the output), 0 for an invalid one (counted into
// *rejected); vals[i] = i
cudaError_t launch_crypt_varlen_keys(bool decrypt, const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_scalars,
                                     uint32_t max_len, uint32_t* keys, uint32_t* vals, unsigned long long* rejected,
                                     cudaStream_t st);
// over the keys sorted ascending (lens) with their values (perm): item perm[k] reads src[offsets[i] - base ..) and writes
// dst from offsets[i] - offsets[0] + i (encrypt, L + 1 scalars) or - i (decrypt, L scalars; ok[i], failures counted into
// *n_failed); tags[L] = p252_encryption_tag(L); a rejected item (L = 0) writes nothing but ok[i] = 0.  Lane-split kernel
// when n <= coop_max
cudaError_t launch_crypt_varlen(bool decrypt, const void* tags, const void* src, uint64_t base, const uint64_t* offsets,
                                const uint32_t* lens, const uint32_t* perm, uint32_t n, const void* secret_uv, const void* nonce,
                                void* dst, uint8_t* ok, unsigned long long* n_failed, size_t coop_max, cudaStream_t st);
// JubJub key exchange (p252_dhke_batch): shared_uv[i] = [secret[i]] pub[i] as (u, v), one thread per item; *_bcast: the
// operand is one item read by all.  ok[i] = item valid (secret < r_J, u, v < p, on the curve); an invalid item writes
// (0, 0) and is counted into *n_invalid (device pointer, may be null)
cudaError_t launch_dhke(const void* secret, bool secret_bcast, const void* pub, bool pub_bcast, size_t n, void* shared_uv,
                        uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// after a fused encrypt / decrypt: items with valid[i] == 0 get ok[i] = 0 and a zeroed row of `row` scalars of out (encrypt
// also sets ok[i] = 1 for the valid ones); count (device, may be null) += invalid items (encrypt) or invalid items
// launch_decrypt had not already counted as failures (decrypt)
cudaError_t launch_dhke_fix(bool decrypt, const uint8_t* valid, size_t n, void* out, uint32_t row, uint8_t* ok,
                            unsigned long long* count, cudaStream_t st);
// Fixed-base JubJub scalar multiplication (p252_fixed_base_batch): a table of kFixedBaseTableBytes built once per base
// (base_uv: (u, v) Montgomery limbs, on the curve, read on the host at launch), then out_uv[i] = [secret[i]] base, one
// thread per item; ok[i] = secret < r_J, an invalid item writes (0, 0) and is counted into *n_invalid (device, may be null)
constexpr size_t kFixedBaseTableBytes = 64 * 8 * 96;
cudaError_t launch_fixed_base_table(const uint64_t base_uv[8], void* table, cudaStream_t st);
cudaError_t launch_fixed_base(const void* secret, size_t n, const void* table, void* out_uv, uint8_t* ok,
                              unsigned long long* n_invalid, cudaStream_t st);
// Stealth addresses (p252_stealth_address_batch / p252_stealth_owns_batch), one thread per item: h[i] is the truncated
// digest of the item's shared point (4 x u64 < 2^250), valid[i] its validity from launch_dhke, table the fixed-base table
// of G.  Counters are device pointers and may be null.
// owns: owned[i] = valid[i], both coordinates of note_pk[i] < p and note_pk[i] == [h[i]] G + B, with B given in Niels
// form b_niels = (v - u, v + u, 2d u v), 3 x 4 u64 Montgomery limbs; *n_owned += owned items, *n_invalid += invalid ones
cudaError_t launch_stealth_owns(const void* h, size_t n, const void* table, const uint64_t b_niels[12], const void* note_pk,
                                const uint8_t* valid, uint8_t* owned, unsigned long long* n_owned,
                                unsigned long long* n_invalid, cudaStream_t st);
// derive: note_pk[i] = [h[i]] G + B_uv[B_bcast ? 0 : i]; ok[i] = valid[i] and B a curve point with u, v < p.  An item
// with ok = 0 gets a zeroed note_pk row and a zeroed R_uv row and is counted into *n_invalid
cudaError_t launch_stealth_derive(const void* h, size_t n, const void* table, const void* B_uv, bool B_bcast,
                                  const uint8_t* valid, void* R_uv, void* note_pk, uint8_t* ok, unsigned long long* n_invalid,
                                  cudaStream_t st);
// Note nullifiers (p252_nullifier_batch), one thread per item: h[i] is the truncated digest of the item's shared point
// [a] R (4 x u64 < 2^250), valid[i] its validity from launch_dhke, table the fixed-base table of G'.  rows[i] =
// [pk'.u, pk'.v, pos[i] as a field element] (96 bytes, Montgomery), pk' = [(h[i] + b) mod r_J] G' with b =
// b[b_bcast ? 0 : i]; valid[i] &= b < r_J (an out-of-range b enters the sum as 0)
cudaError_t launch_nullifier_key(const void* h, const void* b, bool b_bcast, const uint64_t* pos, size_t n, const void* table,
                                 void* rows, uint8_t* valid, cudaStream_t st);
// Schnorr signatures (p252_schnorr_sign_batch / p252_schnorr_verify_batch), challenge c = the truncated digest of the row
// [R.u, R.v, m] (4 x u64 < 2^250).  Counters are device pointers and may be null.
// pack: rows[i] = [R.u, R.v, m] (96 bytes, a value >= p written as 0); flag[i] = (and_flag ? flag[i] : 1) and all three < p
cudaError_t launch_schnorr_pack(const void* R_uv, const void* msg, size_t n, void* rows, uint8_t* flag, bool and_flag,
                                cudaStream_t st);
// sign: ok[i] &= sk[sk_bcast ? 0 : i] < r_J; u_out[i] = (r[i] - c[i] sk) mod r_J.  An item with ok = 0 gets a zeroed u row
// and a zeroed R_uv row and is counted into *n_invalid
cudaError_t launch_schnorr_sign(const void* sk, bool sk_bcast, const void* r, const void* c, size_t n, void* u_out, void* R_uv,
                                uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// verify: verified[i] = valid[i], u[i] < r_J, pk[pk_bcast ? 0 : i] a curve point with u, v < p, and [u[i]] G + [c[i]] pk ==
// R_uv[i] (table: the fixed-base table of G); *n_verified += verified items, *n_invalid += invalid ones
cudaError_t launch_schnorr_verify(const void* pk, bool pk_bcast, const void* u, const void* R_uv, const void* c,
                                  const uint8_t* valid, size_t n, const void* table, uint8_t* verified,
                                  unsigned long long* n_verified, unsigned long long* n_invalid, cudaStream_t st);
// Double-key Schnorr signatures over G and G' (p252_schnorr_{sign,verify}_double_batch, p252_note_sign_double_batch),
// challenge c = the truncated digest of the row [R.u, R.v, R'.u, R'.v, m] (4 x u64 < 2^250).  Counters are device pointers
// and may be null.
// pack: rows[i] = [R.u, R.v, R'.u, R'.v, m] (160 bytes, a value >= p written as 0); flag[i] = (and_flag ? flag[i] : 1) and
// all five < p
cudaError_t launch_schnorr_pack_double(const void* R_uv, const void* Rp_uv, const void* msg, size_t n, void* rows,
                                       uint8_t* flag, bool and_flag, cudaStream_t st);
// sign: ok[i] &= sk[sk_bcast ? 0 : i] < r_J; u_out[i] = (r[i] - c[i] sk) mod r_J.  An item with ok = 0 gets zeroed u, R_uv
// and Rp_uv rows and is counted into *n_invalid
cudaError_t launch_schnorr_sign_double(const void* sk, bool sk_bcast, const void* r, const void* c, size_t n, void* u_out,
                                       void* R_uv, void* Rp_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// note sign: as sign with sk = (h[i] + b[b_bcast ? 0 : i]) mod r_J, h[i] the truncated digest of [a] R_note and valid[i]
// its validity from launch_dhke; ok[i] &= valid[i] and b < r_J; pkp_uv[i] = [sk] G' (table_p: the fixed-base table of G'),
// zeroed with the other rows of an invalid item
cudaError_t launch_note_sign_double(const void* b, bool b_bcast, const void* h, const uint8_t* valid, const void* r,
                                    const void* c, size_t n, const void* table_p, void* u_out, void* R_uv, void* Rp_uv,
                                    void* pkp_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// verify: verified[i] = valid[i], u[i] < r_J, pk and pkp[pk_bcast ? 0 : i] curve points with u, v < p, [u[i]] G + [c[i]] pk
// == R_uv[i] and [u[i]] G' + [c[i]] pkp == Rp_uv[i] (table, table_p: the fixed-base tables of G and G'); *n_verified +=
// verified items, *n_invalid += invalid ones
cudaError_t launch_schnorr_verify_double(const void* pk, const void* pkp, bool pk_bcast, const void* u, const void* R_uv,
                                         const void* Rp_uv, const void* c, const uint8_t* valid, size_t n, const void* table,
                                         const void* table_p, uint8_t* verified, unsigned long long* n_verified,
                                         unsigned long long* n_invalid, cudaStream_t st);
// Note values (p252_value_commit_batch, p252_note_create_batch, p252_note_open_batch): C = [v] G + [blinder] G' (table,
// table_p: the fixed-base tables of G and G'), v one u64 per item, blinder canonical 4 x u64, C as (u, v) Montgomery pairs.
// Counters are device pointers and may be null.
// commit: ok[i] = blinder < r_J; commitment[i] = C, zeroed for an invalid item; *n_invalid += invalid items
cudaError_t launch_value_commit(const uint64_t* value, const void* blinder, size_t n, const void* table, const void* table_p,
                                void* commitment, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// create: commitment[i] = C for every item (the caller zeroes invalid ones), rows[i] = [Fr(v), Fr(blinder)] (64 bytes,
// Montgomery), valid[i] &= blinder < r_J
cudaError_t launch_note_value(const uint64_t* value, const void* blinder, size_t n, const void* table, const void* table_p,
                              void* commitment, void* rows, uint8_t* valid, cudaStream_t st);
// open: rows[i] = the decrypted [m0, m1] (Montgomery), ok[i] their authentication, valid[i] the key exchange's validity.
// ok[i] = ok and valid, m0 < 2^64, m1 < r_J, both coordinates of commitment[i] < p and [m0] G + [m1] G' == commitment[i];
// value[i] = m0 and blinder[i] = m1 (canonical) where ok, zeros elsewhere; *n_failed += items with ok = 0
cudaError_t launch_note_open_value(const void* rows, const uint8_t* valid, const void* commitment, size_t n, const void* table,
                                   const void* table_p, uint64_t* value, void* blinder, uint8_t* ok,
                                   unsigned long long* n_failed, cudaStream_t st);
// Multi-key wallet scans (p252_wallet_scan_batch): k keys (a_j, b_j) (canonical 4 x u64), a chunk of n notes, pair p =
// i k + j for note i and key j.  table / table_p: the fixed-base tables of G and G'.  Counters are device pointers; n_bad and
// n_invalid may be null.
// keys: nb[j] = the Niels form of [b_j] G (96 bytes, Montgomery; b = 0 for a bad key), kvalid[j] = a_j, b_j < r_J;
// *n_owned = 0 (the chunk's owned count, for launch_wallet_select); *n_bad += bad keys
cudaError_t launch_wallet_keys(const void* a, const void* b, uint32_t k, const void* table, void* nb, uint8_t* kvalid,
                               unsigned long long* n_owned, unsigned long long* n_bad, cudaStream_t st);
// dhke: shared_uv[p] = [a_j] R_i as (u, v); valid[p] = kvalid[j] and R_i a curve point with u, v < p, (0, 0) otherwise
cudaError_t launch_wallet_dhke(const void* a, const uint8_t* kvalid, uint32_t k, const void* R_uv, size_t n_pairs, void* shared_uv,
                               uint8_t* valid, cudaStream_t st);
// match: matched[p] = valid[p], both note_pk[i] coordinates < p and note_pk[i] == [h[p]] G + B_j (B_j from nb)
cudaError_t launch_wallet_match(const void* h, size_t n_pairs, uint32_t k, const void* table, const void* nb, const void* note_pk,
                                const uint8_t* valid, uint8_t* matched, cudaStream_t st);
// The dense rows of a chunk's owned notes (row r < *n_owned): meta (uint32 note index, uint32 owner), S (64 bytes), h (32),
// b (32), pos (8), nonce (32), cipher (96), C (64), valid (1 byte, set to 1)
struct WalletRows {
    void *meta, *S, *h, *b;
    uint64_t* pos;
    void *nonce, *cipher, *C;
    uint8_t* valid;
};
// select: owner[i] = the smallest j with matched[i k + j] (-1 if none); nullifier, value, blinder and opened rows of note i
// zeroed; *n_invalid += notes with R not a curve point with u, v < p or a note_pk coordinate >= p; owned notes appended
// to `dense` at *n_owned (which counts them)
cudaError_t launch_wallet_select(uint32_t k, const uint8_t* matched, const void* S, const void* h, const void* b,
                                 const void* R_uv, const void* note_pk, const uint64_t* pos, const void* nonce,
                                 const void* cipher, const void* C, size_t n, int32_t* owner, void* nullifier, uint64_t* value,
                                 void* blinder, uint8_t* opened, const WalletRows& dense, unsigned long long* n_owned,
                                 unsigned long long* n_invalid, cudaStream_t st);
// scatter: dense row r's nullifier, value, blinder and ok to note meta[r].x; totals[4 owner + 0..3] += value (128-bit, low
// word first), 1, ok
cudaError_t launch_wallet_scatter(const void* meta, const void* nul, const uint64_t* value_rows, const void* blinder_rows,
                                  const uint8_t* ok, size_t n_own, void* nullifier, uint64_t* value, void* blinder,
                                  uint8_t* opened, unsigned long long* totals, cudaStream_t st);
// JubJub ElGamal (p252_elgamal_{encrypt,decrypt}_batch, p252_note_sender_{encrypt,decrypt}_batch): (c1, c2) =
// ([r] G, M + [r] PK) with table the fixed-base table of G, and M = c2 - [sk] c1.  Points are (u, v) Montgomery pairs,
// scalars canonical 4 x u64.  Every item runs the same schedule; an item with ok = 0 gets zeroed output rows and is
// counted once into the counter (a device pointer, may be null).
// encrypt: c1_uv[i], c2_uv[i] = encrypt(pk[pk_bcast ? 0 : i], msg[msg_bcast ? 0 : i]; r[i]); ok[i] = r < r_J and both
// points curve points with u, v < p
cudaError_t launch_elgamal_encrypt(const void* pk, bool pk_bcast, const void* msg, bool msg_bcast, const void* r, size_t n,
                                   const void* table, void* c1_uv, void* c2_uv, uint8_t* ok, unsigned long long* n_invalid,
                                   cudaStream_t st);
// sender encrypt: enc[i] = [c1_A, c2_A, c1_B, c2_B] (256 bytes), the encryptions of A and B (row sender_bcast ? 0 : i)
// under note_pk[i] with blinder[2 i], blinder[2 i + 1]; ok as for encrypt, over all five operands
cudaError_t launch_note_sender_encrypt(const void* note_pk, const void* A_uv, const void* B_uv, bool sender_bcast,
                                       const void* blinder, size_t n, const void* table, void* enc, uint8_t* ok,
                                       unsigned long long* n_invalid, cudaStream_t st);
// decrypt: msg_uv[i] = c2_uv[i] - [sk[sk_bcast ? 0 : i]] c1_uv[i]; ok[i] = sk < r_J and c1, c2 curve points with u, v < p
cudaError_t launch_elgamal_decrypt(const void* sk, bool sk_bcast, const void* c1_uv, const void* c2_uv, size_t n,
                                   void* msg_uv, uint8_t* ok, unsigned long long* n_invalid, cudaStream_t st);
// sender decrypt, after launch_dhke ([a] R, valid) and the truncated digest (h): note_sk = (h[i] + b) mod r_J with
// b = b[b_bcast ? 0 : i]; A_uv[i], B_uv[i] = c2 - [note_sk] c1 of enc[i]'s two pairs; ok[i] = valid[i], b < r_J, the four
// ciphertext points curve points with u, v < p, and [note_sk] G == note_pk[i]; *n_failed += items with ok = 0
cudaError_t launch_note_sender_decrypt(const void* h, const void* b, bool b_bcast, const uint8_t* valid, const void* note_pk,
                                       const void* enc, size_t n, const void* table, void* A_uv, void* B_uv, uint8_t* ok,
                                       unsigned long long* n_failed, cudaStream_t st);
// Point compression (p252_points_from_bytes / p252_points_to_bytes): 32-byte encodings <-> (u, v) Montgomery pairs (64
// bytes).  from: ok[i] = v < p and u^2 a square, an invalid item gets (0, 0); to: ok[i] = u, v < p and on the curve, an
// invalid item gets 32 bytes of 0xff.  *n_invalid (a device counter, may be null) += invalid items.
cudaError_t launch_points_from_bytes(const void* bytes, size_t n, void* uv, uint8_t* ok, unsigned long long* n_invalid,
                                     cudaStream_t st);
cudaError_t launch_points_to_bytes(const void* uv, size_t n, void* bytes, uint8_t* ok, unsigned long long* n_invalid,
                                   cudaStream_t st);
// Multi-scalar multiplication (p252_jubjub_msm / p252_schnorr_verify_all), VARIABLE TIME (scalars are public), one chunk
// of m rows at a time with c-bit windows: W = msm_windows(c) windows of B = 2^(c-1) buckets (jubjub_device.cuh).  Rows are
// scalars (p252_jscalar, 32 bytes) and points ((u, v) Montgomery, 64 bytes).
// prep: niels[i] (96 bytes) = the Niels form of row i; keys / vals [w m + i] = the bucket key w B + |e| - 1 of digit e of
// window w (the sentinel W B for e = 0 or an invalid row) and i | (e < 0) << 31.  *n_invalid (device, may be null) +=
// invalid rows (s >= r_J, a coordinate >= p, off the curve).
constexpr int kMsmPiece = 32;   // sorted entries per thread of launch_msm_bucket; each pass shrinks a list to 2 / kMsmPiece
cudaError_t launch_msm_prep(const void* scalars, const void* points, uint32_t m, int c, void* niels, uint32_t* keys,
                            uint32_t* vals, unsigned long long* n_invalid, cudaStream_t st);
// buckets[0, nb) = the identity (128-byte extended points)
cudaError_t launch_msm_fill(void* buckets, uint32_t nb, cudaStream_t st);
// One pass over a key-sorted list of N entries (rows: the sorted digits, vals their values, src the Niels rows; otherwise
// the carries of the previous pass, src their points): whole buckets are stored, runs that cross a piece boundary go to
// (okeys, opts), 2 ceil(N / kMsmPiece) slots (null when N <= kMsmPiece).  Keys >= nb are skipped.
cudaError_t launch_msm_bucket(bool rows, const uint32_t* keys, const uint32_t* vals, const void* src, uint32_t N, uint32_t nb,
                              void* buckets, uint32_t* okeys, void* opts, cudaStream_t st);
// wsum[w] (128 bytes) = sum over the buckets of window w of |digit| B_j, w < W
cudaError_t launch_msm_window(const void* buckets, int c, void* wsum, cudaStream_t st);
int msm_window_parts(int c);   // threads per window of launch_msm_window
int msm_windows(int c);        // W (c)
int msm_bits(size_t rows);     // the window width c for chunks of `rows` rows (DESIGN.md section 4)
// Adds the chunks' window sums (wsum, nchunks x W) and combines the windows.  zsum null: out_uv (device, 64 bytes) = the
// sum, affine.  Otherwise (verify_all) nsum (sum z u, sum z c) pairs modulo r_J are added too, and
// *verified = [8] (sum + [sum z u] G + [sum z c] pk) == identity and *bad == 0 (table: G's fixed-base table; pk: one
// public key (u, v), or null for none)
cudaError_t launch_msm_final(const void* wsum, uint32_t nchunks, int c, void* out_uv, const void* zsum, uint32_t nsum,
                             const void* table, const void* pk, const uint32_t* bad, unsigned long long* verified,
                             cudaStream_t st);
// verify_all rows of n items, after launch_schnorr_pack (valid) and the truncated digest (c): item i is valid iff valid[i],
// u, z < r_J and pk[pk_bcast ? 0 : i] a curve point with u, v < p (counted into *n_invalid, device, may be null); an
// invalid item or an R off the curve sets *bad.  Rows (scalars 32 bytes, points 64): pk_bcast: row i = (z, -R); otherwise
// rows 2 i = (z c mod r_J, PK), 2 i + 1 = (z, -R); (0, identity) for an invalid item or an off-curve R.  zsum[blk0 + b]
// (64 bytes) = the sums modulo r_J of z u and (pk_bcast) z c over block b of kMsmItemsPerSum items.
constexpr int kMsmItemsPerSum = 128;
cudaError_t launch_msmv_prep(const void* pk, bool pk_bcast, const void* u, const void* R_uv, const void* c, const void* z,
                             const uint8_t* valid, uint32_t n, void* row_scalars, void* row_points, void* zsum, uint32_t blk0,
                             uint32_t* bad, unsigned long long* n_invalid, cudaStream_t st);
// verify_double_all rows of n items, after launch_schnorr_pack_double (valid) and the truncated digest (c): item i is valid
// iff valid[i], u, z, zp < r_J and pk, pkp[pk_bcast ? 0 : i] curve points with u, v < p (counted into *n_invalid, device,
// may be null); an invalid item or an R or R' off the curve sets *bad.  Rows: pk_bcast: 2 i = (z, -R), 2 i + 1 =
// (zp, -R'); otherwise 4 i = (z c, PK), 4 i + 1 = (zp c, PK'), 4 i + 2 = (z, -R), 4 i + 3 = (zp, -R'); (0, identity) for
// an invalid item or an off-curve R or R'.  zsum[blk0 + b] (128 bytes) = the sums modulo r_J of z u, zp u and
// (pk_bcast) z c, zp c over block b of kMsmItemsPerSum items.
cudaError_t launch_msmv_prep_double(const void* pk, const void* pkp, bool pk_bcast, const void* u, const void* R_uv,
                                    const void* Rp_uv, const void* c, const void* z, const void* zp, const uint8_t* valid,
                                    uint32_t n, void* row_scalars, void* row_points, void* zsum, uint32_t blk0, uint32_t* bad,
                                    unsigned long long* n_invalid, cudaStream_t st);
// Adds the chunks' window sums (wsum, nchunks x W) and the nsum 4-tuples of zsum modulo r_J, and writes
// *verified = [8] (sum + [sum z u] G + [sum zp u] G' + [sum z c] PK + [sum zp c] PK') == identity and *bad == 0
// (table, table_p: the fixed-base tables of G and G'; pk: one key pair PK, PK' (128 bytes), or null for none)
cudaError_t launch_msmv_final_double(const void* wsum, uint32_t nchunks, int c, const void* zsum, uint32_t nsum,
                                     const void* table, const void* table_p, const void* pk, const uint32_t* bad,
                                     unsigned long long* verified, cudaStream_t st);
// BlsScalar::hash_to_scalar (p252_hash_to_scalar_batch): item i = bytes[offsets[i] - base .. offsets[i+1] - base), valid
// iff offsets[i] - base <= offsets[i+1] - base <= n_bytes and its length is <= max_len; no byte outside
// bytes[0, n_bytes) is read, whatever the offsets.  out[i] = BLAKE2b-512 of the item reduced by from_bytes_wide
// (Montgomery), a zero row for an invalid item (counted into *rejected, device, may be null).  One thread per item;
// perm (may be null): the item order of launch_hash_to_scalar_keys and the ascending sort, hashed longest first.
cudaError_t launch_hash_to_scalar(const void* bytes, uint64_t base, uint64_t n_bytes, const uint64_t* offsets,
                                  const uint32_t* perm, uint32_t n, uint32_t max_len, void* out, unsigned long long* rejected,
                                  cudaStream_t st);
// keys[i] = the block count max(1, ceil(len / 128)) of a valid item, 0 for an invalid one (counted into *rejected);
// vals[i] = i
cudaError_t launch_hash_to_scalar_keys(const uint64_t* offsets, uint32_t n, uint64_t base, uint64_t n_bytes, uint32_t max_len,
                                       uint32_t* keys, uint32_t* vals, unsigned long long* rejected, cudaStream_t st);
// BlsScalar::from_bytes_wide (p252_scalars_from_bytes_wide): n rows of 64 bytes -> n scalars (Montgomery)
cudaError_t launch_from_bytes_wide(const void* in, size_t n, void* out, cudaStream_t st);
// Mixed digest batches (p252_hash_batch_mixed): item i = Hash::new(mode[i] & 3), in[offsets[i] - base .. offsets[i+1] -
// base) of n_scalars, finalize() or (mode[i] & 0x80) finalize_truncated() into the rows [out_offsets[i] - obase,
// out_offsets[i+1] - obase) of out (n_out rows).  keys: the step count ceil(len / 4) + ceil(out_len / 4) of a valid item
// (the rules of p252_hash_tag plus len <= max_len, out_len <= max_out_len and no mode bit outside 0x83), 0 for an invalid
// one (counted into *rejected; zero rows where its output range is valid); vals[i] = i; tags (n rows) and desc (n) the
// item's tag, derived on the device, and (len, out_len | truncated << 31), (0, 0) for an invalid item
cudaError_t launch_mixed_keys(const uint8_t* mode, const uint64_t* offsets, uint64_t base, uint64_t n_scalars,
                              const uint64_t* out_offsets, uint64_t obase, uint64_t n_out, uint32_t n, uint32_t max_len,
                              uint32_t max_out_len, void* out, uint32_t* keys, uint32_t* vals, void* tags, uint2* desc,
                              unsigned long long* rejected, cudaStream_t st);
// over the keys sorted ascending with their values (perm): the digests of the valid items; lane-split kernel when
// n <= coop_max
cudaError_t launch_digest_mixed(const void* tags, const uint2* desc, const void* in, uint64_t base, const uint64_t* offsets,
                                uint64_t obase, const uint64_t* out_offsets, const uint32_t* perm, uint32_t n, void* out,
                                size_t coop_max, cudaStream_t st);
void kernel_launch_shape(int* threads_per_block, int* min_blocks_per_sm);
size_t coop_max_items(int sm_count);   // default small-batch threshold (P252_COOP_MAX or derived from the SM count)
// 32x32->64-bit multiply instructions (IMAD.WIDE / IMAD.HI class) and DFMA per Hades permutation, counted from
// the generated PTX (fr_ptx.cuh) and the round structure of hades_permute()
uint32_t wide_mul_per_permutation();
uint32_t dfma_per_permutation();

}  // namespace p252
