/* poseidon252_b200 -- C ABI of the H100-native batched Poseidon/Hades engine.
 *
 * Drop-in boundary for the hot path of dusk-poseidon (reference = dusk-network/Poseidon252, a pure-Rust,
 * one-state-at-a-time CPU crate with no FFI of its own).  The reference's seam for this path is
 * the trait pair dusk_safe::Safe<BlsScalar,5> (impl: src/hades/permutation/scalar.rs:24-36) +
 * Hades<BlsScalar> (src/hades/permutation.rs:34-124) under the public surface src/lib.rs:13-31.
 * This header is what a Rust `extern "C"` block for the batch entry points
 * (hades::permute_batch, Hash::digest_batch, encrypt_batch, decrypt_batch, merkle4) binds; the
 * binding itself is in bindings/rust/ and INTEGRATION.md.
 *
 * Conventions
 *   - p252_fr is bit-identical to `BlsScalar.0`: 4 x u64 little-endian limbs of x*R mod p
 *     (Montgomery form, R = 2^256 mod p, value < p).  No conversion happens at the boundary.
 *   - All batch buffers are item-major arrays (the layout of `&[BlsScalar]`, src/hash.rs:94).
 *   - The caller owns every buffer; the library owns only the context (reference borrows inputs,
 *     src/hash.rs:94, and returns fresh Vecs, src/hash.rs:128).
 *   - `flags` says where the buffers live: P252_MEM_HOST (library stages H2D/D2H itself) or
 *     P252_MEM_DEVICE (pointers are device pointers of ctx's GPU, 16-byte aligned; add
 *     P252_ASYNC to return right after enqueueing on the context's stream).
 *   - Every function returns a p252_status; nothing unwinds across the boundary.  Positive codes
 *     mirror dusk_poseidon::Error (src/error.rs:11-32); negative codes are engine failures.
 *   - There is NO CPU fallback: without a usable sm_90 (H100) device p252_create fails.
 *   - A context is bound to one device and one stream; calls on one context serialise (a mutex
 *     inside the context: concurrent callers block, they do not race); separate contexts are
 *     independent (the reference is stateless: ScalarPermutation is a ZST,
 *     src/hades/permutation/scalar.rs:15).
 *   - HOST calls are synchronous; on ANY exit path (success or failure) the staging streams are
 *     joined, and for encrypt/decrypt the staging arenas (secrets, nonces, plaintext) are zeroed.
 */
#ifndef POSEIDON252_B200_H
#define POSEIDON252_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define P252_WIDTH 5 /* dusk_poseidon::HADES_WIDTH, src/hades.rs:34 */

typedef struct p252_fr {
    uint64_t l[4];
} p252_fr;

typedef struct p252_ctx p252_ctx;

typedef enum p252_status {
    P252_OK = 0,
    /* dusk_poseidon::Error, src/error.rs:11-32 */
    P252_ERR_IO_PATTERN_VIOLATION = 1,
    P252_ERR_INVALID_IO_PATTERN = 2,
    P252_ERR_TOO_FEW_INPUT_ELEMENTS = 3,
    P252_ERR_ENCRYPTION_FAILED = 4,
    P252_ERR_DECRYPTION_FAILED = 5,
    P252_ERR_INVALID_POINT = 6,
    /* engine */
    P252_ERR_INVALID_ARGUMENT = -1,
    P252_ERR_CUDA = -2,
    P252_ERR_NCCL = -3,
    P252_ERR_NO_DEVICE = -4,
    P252_ERR_OUT_OF_MEMORY = -5
} p252_status;

/* u64::from(Domain), src/hash.rs:38-56 */
typedef enum p252_domain {
    P252_DOMAIN_MERKLE4 = 0,
    P252_DOMAIN_MERKLE2 = 1,
    P252_DOMAIN_ENCRYPTION = 2,
    P252_DOMAIN_OTHER = 3
} p252_domain;

enum {
    P252_MEM_HOST = 0,
    P252_MEM_DEVICE = 1,
    P252_ASYNC = 2,
    /* p252_merkle4_build_dist only (measurement aids, see p252_tree_level_timings): */
    P252_TIMING = 4,     /* bracket every level's kernel and all-gather with CUDA events */
    P252_NO_GATHER = 8   /* skip the collectives: compute-only timing run, node values above level 0 are NOT valid */
};

/* ---- library / context ------------------------------------------------------------------- */
const char* p252_version(void);
const char* p252_strerror(int status);
int p252_device_count(int* count);

/* Create a context on CUDA device `device` with its own stream.  Fails with P252_ERR_NO_DEVICE
 * when there is no sm_90 (H100) GPU (no CPU fallback). */
int p252_create(int device, p252_ctx** out);
/* Same, but enqueue all work on an existing CUDA stream (cudaStream_t passed as void*), e.g. the
 * caller's torch stream, so that the caller's CUDA events bracket the kernels. */
int p252_create_on_stream(int device, void* cuda_stream, p252_ctx** out);
void p252_destroy(p252_ctx* ctx);
int p252_sync(p252_ctx* ctx);
/* Text of the last CUDA/NCCL failure on this context ("" if none). */
const char* p252_last_error(const p252_ctx* ctx);
/* Number of kernels this context has launched since creation. */
uint64_t p252_launch_count(const p252_ctx* ctx);
/* Pinned host memory for P252_MEM_HOST callers that want full PCIe bandwidth. */
int p252_host_alloc(size_t bytes, void** out);
int p252_host_free(void* p);

/* Static facts about the kernels of this build (what one Hades permutation costs in this formulation; used by
 * benchmarks to state the integer-multiplier roofline next to the HBM one).  Set struct_size before the call. */
typedef struct p252_kernel_info {
    uint32_t struct_size;
    uint32_t wide_mul_per_permutation; /* 32x32->64 multiply instructions (IMAD.WIDE / IMAD.HI) per permutation */
    uint32_t dfma_per_permutation;     /* FP64 FMAs of the small-integer MDS layer per permutation              */
    uint32_t montmul_per_permutation;  /* Montgomery products incl. squarings (365; the reference does 2000)    */
    uint32_t threads_per_block;
    uint32_t min_blocks_per_sm;
} p252_kernel_info;
int p252_get_kernel_info(p252_kernel_info* out);

/* Digest and raw-permutation batches of at most `max_items` items run the lane-split kernels (five threads per sponge state: lower latency,
 * ~3x lower throughput per state) -- the regime of single digests and of the top levels of a Merkle tree.  Default:
 * one lane-split warp (6 items) per SM sub-partition, 3168 on a 132-SM H100 (environment variable P252_COOP_MAX
 * overrides it at context creation); 0 disables the lane-split path.  Both
 * kernels produce bit-identical results. */
int p252_set_small_batch_max(p252_ctx* ctx, size_t max_items);

/* Fault injection / inspection for tests (no effect unless called).  p252_debug_fail_chunk: the k-th staged chunk
 * (0-based) of the NEXT host-buffer call on this context fails as if its kernel launch had failed (one shot).
 * p252_debug_staging_nonzero: number of non-zero bytes currently held by the context's staging arenas. */
int p252_debug_fail_chunk(p252_ctx* ctx, long long k);
int p252_debug_staging_nonzero(p252_ctx* ctx, size_t* nonzero_bytes);

/* ---- host-side sponge bookkeeping (no GPU needed) ----------------------------------------- */
/* u64::from(Domain), src/hash.rs:43-55 */
int p252_domain_separator(int domain, uint64_t* out);
/* dusk-safe tag input: `calls` are the io-pattern, absorb(len) = 0x80000000|len, squeeze(len) = len
 * (as produced by io_pattern, src/hash.rs:62-85); consecutive calls of one kind aggregate.
 * Writes the byte string hashed into the tag; *out_len in = capacity, out = length. */
int p252_tag_input(const uint32_t* calls, size_t ncalls, uint64_t domain_sep, uint8_t* out, size_t* out_len);
/* BlsScalar::hash_to_scalar (src/hades/permutation/scalar.rs:29-31): BLAKE2b-512 -> mod p. */
int p252_hash_to_scalar(const uint8_t* bytes, size_t len, p252_fr* out);
/* Safe::tag of the pattern: hash_to_scalar(tag_input(calls, domain_sep)). */
int p252_tag(const uint32_t* calls, size_t ncalls, uint64_t domain_sep, p252_fr* tag);
/* io_pattern(domain, [in_len], out_len) + tag (src/hash.rs:62-85,131-137): checks the Merkle
 * arities (-> P252_ERR_IO_PATTERN_VIOLATION) and zero lengths (-> P252_ERR_INVALID_IO_PATTERN). */
int p252_hash_tag(int domain, size_t in_len, size_t out_len, p252_fr* tag);
/* tag of dusk_safe::encrypt/decrypt for message length L (src/encryption.rs:67-73). */
int p252_encryption_tag(size_t L, p252_fr* tag);

/* ---- batch entry points (the GPU path) ----------------------------------------------------- */
/* hades::permute_batch: n independent Safe::permute calls (src/hades/permutation/scalar.rs:25-27
 * -> Hades::perm, src/hades/permutation.rs:105-123).  states: n x 5, in place. */
int p252_permute_batch(p252_ctx* ctx, p252_fr* states, size_t n, int flags);
/* The reference's dense formulation executed on the device (cross-check / cost comparison). */
int p252_permute_batch_dense(p252_ctx* ctx, p252_fr* states, size_t n, int flags);

/* Sponge with a caller-supplied tag: start(tag) -> absorb(in_len) -> squeeze(out_len)
 * (Hash::finalize, src/hash.rs:128-155).  in: n x in_len, out: n x out_len. */
int p252_digest_batch(p252_ctx* ctx, const p252_fr* tag, const p252_fr* in, size_t n, size_t in_len,
                      p252_fr* out, size_t out_len, int flags);
/* Hash::digest_batch: n x Hash::digest(domain, in[i]) with Hash::output_len(out_len)
 * (src/hash.rs:111-115,191-195); tag computed on the host once per batch. */
int p252_hash_batch(p252_ctx* ctx, int domain, const p252_fr* in, size_t n, size_t in_len, p252_fr* out,
                    size_t out_len, int flags);

/* Hash::digest_truncated batch (src/hash.rs:164-183,203-210): every output scalar is taken out of Montgomery
 * form and masked to 250 bits; out_raw receives the raw limbs the reference passes to JubJubScalar::from_raw. */
int p252_hash_batch_truncated(p252_ctx* ctx, int domain, const p252_fr* in, size_t n, size_t in_len, p252_fr* out_raw,
                              size_t out_len, int flags);

/* Variable-length digest batch: out[i] = Hash::digest(domain, in[offsets[i] .. offsets[i+1])) with
 * Hash::output_len(out_len) (src/hash.rs:111-115,191-195) for i < n, one call for inputs of any mix of lengths.
 *   in: n_scalars scalars; offsets: n + 1 entries in the same memory space as in / out (offsets[0] need not be 0, so a
 *   slice of a larger CSR array works); out: n x out_len, item-major, in input order; n < 2^31.
 *   Batch checks, before anything runs: out_len == 0 -> INVALID_IO_PATTERN; a Merkle domain with out_len != 1 ->
 *   IO_PATTERN_VIOLATION; max_len == 0 or > P252_VARLEN_MAX_LEN -> INVALID_ARGUMENT; DEVICE in / out not 16-byte or
 *   offsets not 8-byte aligned -> INVALID_ARGUMENT.
 *   Item i is valid iff offsets[i] <= offsets[i+1] <= n_scalars, 1 <= len_i <= max_len (len_i = offsets[i+1] -
 *   offsets[i]) and p252_hash_tag(domain, len_i, out_len) accepts it (Merkle domains: len_i == arity).
 *   HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written:
 *   INVALID_ARGUMENT for a range outside [0, n_scalars] or decreasing offsets, IO_PATTERN_VIOLATION for a Merkle length
 *   other than the arity, INVALID_IO_PATTERN for length 0, INVALID_ARGUMENT for length > max_len.
 *   DEVICE: offsets are not inspected on the host; an invalid item is skipped on the device, its out_len output
 *   scalars are written as zero and it is counted into *n_rejected (optional HOST pointer, 0 for HOST calls; lifetime as
 *   for p252_mtree_update).  No offset value makes a kernel read outside in[0, n_scalars) or write outside out.
 *   With P252_ASYNC nothing is synchronised.
 * The tags of lengths 1..max_len for (domain, out_len) are derived on the host and kept on the device in the context;
 * the table is rebuilt only when max_len grows or (domain, out_len) changes, so a steady max_len costs nothing.  Items
 * are sorted by length on the device so that a warp hashes items of (nearly) equal length together. */
#define P252_VARLEN_MAX_LEN 65536
int p252_hash_batch_varlen(p252_ctx* ctx, int domain, const p252_fr* in, size_t n_scalars, const uint64_t* offsets, size_t n,
                           size_t max_len, p252_fr* out, size_t out_len, size_t* n_rejected, int flags);

/* Mixed digest batch: every Hash the reference can build, one call for items of different domains, input and output
 * lengths, finalized or truncated.  Item i is Hash::new(mode[i] & 3), update(in[offsets[i] .. offsets[i+1])),
 * output_len(out_len_i), then finalize() -- or, with mode[i] & P252_MIXED_TRUNCATED, finalize_truncated(), whose
 * rows are the raw limbs masked to 250 bits as in p252_hash_batch_truncated (src/hash.rs:128-183).  The chunk layout
 * of update() never changes a digest (consecutive absorbs aggregate into one tag word), so the concatenated input
 * describes the item.
 *   mode: n bytes, mode[i] & 3 the item's p252_domain; in: n_scalars scalars; offsets, out_offsets: n + 1 entries each;
 *   out: n_out rows, item i writes the rows out[out_offsets[i] .. out_offsets[i+1]), so out_len_i = out_offsets[i+1] -
 *   out_offsets[i].  mode, offsets and out_offsets live in the same memory space as in / out; offsets[0] and
 *   out_offsets[0] need not be 0.
 *   Batch checks, before anything runs, all INVALID_ARGUMENT: a NULL buffer the call needs, n >= 2^31, max_len or
 *   max_out_len == 0 or > P252_VARLEN_MAX_LEN, DEVICE in / out not 16-byte or offsets / out_offsets not 8-byte aligned.
 *   Item checks, in this order: a mode bit outside 0x83 -> INVALID_ARGUMENT; an input range that decreases or lies
 *   outside [0, n_scalars] -> INVALID_ARGUMENT; an output range that decreases or lies outside [0, n_out] ->
 *   INVALID_ARGUMENT; a Merkle domain with len_i != arity or out_len_i != 1 -> IO_PATTERN_VIOLATION; len_i == 0 or
 *   out_len_i == 0 -> INVALID_IO_PATTERN; len_i > max_len or out_len_i > max_out_len -> INVALID_ARGUMENT.  Apart from
 *   the mode bits these are the rules of p252_hash_tag; a non-Merkle domain with out_len_i > 1 is accepted (the
 *   reference's output_len() rule is applied by the front ends).
 *   HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written.
 *   DEVICE: descriptors are not inspected on the host; an invalid item is counted into *n_rejected (optional HOST
 *   pointer, 0 for HOST calls; lifetime as for p252_mtree_update) and gets zero rows where its output range is valid,
 *   nothing otherwise.  No descriptor value makes a kernel read outside in or write outside out; where the valid
 *   output ranges of a non-monotone out_offsets overlap, the rows are unspecified.  With P252_ASYNC nothing is
 *   synchronised.  n == 0 runs nothing.
 * Each item's tag (hash_to_scalar of its 16-byte tag input, one BLAKE2b block) is derived on the device; items are
 * sorted on the device by step count ceil(len / 4) + ceil(out_len / 4), so that a warp hashes items of (nearly) equal
 * work. */
#define P252_MIXED_TRUNCATED 0x80
int p252_hash_batch_mixed(p252_ctx* ctx, const uint8_t* mode, const p252_fr* in, size_t n_scalars,
                          const uint64_t* offsets, size_t n, size_t max_len, p252_fr* out, size_t n_out,
                          const uint64_t* out_offsets, size_t max_out_len, size_t* n_rejected, int flags);

/* Wire format (BlsScalar::from_bytes / to_bytes as used at src/hades.rs:94-105,131): n canonical 32-byte
 * little-endian integers <-> BlsScalar.0.  from_bytes: ok[i] = 0 and out[i] = 0 when the value is >= p (the
 * reference returns None); ok may be NULL. */
int p252_scalars_from_bytes(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out, uint8_t* ok, int flags);
int p252_scalars_to_bytes(p252_ctx* ctx, const p252_fr* in, size_t n, uint8_t* bytes, int flags);
/* BlsScalar::from_bytes_wide on n rows of 64 bytes: out[i] = (lo + hi * 2^256) mod p in Montgomery form, lo / hi the
 * row's first / last 32 bytes as little-endian integers.  Every input is valid.  DEVICE bytes and out must be 16-byte
 * aligned. */
int p252_scalars_from_bytes_wide(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out, int flags);

/* Batched BlsScalar::hash_to_scalar (src/hades/permutation/scalar.rs:29-31; p252_hash_to_scalar is one call of it):
 * out[i] = from_bytes_wide(BLAKE2b-512(bytes[offsets[i] .. offsets[i+1]))) in Montgomery form (BlsScalar.0), for i < n,
 * one call for byte strings of any mix of lengths.  The rows can go straight in as the msg of the Schnorr calls.
 *   bytes: n_bytes bytes, any alignment; offsets: n + 1 absolute byte offsets in the same memory space as bytes / out
 *   (offsets[0] need not be 0, so a slice of a larger CSR array works); out: n rows, in input order.
 *   Batch checks, before anything runs: n >= 2^31, max_len > P252_HASH_TO_SCALAR_MAX_LEN, a NULL buffer (bytes with
 *   n_bytes > 0, offsets or out with n > 0), DEVICE offsets not 8-byte or out not 16-byte aligned -> INVALID_ARGUMENT.
 *   Item i is valid iff offsets[i] <= offsets[i+1] <= n_bytes and its length is <= max_len.  Length 0 is valid (the
 *   hash of the empty string), so max_len == 0 is allowed.
 *   HOST: the whole batch is checked first; the lowest-index invalid item decides the status (INVALID_ARGUMENT) and
 *   nothing is written.  The batch is staged in chunks of about 24 MiB of message bytes.
 *   DEVICE: offsets are not inspected on the host; an invalid item gets a zero row and is counted into *n_rejected
 *   (optional HOST pointer, 0 for HOST calls; lifetime as for p252_mtree_update).  No offset value makes a kernel read
 *   a byte outside bytes[0, n_bytes) or write outside out.  With P252_ASYNC nothing is synchronised.
 * n == 0 runs nothing.  The messages are public data, like the inputs of p252_hash_batch: they are staged in ordinary
 * (not wiped) buffers.  One thread hashes one message: BLAKE2b is a serial chain of 128-byte blocks, so a very long item
 * takes one thread ceil(len / 128) compressions while the rest of the batch has finished.  With max_len > 128 the items
 * are sorted by block count on the device first, so that a warp hashes messages of nearly equal length together. */
#define P252_HASH_TO_SCALAR_MAX_LEN (1u << 20) /* bytes per item */
int p252_hash_to_scalar_batch(p252_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const uint64_t* offsets, size_t n,
                              size_t max_len, p252_fr* out, size_t* n_rejected, int flags);

/* encrypt_batch: n x encrypt(msg[i], (u,v)[i], nonce[i]) (src/encryption.rs:62-74).
 * msg: n x L, secret_uv: n x 2 (JubJubAffine::get_u/get_v), nonce: n, cipher: n x (L+1). */
int p252_encrypt_batch(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_fr* secret_uv,
                       const p252_fr* nonce, p252_fr* cipher, int flags);
/* decrypt_batch (src/encryption.rs:83-95).  cipher: n x (L+1), msg: n x L, ok: n bytes; ok[i] = 0
 * <=> the reference returns Error::DecryptionFailed for item i (its msg is zeroed; device callers must look at
 * ok[i] before trusting msg[i]).  Returns P252_OK even when some items fail; *n_failed (optional, a HOST pointer
 * for both memory spaces) receives their count -- for device buffers it is counted on the device and, with
 * P252_ASYNC, written by an asynchronous copy that is complete after p252_sync; until then the size_t must stay
 * valid. */
int p252_decrypt_batch(p252_ctx* ctx, const p252_fr* cipher, size_t n, size_t L, const p252_fr* secret_uv,
                       const p252_fr* nonce, p252_fr* msg, uint8_t* ok, size_t* n_failed, int flags);

/* Variable-length encrypt / decrypt batches: one call for messages (ciphers) of any mix of lengths.
 *   encrypt: cipher item i = encrypt(msg[offsets[i] .. offsets[i+1]), secret_uv[i], nonce[i]) (src/encryption.rs:62-74);
 *   decrypt: message item i = decrypt(cipher[offsets[i] .. offsets[i+1]), secret_uv[i], nonce[i]) (src/encryption.rs:83-95).
 *   Input: n_scalars scalars; offsets: n + 1 absolute indices into it (offsets[0] need not be 0, so a slice of a larger
 *   CSR array works); secret_uv: n x 2 (JubJubAffine::get_u/get_v), nonce: n; n < 2^31; all buffers, offsets included,
 *   in one memory space.  max_len bounds the message length L: 1 <= L <= max_len <= P252_VARLEN_MAX_LEN; a cipher has
 *   L + 1 scalars.
 *   Output: the input CSR with every item one scalar longer (encrypt) or shorter (decrypt), packed from 0.  With
 *   a0 = offsets[0] and an = offsets[n], encrypt writes cipher item i to cipher[offsets[i] - a0 + i, offsets[i+1] - a0 +
 *   i + 1) of an - a0 + n scalars; decrypt writes message item i to msg[offsets[i] - a0 - i, offsets[i+1] - a0 - i - 1)
 *   of an - a0 - n scalars, and ok[i] (n bytes) as p252_decrypt_batch does: ok[i] = 0 <=> the reference returns
 *   Error::DecryptionFailed, and that item's message is zeroed.  A decrypt output fed straight back into encrypt (and the
 *   reverse) needs no second offsets array: its offsets are offsets[i] - a0 -+ i.
 *   Batch checks, before anything runs: max_len == 0 or > P252_VARLEN_MAX_LEN, n >= 2^31, a NULL buffer with n > 0,
 *   DEVICE data buffers not 16-byte or offsets not 8-byte aligned -> INVALID_ARGUMENT.
 *   Item i (a = offsets[i], b = offsets[i+1]) is valid iff a0 <= a <= b <= an <= n_scalars and, for encrypt,
 *   1 <= b - a <= max_len; for decrypt 2 <= b - a <= max_len + 1, a - a0 >= i and an - b >= n - 1 - i (its output range
 *   lies inside msg; both hold by themselves when every item is valid).
 *   HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written:
 *   INVALID_ARGUMENT for a range outside the bounds or decreasing offsets, INVALID_IO_PATTERN for a message length of 0
 *   or a cipher length below 2 (as p252_encryption_tag(0)), INVALID_ARGUMENT for a length above max_len (+1 for
 *   decrypt).  The batch is then staged in chunks of about 24 MiB of input on the staging streams; secrets, nonces and
 *   plaintext live only in the staging arenas, which are zeroed on every exit path.  *n_failed counts the ok[i] == 0.
 *   DEVICE: offsets are not inspected on the host; an invalid item is skipped on the device and counted into
 *   *n_rejected; nothing is written for it (its output position is not trustworthy), except ok[i] = 0 for decrypt.  No
 *   offset value makes a kernel read outside in[0, n_scalars) or write outside the output range above.  *n_failed
 *   counts authentication failures among valid items only.  With P252_ASYNC nothing is synchronised.
 *   n_failed / n_rejected: optional HOST pointers for both memory spaces (*n_rejected is 0 for HOST calls), counted on
 *   the device for DEVICE calls; lifetime as for p252_mtree_update.
 * The tags of L = 1..max_len are derived on the host and kept on the device in the context (a table of their own, next
 * to the one of p252_hash_batch_varlen); it is rebuilt only when max_len grows.  Items are sorted by length on the
 * device so that a warp runs messages of (nearly) equal length together; batches of at most p252_set_small_batch_max
 * items run the lane-split kernel. */
int p252_encrypt_batch_varlen(p252_ctx* ctx, const p252_fr* msg, size_t n_scalars, const uint64_t* offsets, size_t n,
                              size_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* cipher,
                              size_t* n_rejected, int flags);
int p252_decrypt_batch_varlen(p252_ctx* ctx, const p252_fr* cipher, size_t n_scalars, const uint64_t* offsets, size_t n,
                              size_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* msg, uint8_t* ok,
                              size_t* n_failed, size_t* n_rejected, int flags);

/* ---- JubJub key exchange ------------------------------------------------------------------------
 * dhke(secret, public) = [secret] public as JubJubAffine (u, v): the shared secret that encrypt / decrypt take
 * (src/encryption.rs:11-43, "Poseidon + JubJub DHKE + SAFE").  JubJub: -u^2 + v^2 = 1 + d u^2 v^2 over the same field
 * as p252_fr, d = -10240/10241; prime subgroup order r_J (252 bits), cofactor 8.
 *
 * A secret scalar is p252_jscalar: the CANONICAL integer s < r_J as 4 x u64 little-endian limbs, i.e. the 32 bytes of
 * JubJubScalar::to_bytes().  Unlike p252_fr it is NOT a Montgomery image (the limbs of dusk-jubjub's Fr are not public
 * API, to_bytes is).  Points are (u, v) as two p252_fr (JubJubAffine::get_u / get_v, i.e. BlsScalar.0): the layout of
 * secret_uv of p252_{en,de}crypt_batch[_varlen], so a p252_dhke_batch output feeds those calls unchanged.
 *
 * Shapes: item i uses secret[n_secret == 1 ? 0 : i] and public_uv[n_public == 1 ? 0 : i] (n_public points of 2
 * scalars); n_secret and n_public are each 1 or n.  (1, n) is a receiver's scan (one view key, the notes' keys), (n, 1) a
 * sender's R_i = [r_i] G or [r_i] pk.
 * Item validity: s < r_J, u, v < p and (u, v) on the curve.  There is no subgroup check (the reference does none): a
 * torsion component passes through.  Validity is a per-item data condition checked on the device for both memory spaces;
 * the call returns P252_OK and marks an invalid item with ok[i] = 0 and
 *   p252_dhke_batch:           output (0, 0), which is not a curve point (the identity is (0, 1));
 *   p252_encrypt_batch_dhke:   a zeroed cipher row;
 *   p252_decrypt_batch_dhke:   a zeroed message, counted into *n_failed together with the authentication failures (an
 *                              item counts once).
 * n_invalid / n_failed: optional HOST pointers for both memory spaces (lifetime as for p252_decrypt_batch).
 * P252_ERR_INVALID_POINT is returned by the single-item front ends (Python dhke(), p252::dhke), not by these calls.
 * Batch checks, before anything runs: n_secret or n_public not 1 or n, a NULL buffer with n > 0, DEVICE buffers other
 * than ok not 16-byte aligned -> INVALID_ARGUMENT; L == 0 -> INVALID_IO_PATTERN (as p252_encryption_tag).
 * The fused calls run the key exchange and then the kernels of p252_encrypt_batch / p252_decrypt_batch (same shapes:
 * msg n x L, cipher n x (L + 1), nonce n).  Their intermediate shared secrets never leave the context's staging arenas,
 * for DEVICE buffers too, and the arenas are zeroed on every exit path; so these calls are synchronous for both memory
 * spaces (P252_ASYNC only defers the publication of the count to p252_sync).  HOST calls stage secrets, points, nonces and
 * plaintext through the same zeroed arenas; a broadcast operand is staged once per chunk.
 * Each item is one scalar multiplication in constant time (no branch and no address depends on secret bits); see
 * DESIGN.md section 4. */
typedef struct p252_jscalar {
    uint64_t l[4];
} p252_jscalar;
int p252_dhke_batch(p252_ctx* ctx, const p252_jscalar* secret, size_t n_secret, const p252_fr* public_uv, size_t n_public,
                    size_t n, p252_fr* shared_uv, uint8_t* ok, size_t* n_invalid, int flags);
int p252_encrypt_batch_dhke(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_jscalar* secret, size_t n_secret,
                            const p252_fr* public_uv, size_t n_public, const p252_fr* nonce, p252_fr* cipher, uint8_t* ok,
                            size_t* n_invalid, int flags);
int p252_decrypt_batch_dhke(p252_ctx* ctx, const p252_fr* cipher, size_t n, size_t L, const p252_jscalar* secret,
                            size_t n_secret, const p252_fr* public_uv, size_t n_public, const p252_fr* nonce, p252_fr* msg,
                            uint8_t* ok, size_t* n_failed, int flags);

/* ---- Fixed-base JubJub scalar multiplication and the sender's encrypt batch ----------------------------------------
 * [secret] base for ONE base shared by the batch: a public key GENERATOR_EXTENDED * secret, or a note's ephemeral key
 * R = GENERATOR_EXTENDED * r (src/encryption.rs:22-42).  There is no built-in generator: the caller passes the base, e.g.
 * dusk_jubjub::GENERATOR's (u, v).  base_uv is a HOST pointer to (u, v) (two p252_fr) for every memory space; any point on
 * the curve is a valid base, small-order points included.  A base with a coordinate >= p or off the curve is refused
 * with P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.  The context keeps the table
 * of its last base (48 KB of device memory, built on the device on the first call with that base, then reused).
 * Secrets and points are laid out as for p252_dhke_batch.  Item validity: secret / r < r_J and, in the fused call,
 * public_uv a curve point with u, v < p.  An invalid item gets ok[i] = 0, a zeroed output (and, in the fused call, a
 * zeroed cipher row and R row) and is counted once into *n_invalid (optional HOST pointer, lifetime as for
 * p252_decrypt_batch); the call returns P252_OK.
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_public not 1 or n, DEVICE buffers other than ok not
 * 16-byte aligned -> INVALID_ARGUMENT; L == 0 -> INVALID_IO_PATTERN.
 * p252_encrypt_batch_ephemeral derives the shared secret dhke(r[i], public_uv[...]) on the device, with the kernels of
 * p252_encrypt_batch_dhke, and never returns it: like that call it is synchronous for both memory spaces.  HOST calls
 * stage secrets, points, nonces and plaintext through the context's zeroed staging arenas.  Each item is constant time
 * (no branch and no address depends on secret bits); see DESIGN.md section 4. */
/* out_uv[i] = [secret[i]] base (JubJubAffine), n items; base_uv is a HOST pointer to (u, v). */
int p252_fixed_base_batch(p252_ctx* ctx, const p252_fr* base_uv, const p252_jscalar* secret, size_t n, p252_fr* out_uv,
                          uint8_t* ok, size_t* n_invalid, int flags);
/* The reference's sender (src/encryption.rs:22-42) as a batch: R_uv[i] = [r[i]] base,
 * cipher[i] = encrypt(msg[i], dhke(r[i], public_uv[n_public == 1 ? 0 : i]), nonce[i]); msg n x L, cipher n x (L + 1). */
int p252_encrypt_batch_ephemeral(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_jscalar* r,
                                 const p252_fr* base_uv, const p252_fr* public_uv, size_t n_public, const p252_fr* nonce,
                                 p252_fr* cipher, p252_fr* R_uv, uint8_t* ok, size_t* n_invalid, int flags);

/* ---- Stealth addresses: the sender's (R, note_pk) and the receiver's ownership scan (Phoenix notes) ----------------
 *   hash(P)                       = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]   (P affine, < 2^250 < r_J)
 *   sender   (r; A, B):             R = [r] G,  note_pk = [hash([r] A)] G + B
 *   receiver (a, B; R, note_pk):    owns  <=>  note_pk == [hash([a] R)] G + B
 * (A, B) = ([a] G, [b] G) is the receiver's public key and a its view key; [r] A = [a] R, so a note is owned by its
 * receiver.  Scalars and points are laid out as for p252_dhke_batch.  base_uv (G) is a HOST pointer for every memory space,
 * as in p252_fixed_base_batch, and so is spend_B_uv in the scan.  Either one with a coordinate >= p or off the curve is
 * refused with P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.
 * Item validity:
 *   sender:   r < r_J, and A and B curve points with u, v < p (checked on the device per item, also for n_public == 1).  An
 *             invalid item gets ok[i] = 0, a zeroed R row and a zeroed note_pk row, and is counted once into *n_invalid.
 *   receiver: view_a < r_J (one scalar; if it is out of range every item is invalid), R a curve point with u, v < p, and
 *             both note_pk coordinates < p.  An invalid item gets owned[i] = 0 and is counted into *n_invalid, not
 *             *n_owned.  A note_pk with canonical coordinates off the curve is simply not owned.
 * *n_owned = number of owned[i] == 1.  n_owned / n_invalid: optional HOST pointers for both memory spaces (lifetime as for
 * p252_decrypt_batch).
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_public not 1 or n, DEVICE buffers other than ok / owned
 * not 16-byte aligned -> INVALID_ARGUMENT.
 * r, view_a, the shared points [r] A = [a] R and their hashes live only in the context's staging arenas, for both memory
 * spaces, and the arenas are zeroed on every exit path: both calls are synchronous (P252_ASYNC only defers the
 * publication of the counts to p252_sync).  Each item is constant time (no branch and no address depends on secret bits);
 * see DESIGN.md section 4. */
/* Sender: R_uv[i] = [r[i]] base, note_pk_uv[i] = [hash([r[i]] A)] base + B, with (A, B) =
 * (A_uv, B_uv)[n_public == 1 ? 0 : i]. */
int p252_stealth_address_batch(p252_ctx* ctx, const p252_jscalar* r, size_t n, const p252_fr* base_uv, const p252_fr* A_uv,
                               const p252_fr* B_uv, size_t n_public, p252_fr* R_uv, p252_fr* note_pk_uv, uint8_t* ok,
                               size_t* n_invalid, int flags);
/* Receiver: owned[i] = note_pk_uv[i] == [hash([view_a] R_uv[i])] base + spend_B. */
int p252_stealth_owns_batch(p252_ctx* ctx, const p252_jscalar* view_a, const p252_fr* spend_B_uv, const p252_fr* base_uv,
                            const p252_fr* R_uv, const p252_fr* note_pk_uv, size_t n, uint8_t* owned, size_t* n_owned,
                            size_t* n_invalid, int flags);

/* ---- Schnorr signatures over JubJub (jubjub-schnorr's SecretKey::sign / PublicKey::verify) -------------------------
 *   challenge(R, m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0]          (R affine; c < 2^250 < r_J)
 *   sign   (sk, r; m):        R = [r] G,  c = challenge(R, m),  u = (r - c sk) mod r_J,  signature = (u, R)
 *   verify (PK; (u, R), m):   ok  <=>  [u] G + [c] PK == R,  c = challenge(R, m)
 * PK = [sk] G.  Both scalar multiplications multiply by the canonical integer; there is no subgroup check (a torsion
 * component of PK passes through, as in p252_dhke_batch).  Scalars (sk, r, u) are p252_jscalar, points (u, v) pairs of
 * p252_fr, messages p252_fr, all laid out as for p252_dhke_batch.  base_uv (G) is a HOST pointer for every memory space,
 * as in p252_fixed_base_batch: a coordinate >= p or a point off the curve is refused with P252_ERR_INVALID_POINT before
 * anything runs, for every memory space and for n == 0.
 * r is one nonce per item; there is no broadcast on purpose.  The nonce must be secret, uniformly random and never used
 * twice: two signatures with the same sk and r on different messages reveal sk = (u1 - u2) / (c2 - c1) mod r_J.
 * Item validity (checked on the device, for both memory spaces):
 *   sign:   sk < r_J, r < r_J, msg < p.  An invalid item gets ok[i] = 0, a zeroed u row and a zeroed R row, and is counted
 *           once into *n_invalid.
 *   verify: u < r_J, msg < p, both coordinates of R < p, and PK a curve point with u, v < p (per item, also for
 *           n_public == 1).  An invalid item gets verified[i] = 0 and is counted into *n_invalid, not *n_verified.  An R
 *           with canonical coordinates off the curve is simply not verified (the projective equality implies R on the curve).
 * n_verified / n_invalid: optional HOST pointers for both memory spaces (lifetime as for p252_decrypt_batch).
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_secret / n_public not 1 or n, DEVICE buffers other than
 * ok / verified not 16-byte aligned -> INVALID_ARGUMENT.
 * Signing: sk and r live only in the context's staging arenas, for both memory spaces, and the arenas are zeroed on every
 * exit path: the call is synchronous (P252_ASYNC only defers the publication of *n_invalid to p252_sync).  Each item is
 * constant time (no branch and no address depends on sk or r); see DESIGN.md section 4.  Verification reads public data
 * only; as for p252_stealth_owns_batch, P252_ASYNC defers the publication of the counts to p252_sync. */
/* u[i], R_uv[i] = sign(sk[n_secret == 1 ? 0 : i], r[i]; msg[i]) */
int p252_schnorr_sign_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_jscalar* r,
                            const p252_fr* msg, size_t n, const p252_fr* base_uv, p252_jscalar* u_out, p252_fr* R_uv,
                            uint8_t* ok, size_t* n_invalid, int flags);
/* verified[i] = verify(pk_uv[n_public == 1 ? 0 : i]; (u[i], R_uv[i]), msg[i]) */
int p252_schnorr_verify_batch(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_jscalar* u,
                              const p252_fr* R_uv, const p252_fr* msg, size_t n, const p252_fr* base_uv,
                              uint8_t* verified, size_t* n_verified, size_t* n_invalid, int flags);

/* ---- Note nullifiers: which owned notes are spent (Phoenix SecretKey::gen_note_sk, Note::gen_nullifier) --------------
 *   hash(P)   = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]                  (the stealth calls' hash, < 2^250)
 *   note_sk   = (hash([a] R) + b) mod r_J
 *   pk'       = [note_sk] G'                                                          (affine)
 *   nullifier = Hash::digest(Domain::Other, [pk'.u, pk'.v, BlsScalar::from(pos)])[0]  (NOT truncated)
 * (a, b) is the wallet's secret key, R a note's ephemeral key and pos its position in the note tree; note_sk is the
 * discrete log of the note's stealth key: [note_sk] G = note_pk for the notes of p252_stealth_address_batch.  Scalars
 * and points are laid out as for p252_dhke_batch; pos is one u64 per note.  base_uv (G', GENERATOR_NUMS) is a HOST pointer
 * for every memory space, as in p252_fixed_base_batch: a coordinate >= p or a point off the curve is refused with
 * P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.  There is no built-in generator.
 * n_secret is 1 (one wallet key for every note) or n; a and b share it.
 * Item validity (checked on the device, for both memory spaces): a < r_J, b < r_J, and R a curve point with u, v < p.  pos
 * is any u64.  An invalid item gets ok[i] = 0 and a zeroed nullifier row, and is counted once into *n_invalid (optional
 * HOST pointer for both memory spaces, lifetime as for p252_decrypt_batch); the call returns P252_OK.
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_secret not 1 or n -> INVALID_ARGUMENT; so are DEVICE
 * buffers a, b, R_uv or nullifier not 16-byte aligned, and a DEVICE pos not 8-byte aligned (as the positions of the tree
 * calls).
 * a, b, the shared points [a] R, their hashes, note_sk and pk' live only in the context's staging arenas, for both memory
 * spaces, and the arenas are zeroed on every exit path: the call is synchronous (P252_ASYNC only defers the publication
 * of *n_invalid to p252_sync).  Each item is constant time (no branch and no address depends on a, b or note_sk); see
 * DESIGN.md section 4.  The context keeps the fixed-base table of one base: alternating calls with G (the stealth calls)
 * and G' on one context rebuild the 48 KB table on every switch; a context of its own for nullifiers avoids that. */
/* nullifier[i] = Hash::digest(Domain::Other, [pk'.u, pk'.v, BlsScalar::from(pos[i])])[0],
 *   pk' = [note_sk] base,  note_sk = (hash([a] R_uv[i]) + b) mod r_J,  (a, b) = (a, b)[n_secret == 1 ? 0 : i] */
int p252_nullifier_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret,
                         const p252_fr* base_uv, const p252_fr* R_uv, const uint64_t* pos, size_t n,
                         p252_fr* nullifier, uint8_t* ok, size_t* n_invalid, int flags);

/* ---- Double-key Schnorr signatures over G and G' (jubjub-schnorr's SignatureDouble) and spending a note -------------
 *   challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0]      (c < 2^250 < r_J)
 *   sign_double   (sk, r; m):            R = [r] G,  R' = [r] G',  u = (r - c sk) mod r_J,  signature = (u, R, R')
 *   verify_double ((PK, PK'); (u, R, R'), m):  ok  <=>  [u] G + [c] PK == R  AND  [u] G' + [c] PK' == R'
 *   note_sk(a, b, R_note) = (hash([a] R_note) + b) mod r_J     (hash: the stealth and nullifier calls' truncated digest)
 * The key pair of a signature is (PK, PK') = ([sk] G, [sk] G'); a Phoenix note is spent under (note_pk, pk') =
 * ([note_sk] G, [note_sk] G'), and pk' is the point p252_nullifier_batch hashes.  Both generators are caller arguments:
 * G_uv and Gp_uv (G' = GENERATOR_NUMS) are HOST pointers for every memory space, and a coordinate >= p or a point off the
 * curve in either is refused with P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.
 * There is no built-in generator.  Scalars, points and messages are laid out as for p252_schnorr_sign_batch; both scalar
 * multiplications multiply by the canonical integer and there is no subgroup check on PK or PK'.
 * r is one nonce per item (no broadcast), with the same rules as for p252_schnorr_sign_batch.  n_secret (shared by a and b
 * in the note call) and n_public (shared by PK and PK') are 1 or n.
 * Item validity (checked on the device, for both memory spaces):
 *   sign:      sk < r_J, r < r_J, msg < p.
 *   note sign: a < r_J, b < r_J, R_note a curve point with u, v < p, r < r_J, msg < p.
 *   verify:    u < r_J, msg < p, every coordinate of R and R' < p, PK and PK' curve points with u, v < p.
 * An invalid item gets ok[i] = 0 (verified[i] = 0) and zeroed u, R, R' (and pk') rows, and is counted once into
 * *n_invalid however many of its checks fail; verification counts it into *n_invalid, not *n_verified.  n_verified /
 * n_invalid: optional HOST pointers for both memory spaces (lifetime as for p252_decrypt_batch).
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_secret / n_public not 1 or n, DEVICE buffers other than
 * ok / verified not 16-byte aligned -> INVALID_ARGUMENT.
 * Signing: sk, r, a, b, [a] R_note, its hash and note_sk live only in the context's staging arenas, for both memory
 * spaces, and the arenas are zeroed on every exit path: both signing calls are synchronous (P252_ASYNC only defers the
 * publication of *n_invalid to p252_sync).  Each item is constant time (no branch and no address depends on a secret); see
 * DESIGN.md section 4.  pkp_uv, the note's pk' = [note_sk] G', is returned because a spend proof takes it as a witness: it
 * links the spend to the note (it is the preimage of the note's nullifier) and must stay as private as the note itself.
 * Verification reads public data only; P252_ASYNC defers the publication of the counts to p252_sync.
 * The context caches the fixed-base tables of G and G' of these three calls in two slots of their own, apart from the
 * one-base table of the other JubJub calls: none of these calls evicts that table, and no other call evicts theirs. */
/* u[i], R_uv[i], Rp_uv[i] = sign_double(sk[n_secret == 1 ? 0 : i], r[i]; msg[i]) */
int p252_schnorr_sign_double_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_jscalar* r,
                                   const p252_fr* msg, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv,
                                   p252_jscalar* u, p252_fr* R_uv, p252_fr* Rp_uv, uint8_t* ok, size_t* n_invalid,
                                   int flags);
/* verified[i] = verify_double((pk_uv, pkp_uv)[n_public == 1 ? 0 : i]; (u[i], R_uv[i], Rp_uv[i]), msg[i]) */
int p252_schnorr_verify_double_batch(p252_ctx* ctx, const p252_fr* pk_uv, const p252_fr* pkp_uv, size_t n_public,
                                     const p252_jscalar* u, const p252_fr* R_uv, const p252_fr* Rp_uv, const p252_fr* msg,
                                     size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, uint8_t* verified,
                                     size_t* n_verified, size_t* n_invalid, int flags);
/* u[i], R_uv[i], Rp_uv[i] = sign_double(note_sk, r[i]; msg[i]),  pkp_uv[i] = [note_sk] Gp,
 *   note_sk = (hash([a] note_R_uv[i]) + b) mod r_J,  (a, b) = (a, b)[n_secret == 1 ? 0 : i] */
int p252_note_sign_double_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret,
                                const p252_fr* note_R_uv, const p252_jscalar* r, const p252_fr* msg, size_t n,
                                const p252_fr* G_uv, const p252_fr* Gp_uv, p252_jscalar* u, p252_fr* R_uv, p252_fr* Rp_uv,
                                p252_fr* pkp_uv, uint8_t* ok, size_t* n_invalid, int flags);

/* ---- Phoenix note values: commitments, creating obfuscated notes and opening them ------------------------------------
 *   commit(v, blinder)    = C = [v] G + [blinder] G'                     (v a u64, blinder < r_J; G' = GENERATOR_NUMS)
 *   create (r, v, blinder, nonce; A, B):  R = [r] G,  S = [r] A,  note_pk = [hash(S)] G + B,  C = commit(v, blinder),
 *                                         cipher = encrypt([Fr(v), Fr(blinder)], S, nonce)       (L = 2: 3 scalars)
 *   open  (a; R, nonce, cipher, C):       S = [a] R,  (m0, m1) = decrypt(cipher, S, nonce); the note OPENS iff the
 *                                         authentication passes, m0 < 2^64, m1 < r_J and [m0] G + [m1] G' == C;
 *                                         then value = m0, blinder = m1
 *   hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0], as in the stealth calls; (A, B) is the receiver's
 *   public key and a its view key.  The range checks are this library's rule: an opening with m0 >= 2^64 or m1 >= r_J does
 *   not open even when its commitment matches.  A sender may encrypt an opening that does not match C; such a note cannot
 *   be spent, so a wallet counts only the value of notes that open.
 * G_uv and Gp_uv are HOST pointers for every memory space, as for the double-key calls; a coordinate >= p or a point off
 * the curve in either is refused with P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.
 * value: one uint64_t per item; blinder, r, a: p252_jscalar; nonce: p252_fr; points, C: (u, v) pairs of p252_fr; cipher:
 * 3 p252_fr per item.  n_public (shared by A and B) and n_secret (a) are 1 or n.
 * Item validity (checked on the device, for both memory spaces):
 *   commit: blinder < r_J.
 *   create: r < r_J, blinder < r_J, A and B curve points with u, v < p.
 *   open:   a < r_J, R a curve point with u, v < p.
 * An invalid item gets ok[i] = 0 and every output row it has zeroed (commitment; R, note_pk, commitment and cipher; value
 * and blinder), and is counted once however many of its checks fail.  In p252_note_open_batch ok[i] = 0 with zeroed value
 * and blinder also means the note did not open, and *n_failed counts every item with ok = 0 once, whatever the reason, as
 * p252_decrypt_batch_dhke does.  n_invalid / n_failed: optional HOST pointers for both memory spaces.
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_public / n_secret not 1 or n, DEVICE buffers not aligned
 * (value to 8 bytes, every other buffer but ok to 16) -> INVALID_ARGUMENT.
 * Secrets: r, v, blinder, a, the shared point S, hash(S) and the plaintext rows live only in the context's staging
 * arenas, for both memory spaces, and the arenas are zeroed on every exit path: all three calls are synchronous
 * (P252_ASYNC only defers the publication of the count to p252_sync).  Each item is constant time (no branch and no address
 * depends on a secret); see DESIGN.md section 4.  p252_note_open_batch returns value and blinder to the caller on purpose:
 * a spend proof takes them as witnesses, and they must stay as private as the note's secret key.
 * The fixed-base tables of G and G' are the double-key signature calls' two cache slots: a wallet that alternates these
 * calls with scans, nullifiers and spend signing rebuilds no table. */
/* commitment_uv[i] = commit(value[i], blinder[i]) */
int p252_value_commit_batch(p252_ctx* ctx, const uint64_t* value, const p252_jscalar* blinder, size_t n, const p252_fr* G_uv,
                            const p252_fr* Gp_uv, p252_fr* commitment_uv, uint8_t* ok, size_t* n_invalid, int flags);
/* R_uv[i], note_pk_uv[i], commitment_uv[i], cipher[3 i .. 3 i + 2] = create(r[i], value[i], blinder[i], nonce[i];
 *   (A_uv, B_uv)[n_public == 1 ? 0 : i]) */
int p252_note_create_batch(p252_ctx* ctx, const p252_jscalar* r, const uint64_t* value, const p252_jscalar* blinder,
                           const p252_fr* nonce, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, const p252_fr* A_uv,
                           const p252_fr* B_uv, size_t n_public, p252_fr* R_uv, p252_fr* note_pk_uv, p252_fr* commitment_uv,
                           p252_fr* cipher, uint8_t* ok, size_t* n_invalid, int flags);
/* value[i], blinder[i], ok[i] = open(a[n_secret == 1 ? 0 : i]; R_uv[i], nonce[i], cipher[3 i .. 3 i + 2],
 *   commitment_uv[i]) */
int p252_note_open_batch(p252_ctx* ctx, const p252_jscalar* a, size_t n_secret, const p252_fr* R_uv, const p252_fr* nonce,
                         const p252_fr* cipher, const p252_fr* commitment_uv, size_t n, const p252_fr* G_uv,
                         const p252_fr* Gp_uv, uint64_t* value, p252_jscalar* blinder, uint8_t* ok, size_t* n_failed,
                         int flags);

/* ---- Phoenix wallet scans: which of several keys owns each note, and the owned notes' nullifiers, openings and totals ---
 * The keys are (a_j, b_j) for j < n_keys, 1 <= n_keys <= P252_WALLET_MAX_KEYS; B_j = [b_j] G is derived on the device.
 * For note i (R, note_pk, pos, nonce, cipher, C):
 *   owner[i]      = the smallest j whose key owns the note as p252_stealth_owns_batch decides it (note_pk ==
 *                   [hash([a_j] R)] G + B_j), -1 if none does; with duplicate keys the smallest index wins
 *   nullifier[i]  = the row p252_nullifier_batch(a_j, b_j, G', R, pos) returns, for j = owner[i]
 *   value[i], blinder[i], opened[i] = what p252_note_open_batch(a_j; R, nonce, cipher, C, G, G') returns, range and
 *                   commitment checks included.  An owned note that does not open keeps its owner and nullifier (it is
 *                   the wallet's, but cannot be spent), with opened = 0 and value and blinder zeroed.
 *   A note no key owns gets zeroed nullifier, value and blinder rows and opened = 0.
 * key_totals: n_keys rows of 4 uint64_t, row j = {value_lo, value_hi, n_owned, n_opened}: the exact 128-bit sum of value
 * over the notes key j owns that opened, how many notes it owns and how many of them opened.
 * Validity (checked on the device, for both memory spaces):
 *   a key is bad when a_j >= r_J or b_j >= r_J: it owns no note, and *n_bad_keys counts it;
 *   a note is invalid when R is not a curve point with u, v < p or a coordinate of note_pk is >= p: owner -1, zeroed
 *   rows, and *n_invalid counts it once.  A note_pk with canonical coordinates off the curve is simply not owned.  Cipher,
 *   nonce and C are judged as p252_note_open_batch judges them.
 * G_uv and Gp_uv are HOST pointers for every memory space, as for the note calls; a coordinate >= p or a point off the
 * curve in either is refused with P252_ERR_INVALID_POINT before anything runs, also for n == 0.  n == 0 runs nothing: it
 * writes nothing and counts nothing (both counts are 0, bad keys included).
 * a, b: n_keys p252_jscalar rows; R, note_pk, C: (u, v) pairs of p252_fr; pos: uint64_t; nonce: p252_fr; cipher: 3
 * p252_fr per note; owner: int32_t; value: uint64_t; blinder: p252_jscalar; opened: bytes.  n_invalid, n_bad_keys:
 * optional HOST pointers for both memory spaces.
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_keys == 0 or > P252_WALLET_MAX_KEYS, DEVICE buffers
 * not aligned (pos and value to 8 bytes, owner to 4, opened to none, every other buffer to 16) -> INVALID_ARGUMENT.
 * Secrets and timing: a, b, every [a_j] R, its hash, note_sk, pk' and the plaintexts live only in the context's staging
 * arenas, for both memory spaces, and the arenas are zeroed on every exit path.  The call is synchronous: P252_ASYNC only
 * defers the publication of the counts to p252_sync.  Each (note, key) pair runs the same schedule, and so does the second
 * phase of each owned note; the one thing that steers the schedule is ownership, which the call returns anyway: owned
 * notes are compacted before the second phase.  The owner's rows are read by masked selects over all n_keys rows, so no
 * address depends on which key matched (DESIGN.md section 4).
 * The fixed-base tables of G and G' are the double-key and note calls' two cache slots: the call evicts no table, and
 * alternating it with those calls rebuilds none. */
#define P252_WALLET_MAX_KEYS 256
/* owner[i], nullifier[i], value[i], blinder[i], opened[i] = scan(keys; note i);  key_totals[4 j .. 4 j + 3] = totals of
 * key j */
int p252_wallet_scan_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_keys, const p252_fr* R_uv,
                           const p252_fr* note_pk_uv, const uint64_t* pos, const p252_fr* nonce, const p252_fr* cipher,
                           const p252_fr* commitment_uv, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, int32_t* owner,
                           p252_fr* nullifier, uint64_t* value, p252_jscalar* blinder, uint8_t* opened, uint64_t* key_totals,
                           size_t* n_invalid, size_t* n_bad_keys, int flags);

/* ---- JubJub ElGamal and the encrypted sender of a Phoenix note (phoenix-core's elgamal, Sender::Encryption) ---------
 *   elgamal_encrypt(PK, M; r)  = (c1, c2) = ([r] G, M + [r] PK)
 *   elgamal_decrypt(sk; c1, c2) = c2 - [sk] c1
 *   sender_encrypt(note_pk; (A, B); (r_A, r_B)) = [encrypt(note_pk, A; r_A), encrypt(note_pk, B; r_B)]
 *   sender_decrypt(a, b; R, note_pk, enc): note_sk = (hash([a] R) + b) mod r_J (p252_nullifier_batch's note_sk); the note
 *     is OWNED iff [note_sk] G == note_pk, and then A = c2_A - [note_sk] c1_A, B = c2_B - [note_sk] c1_B
 * hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0], as in the stealth calls; (A, B) is the sender's public
 * key and (a, b) the receiver's secret key.  Scalar multiplications multiply by the canonical integer; there is no
 * subgroup check, as in p252_dhke_batch.
 * ElGamal is NOT authenticated: p252_elgamal_decrypt_batch under a wrong key returns some other curve point with ok = 1.
 * That is why the sender decrypt checks ownership first: a note the key does not own gets ok = 0 and zeroed A and B rows,
 * not a plausible-looking wrong sender.
 * Layouts: scalars p252_jscalar; points (u, v) pairs of p252_fr, outputs affine.  blinder: 2 p252_jscalar per note,
 * [r_A, r_B]; sender_enc: 8 p252_fr per note (256 bytes), [c1_A, c2_A, c1_B, c2_B] as (u, v) pairs.  n_public (PK),
 * n_sender (A and B together) and n_secret (sk; a and b together) are 1 or n.  r and the blinders are one per item, with
 * no broadcast: two messages encrypted under one PK with the same r reveal M1 - M2 (c2 - c2'), so never reuse r.
 * G_uv is a HOST pointer for every memory space, as for the note calls: a coordinate >= p or a point off the curve is
 * refused with P252_ERR_INVALID_POINT before anything runs, for every memory space and for n == 0.
 * p252_elgamal_decrypt_batch takes no G.
 * Item validity (checked on the device, for both memory spaces):
 *   encrypt:        r < r_J (each blinder), PK / note_pk and M / A / B curve points with u, v < p.
 *   decrypt:        sk < r_J (a and b), every ciphertext point a curve point with u, v < p, R a curve point with u, v < p.
 * r = 0, sk = 0, note_sk = 0, an identity M or PK and small-order points are valid and give what the formulas give.
 * An invalid item gets ok[i] = 0 and zeroed output rows, and is counted once however many of its checks fail.  In
 * p252_note_sender_decrypt_batch ok[i] = 0 also means the note is not owned (a note_pk off the curve or with a coordinate
 * >= p is not owned), and *n_failed counts every item with ok = 0 once, whatever the reason, as p252_note_open_batch
 * does.  n_invalid / n_failed: optional HOST pointers for both memory spaces.  n == 0 writes and counts nothing.
 * Batch checks, before anything runs: a NULL buffer with n > 0, n_public / n_sender / n_secret not 1 or n, DEVICE buffers
 * other than ok not 16-byte aligned -> INVALID_ARGUMENT.
 * Secrets: r, the blinders, M, (A, B), sk, a, b, [a] R, its hash and note_sk live only in the context's staging arenas,
 * for both memory spaces, and the arenas are zeroed on every exit path: all four calls are synchronous (P252_ASYNC only
 * defers the publication of the count to p252_sync).  Each item is constant time (no branch and no address depends on a
 * secret); see DESIGN.md section 4.
 * G's fixed-base table is the first of the double-key and note calls' two cache slots: after p252_note_create_batch with
 * the same G the encrypt calls and the sender decrypt build no table, and none of them evicts G' or the one-base table. */
/* c1_uv[i], c2_uv[i] = elgamal_encrypt(pk_uv[n_public == 1 ? 0 : i], msg_uv[i]; r[i]) */
int p252_elgamal_encrypt_batch(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_fr* msg_uv,
                               const p252_jscalar* r, size_t n, const p252_fr* G_uv, p252_fr* c1_uv, p252_fr* c2_uv,
                               uint8_t* ok, size_t* n_invalid, int flags);
/* msg_uv[i] = elgamal_decrypt(sk[n_secret == 1 ? 0 : i]; c1_uv[i], c2_uv[i]) */
int p252_elgamal_decrypt_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_fr* c1_uv,
                               const p252_fr* c2_uv, size_t n, p252_fr* msg_uv, uint8_t* ok, size_t* n_invalid, int flags);
/* sender_enc[8 i .. 8 i + 7] = sender_encrypt(note_pk_uv[i]; (sender_A_uv, sender_B_uv)[n_sender == 1 ? 0 : i];
 *   (blinder[2 i], blinder[2 i + 1])) */
int p252_note_sender_encrypt_batch(p252_ctx* ctx, const p252_fr* note_pk_uv, const p252_fr* sender_A_uv,
                                   const p252_fr* sender_B_uv, size_t n_sender, const p252_jscalar* blinder, size_t n,
                                   const p252_fr* G_uv, p252_fr* sender_enc, uint8_t* ok, size_t* n_invalid, int flags);
/* sender_A_uv[i], sender_B_uv[i], ok[i] = sender_decrypt((a, b)[n_secret == 1 ? 0 : i]; R_uv[i], note_pk_uv[i],
 *   sender_enc[8 i .. 8 i + 7]) */
int p252_note_sender_decrypt_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret,
                                   const p252_fr* R_uv, const p252_fr* note_pk_uv, const p252_fr* sender_enc, size_t n,
                                   const p252_fr* G_uv, p252_fr* sender_A_uv, p252_fr* sender_B_uv, uint8_t* ok,
                                   size_t* n_failed, int flags);

/* ---- JubJub point compression (dusk-jubjub's JubJubAffine::to_bytes / from_bytes) -----------------------------------
 *   encoding:  the 32 little-endian bytes of canonical v, with bit 255 (bytes[31] >> 7) = the low bit of canonical u
 *   decoding:  sign = bit 255, cleared; the remaining 255-bit value is v (rejected if >= p); u^2 = (v^2 - 1) / (1 + d v^2)
 *              (rejected if not a square); u is the root whose canonical low bit is sign.
 * A set sign bit with u = 0 (v = +-1) is accepted and decodes to the same point, as pre-ZIP-216 jubjub does; 32 zero
 * bytes decode to (sqrt(-1), 0), a point of order 4.  There is no subgroup check.  Points are (u, v) pairs of p252_fr
 * (Montgomery limbs), laid out as for p252_dhke_batch; bytes are n x 32.
 * Item validity (checked on the device, for both memory spaces):
 *   from_bytes: v < p and u^2 a square.  An invalid item gets ok[i] = 0 and the row (0, 0), which is not a curve point.
 *   to_bytes:   u, v < p and (u, v) on the curve.  An invalid item gets ok[i] = 0 and 32 bytes of 0xff (v = 2^255 - 1 >= p,
 *               so from_bytes rejects it; zero bytes would decode).
 * Invalid items are counted into *n_invalid (optional HOST pointer, lifetime as for p252_decrypt_batch); the call still
 * returns P252_OK.  Batch checks, before anything runs: a NULL buffer (ok included) with n > 0, DEVICE buffers other than
 * ok not 16-byte aligned -> INVALID_ARGUMENT.  Public data only: with P252_ASYNC, DEVICE calls defer the publication of
 * *n_invalid to p252_sync. */
/* out_uv[i] = JubJubAffine::from_bytes(bytes[32 i .. 32 i + 32]) */
int p252_points_from_bytes(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out_uv, uint8_t* ok,
                           size_t* n_invalid, int flags);
/* bytes[32 i ..] = JubJubAffine::to_bytes(uv[i]) */
int p252_points_to_bytes(p252_ctx* ctx, const p252_fr* uv, size_t n, uint8_t* bytes, uint8_t* ok,
                         size_t* n_invalid, int flags);

/* ---- JubJub multi-scalar multiplication and all-or-nothing Schnorr batch verification ------------------------------
 * VARIABLE TIME: both calls read public data only, and scalar bits become bucket indexes (memory addresses) and branch
 * conditions on the device.  Never pass a secret scalar.
 * Layouts: scalars, weights and u are p252_jscalar; points, R and PK (u, v) pairs of p252_fr; messages p252_fr; all as in
 * p252_schnorr_verify_batch, and challenge(R, m) is its challenge.  base_uv (G) is a HOST pointer for every memory space,
 * checked on the host as in p252_fixed_base_batch: a coordinate >= p or a point off the curve is refused with
 * P252_ERR_INVALID_POINT before anything runs, also for n == 0.  out_uv lives in the call's memory space; all_verified is a
 * HOST pointer and must not be NULL.
 * Item validity (checked on the device, for both memory spaces):
 *   msm:        scalar < r_J, both coordinates < p, the point on the curve.  An invalid item is skipped (it adds the
 *               identity) and counted into *n_invalid.
 *   verify_all: as an invalid item of p252_schnorr_verify_batch (u >= r_J, msg >= p, an R coordinate >= p, PK not a curve
 *               point with u, v < p), or weight >= r_J.  An invalid item is counted into *n_invalid and makes the answer 0.
 *               An R with canonical coordinates off the curve is not invalid, but makes the answer 0 too.
 * Cofactored semantics: *all_verified = 1 iff no item is invalid, every R is on the curve and
 *   [8] ( [sum z_i u_i] G + sum [z_i c_i] PK_i - sum [z_i] R_i ) == identity,   c_i = challenge(R_i, msg_i), z_i = weight[i].
 * Except with probability about 2^-128 over uniformly random 128-bit weights, that is exactly when every item satisfies
 * the cofactored equation [8] ([u_i] G + [c_i] PK_i - R_i) == identity.  For PK and R in the prime-order subgroup this is
 * per-item verification; a signature whose R is shifted by a small-order point fails p252_schnorr_verify_batch and passes
 * here.  (Without the cofactor a random combination is not sound against torsion components.)
 * Weights come from the caller: uniformly random, unpredictable to the signers and nonzero (128 bits are enough).  Any
 * z < r_J is accepted; a zero weight leaves its item unchecked.  The library generates no randomness.
 * n == 0: the MSM is the identity (0, 1) and *all_verified = 1.  n_invalid: optional HOST pointer for both memory spaces
 * (lifetime as for p252_decrypt_batch).
 * Batch checks, before anything runs: a NULL buffer with n > 0 (out_uv and all_verified always), n_public not 1 or n,
 * DEVICE buffers not 16-byte aligned -> INVALID_ARGUMENT.  With P252_ASYNC, DEVICE calls defer the publication of
 * *n_invalid and *all_verified to p252_sync (and out_uv is complete after it); HOST calls return with them published.
 * The work is one bucket (Pippenger) multi-scalar multiplication over chunks of the batch; see DESIGN.md section 4.  Its
 * temporaries live in the context's staging arenas, which the first call grows to about 100-145 MiB each (three per
 * context) and which are kept until p252_destroy. */
/* out_uv = sum over valid items of [scalars[i]] points_uv[i] (JubJubAffine; the identity is (0, 1), also for n == 0) */
int p252_jubjub_msm(p252_ctx* ctx, const p252_jscalar* scalars, const p252_fr* points_uv, size_t n,
                    p252_fr* out_uv, size_t* n_invalid, int flags);
/* *all_verified = 1 iff no item is invalid, every R is on the curve, and
 *   [8] ( [sum z_i u_i] G + sum [z_i c_i] PK_i - sum [z_i] R_i ) == identity,   c_i = challenge(R_i, msg_i),
 * with PK_i = pk_uv[n_public == 1 ? 0 : i] and z_i = weight[i] */
int p252_schnorr_verify_all(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_jscalar* u,
                            const p252_fr* R_uv, const p252_fr* msg, const p252_jscalar* weight, size_t n,
                            const p252_fr* base_uv, uint8_t* all_verified, size_t* n_invalid, int flags);

/* ---- All-or-nothing batch verification of double-key Schnorr signatures (SignatureDouble) ---------------------------
 * One answer for n double-key signatures, by one bucket multi-scalar multiplication over G and G'.  VARIABLE TIME, public
 * data only, as p252_schnorr_verify_all.  Layouts, challenge2(R, R', m), G_uv / Gp_uv (HOST pointers, a bad one refused
 * with P252_ERR_INVALID_POINT before anything runs, also for n == 0) and n_public (shared by PK and PK') are those of
 * p252_schnorr_verify_double_batch; weight and weight_p are p252_jscalar rows in the call's memory space; all_verified is
 * a HOST pointer and must not be NULL.
 * Item validity (checked on the device, for both memory spaces): as an invalid item of p252_schnorr_verify_double_batch
 * (u >= r_J, msg >= p, a coordinate of R or R' >= p, PK or PK' not a curve point with u, v < p), or weight >= r_J, or
 * weight_p >= r_J.  An invalid item is counted once into *n_invalid and makes the answer 0.  An R or R' with canonical
 * coordinates off the curve is not invalid, but makes the answer 0 too.
 * Cofactored semantics: *all_verified = 1 iff no item is invalid, every R and R' is on the curve and
 *   [8] ( [sum z_i u_i] G + [sum z'_i u_i] G' + sum [z_i c_i] PK_i + sum [z'_i c_i] PK'_i - sum [z_i] R_i - sum [z'_i] R'_i )
 *   == identity,   c_i = challenge2(R_i, R'_i, msg_i),  z_i = weight[i],  z'_i = weight_p[i].
 * Except with probability about 2^-128 over independent uniformly random 128-bit weights, that is exactly when every item
 * satisfies both cofactored equations [8] ([u_i] G + [c_i] PK_i - R_i) == identity and
 * [8] ([u_i] G' + [c_i] PK'_i - R'_i) == identity.  A signature whose R (or R') is shifted by a small-order point fails
 * p252_schnorr_verify_double_batch and passes here.
 * The two weight arrays must be drawn independently: with weight_p == weight the two equations of an item are only
 * checked as a sum, and a signer can make them fail by opposite amounts that cancel.  (R = [r] G + D and R' = [r] G' - D
 * for any point D, signed as usual, fail per-item verification and pass the sum with equal weights.)  Weights come from
 * the caller: uniformly random, unpredictable to the signers and nonzero (128 bits are enough); any z < r_J is accepted,
 * and a zero weight leaves its equation unchecked.  The library generates no randomness.
 * n == 0: *all_verified = 1.  n_invalid: optional HOST pointer for both memory spaces (lifetime as for
 * p252_decrypt_batch).
 * Batch checks, before anything runs: a NULL buffer with n > 0 (all_verified always), n_public not 1 or n, DEVICE buffers
 * not 16-byte aligned -> INVALID_ARGUMENT.  With P252_ASYNC, DEVICE calls defer the publication of *n_invalid and
 * *all_verified to p252_sync; HOST calls return with them published.
 * The tables of G and G' come from the two cache slots of the double-key calls: this call, schnorr_verify_double_batch and
 * the double-key signing calls on one context build no table when they alternate, and none of them evicts the one-base
 * table.  The MSM temporaries live in the context's staging arenas, as for p252_schnorr_verify_all; see DESIGN.md
 * section 4. */
/* *all_verified = 1 iff no item is invalid, every R and R' is on the curve, and the cofactored sum above is the identity,
 * with (PK_i, PK'_i) = (pk_uv, pkp_uv)[n_public == 1 ? 0 : i] */
int p252_schnorr_verify_double_all(p252_ctx* ctx, const p252_fr* pk_uv, const p252_fr* pkp_uv, size_t n_public,
                                   const p252_jscalar* u, const p252_fr* R_uv, const p252_fr* Rp_uv, const p252_fr* msg,
                                   const p252_jscalar* weight, const p252_jscalar* weight_p, size_t n,
                                   const p252_fr* G_uv, const p252_fr* Gp_uv, uint8_t* all_verified,
                                   size_t* n_invalid, int flags);

/* One level of an arity-4 tree: parents[i] = Hash::digest(Domain::Merkle4, children[4i..4i+4])
 * (src/hash.rs:22-26). */
int p252_merkle4_level(p252_ctx* ctx, const p252_fr* children, size_t n_parents, p252_fr* parents, int flags);
/* Number of nodes above the leaves of a full arity-4 tree: (n_leaves-1)/3; n_leaves must be 4^k. */
int p252_merkle4_tree_nodes(size_t n_leaves, size_t* n_internal, int* n_levels);
/* Whole tree on one GPU.  nodes_out: all internal levels, bottom-up, concatenated
 * (n_leaves/4 + n_leaves/16 + ... + 1 scalars); the root is the last element. */
int p252_merkle4_build(p252_ctx* ctx, const p252_fr* leaves, size_t n_leaves, p252_fr* nodes_out, int flags);

/* The same for arity 2 or 4 (node = Hash::digest(Domain::Merkle2 | Merkle4, children), src/hash.rs:22-31):
 * internal nodes = (n_leaves - 1) / (arity - 1); n_leaves must be a power of the arity. */
int p252_merkle_tree_nodes(int arity, size_t n_leaves, size_t* n_internal, int* n_levels);
int p252_merkle_build(p252_ctx* ctx, int arity, const p252_fr* leaves, size_t n_leaves, p252_fr* nodes_out, int flags);

/* ---- Merkle openings (consumer: poseidon-merkle `Opening`, AGENTS.md:62-66; node hash src/hash.rs:22-31) ------
 * A tree is `leaves` (n_leaves = arity^depth) + `nodes` as written by p252_merkle_build.  The opening of leaf i
 * holds, for every level l = 0..depth-1 (0 = the leaf level), the WHOLE sibling group of the path node: the
 * `arity` items at [g*arity, (g+1)*arity) of level l with g = i / arity^(l+1); the path node sits at offset
 * (i / arity^l) % arity inside its group.  Empty slots of a sparse tree are the zero scalar (src/hash.rs:22-31).
 * paths: n x depth x arity scalars, item-major.  leaf_idx lives in the same memory space as the other buffers.  An index
 * >= n_leaves is P252_ERR_INVALID_ARGUMENT for HOST buffers; for DEVICE buffers (not inspected on the host) its opening
 * is all zero, which no root verifies. */
int p252_merkle_open_batch(p252_ctx* ctx, int arity, const p252_fr* leaves, size_t n_leaves, const p252_fr* nodes,
                           const uint64_t* leaf_idx, size_t n, p252_fr* paths_out, int flags);
/* n x Opening::verify: cur = leaf_items[i]; for every level: paths[i][l][pos] must equal cur, then
 * cur = Hash::digest(Domain::Merkle{arity}, paths[i][l]); finally cur must equal *root.  ok[i] = 1 iff all hold
 * (depth permutations per item, fused with the checks in one kernel).  root is a HOST pointer; *n_failed as in
 * p252_decrypt_batch. */
int p252_merkle_verify_batch(p252_ctx* ctx, int arity, int depth, const p252_fr* leaf_items, const uint64_t* leaf_idx,
                             const p252_fr* paths, const p252_fr* root, size_t n, uint8_t* ok, size_t* n_failed,
                             int flags);

/* ---- fixed-height trees with batched updates (consumer: poseidon-merkle `Tree<T, H, A>`) ------------------------
 * A tree of arity A (2 or 4) and height H (1..64) has room for capacity <= A^H leaves and holds an occupied prefix
 * [0, n_leaves).  Level l has m_l = ceil(n_leaves / A^l) occupied nodes; node j of level l+1 is
 * Hash::digest(Domain::Merkle{A}, level_l[j*A .. j*A+A]) where slots at or beyond m_l read as the zero scalar, and a
 * node whose whole subtree is empty IS the zero scalar (not the digest of zeros; src/hash.rs:24-26).  The root is the
 * single node of level H; for n_leaves = 0 it is zero.
 * Layout (p252_mtree_layout): level l < H has A * ceil(ceil(capacity / A^l) / A) slots, level H one slot; `leaves`
 * holds level 0, `nodes` levels 1..H bottom-up, root last.  With capacity = n_leaves = A^H this is exactly the layout of
 * p252_merkle_build.  The library owns every slot beyond a level's prefix, leaves[n_leaves, leaf_slots) included:
 * build and update keep them zero, and the caller must not write them.
 * The struct and both buffers belong to the caller; flags say where the buffers live (as for every batch call). */
typedef struct p252_mtree {
    uint32_t struct_size; /* sizeof(p252_mtree)                                                        */
    int32_t arity;        /* 2 or 4                                                                    */
    int32_t height;       /* levels above the leaves; capacity <= arity^height                         */
    int32_t reserved;
    uint64_t capacity;    /* leaves the buffers are laid out for                                       */
    uint64_t n_leaves;    /* occupied prefix; advanced by p252_mtree_update on success                 */
    p252_fr* leaves;      /* leaf_slots scalars  (HOST or DEVICE per the call's flags)                 */
    p252_fr* nodes;       /* node_slots scalars, levels 1..height bottom-up, root last                 */
} p252_mtree;
/* Slot counts of a tree; level_offset (height+1 entries, or NULL): [l] = first slot of level l inside nodes for
 * l >= 1, [0] = 0.  Pure host arithmetic (no GPU needed). */
int p252_mtree_layout(int arity, int height, uint64_t capacity, uint64_t* leaf_slots, uint64_t* node_slots,
                      uint64_t* level_offset);
/* Rebuild every node from leaves[0, n_leaves) (and zero every slot beyond the prefixes).  HOST trees are staged to
 * the device and the node slots copied back. */
int p252_mtree_build(p252_ctx* ctx, p252_mtree* tree, int flags);
/* One batch: overwrite leaves idx[i] < n_leaves with values[i] (the last write in batch order wins), then append
 * n_append leaves at [n_leaves, n_leaves + n_append); afterwards leaves and nodes are bit-identical to a fresh build
 * and tree->n_leaves has advanced by n_append.  Only the nodes on the touched paths are rehashed: each distinct dirty
 * node once, about (n_upd + n_append) * height permutations for a sparse batch.  idx / values / append live in the
 * same memory space as the tree; n_upd + n_append < 2^31.
 *   HOST: an index >= n_leaves is P252_ERR_INVALID_ARGUMENT and nothing is modified.
 *   DEVICE: indices are not inspected on the host; an update with idx >= n_leaves is skipped on the device and
 *   counted into *n_rejected (optional HOST pointer, 0 for HOST calls).  Temporaries are stream-ordered; with
 *   P252_ASYNC nothing is synchronised.
 * n_leaves + n_append > capacity is P252_ERR_INVALID_ARGUMENT (nothing modified).  After a CUDA failure the tree's
 * contents are unspecified and n_leaves is unchanged: rebuild it.
 * Lifetime of *n_rejected (and of *n_failed of p252_decrypt_batch / p252_merkle_verify_batch): for DEVICE calls with
 * P252_ASYNC it is written by a host function on the context's stream, so the size_t must stay valid until
 * p252_sync (or p252_destroy) has returned. */
int p252_mtree_update(p252_ctx* ctx, p252_mtree* tree, const uint64_t* idx, const p252_fr* values, size_t n_upd,
                      const p252_fr* append, size_t n_append, size_t* n_rejected, int flags);
/* Openings of leaves leaf_idx[0..n) in the format of p252_merkle_open_batch (n x height x arity, slots beyond a level's
 * prefix are zero); p252_merkle_verify_batch with depth = height verifies them.  An index >= n_leaves is
 * P252_ERR_INVALID_ARGUMENT for HOST buffers and an all-zero opening for DEVICE buffers. */
int p252_mtree_open_batch(p252_ctx* ctx, const p252_mtree* tree, const uint64_t* leaf_idx, size_t n, p252_fr* paths_out,
                          int flags);

/* ---- sparse fixed-height trees: inserts and removals at any position (poseidon-merkle `Tree::insert` / `remove`) ----
 * Arity A (2 or 4), height H (1..64), capacity <= A^H.  Each position in [0, capacity) is present (holds a value) or
 * absent.  Level-0 slot j holds the leaf value if j is present and 0 otherwise.  A node of level l >= 1 is present iff
 * one of its A children is present; a present node is Hash::digest(Domain::Merkle{A}, its A children's slots) (absent
 * children read as 0), an absent node IS 0 and is never hashed (src/hash.rs:24-26).  The root is the single node of
 * level H, 0 for an empty tree.  A present leaf whose value is zero is not an absent one: its parent is H(0, ..).
 * Layout: exactly p252_mtree_layout's, plus one presence byte per slot (1 = present) in the same order -- leaf_slots
 * bytes for the leaves, then node_slots bytes for levels 1..H.  If the present set is [0, n), leaves and nodes are
 * bit-identical to those of a p252_mtree with n_leaves = n.  The library owns every absent slot (value and presence of
 * absent leaves, every node and node presence byte, slots at or beyond capacity) and keeps them consistent; the caller
 * writes leaves and leaf presence only before p252_smtree_build.  Struct and buffers belong to the caller; flags say
 * where the buffers live.  DEVICE buffers: leaves / nodes 16-byte aligned, present 4-byte aligned, positions 8-byte
 * aligned. */
typedef struct p252_smtree {
    uint32_t struct_size; /* sizeof(p252_smtree)                                                       */
    int32_t arity;        /* 2 or 4                                                                    */
    int32_t height;       /* levels above the leaves; capacity <= arity^height                         */
    int32_t reserved;
    uint64_t capacity;    /* positions [0, capacity)                                                   */
    p252_fr* leaves;      /* leaf_slots scalars (p252_mtree_layout)                                    */
    p252_fr* nodes;       /* node_slots scalars, levels 1..height bottom-up, root last                 */
    uint8_t* present;     /* leaf_slots + node_slots bytes, leaves then nodes: 1 = present, 0 = absent  */
} p252_smtree;
/* Rebuild every node and node presence byte from the leaves and the leaf presence bytes (a non-zero byte below capacity
 * is present; build stores 1), and zero the value of every absent leaf.  Hashes only present nodes: the work is
 * proportional to the present nodes, plus a pass over the leaf presence bytes.  HOST trees are staged to the device. */
int p252_smtree_build(p252_ctx* ctx, p252_smtree* tree, int flags);
/* One batch of operations (pos[i], op[i], values[i]): op 0 inserts or overwrites, op 1 removes (values[i] is not read);
 * op = NULL means all inserts.  The result equals applying the operations one after another in batch order: the last
 * operation on a position wins, removing an absent position does nothing.  Only the nodes on the touched paths are
 * revisited, each distinct one once; a node whose children all became absent is zeroed without hashing.  pos / op /
 * values live in the same memory space as the tree (values is required for n > 0); n < 2^31.
 *   HOST: a position >= capacity or an op other than 0/1 is P252_ERR_INVALID_ARGUMENT and nothing is modified.
 *   DEVICE: such an item is skipped on the device and counted into *n_rejected (optional HOST pointer, 0 for HOST
 *   calls; lifetime as for p252_mtree_update).  Temporaries are stream-ordered; with P252_ASYNC nothing is synchronised.
 * After a CUDA failure the tree's contents are unspecified: rebuild it. */
int p252_smtree_update(p252_ctx* ctx, p252_smtree* tree, const uint64_t* pos, const uint8_t* op, const p252_fr* values,
                       size_t n, size_t* n_rejected, int flags);
/* *n_present (HOST pointer) = number of present positions.  DEVICE trees: counted on the device; with P252_ASYNC the
 * value is written by a host function on the context's stream (lifetime as *n_rejected). */
int p252_smtree_len(p252_ctx* ctx, const p252_smtree* tree, uint64_t* n_present, int flags);
/* Openings of positions pos[0..n) in the format of p252_mtree_open_batch (n x height x arity, absent slots 0); they
 * verify with p252_merkle_verify_batch, depth = height.  An absent position or one >= capacity is
 * P252_ERR_INVALID_ARGUMENT for HOST buffers and an all-zero opening for DEVICE buffers. */
int p252_smtree_open_batch(p252_ctx* ctx, const p252_smtree* tree, const uint64_t* pos, size_t n, p252_fr* paths_out,
                           int flags);

/* ---- compact sparse trees: storage proportional to the present leaves (poseidon-merkle `Tree<T, H, A>` at any height) --
 * The semantics of p252_smtree at positions [0, arity^height): presence, and the empty-subtree rule (a node is present
 * iff one of its children is; a present node is Hash::digest(Domain::Merkle{A}, its A child slots) with absent children
 * read as 0; an absent node is 0 and never hashed).  Heights up to 64 with arity 2 and 32 with arity 4, so that every
 * u64 can be a position.  Storage is the sorted list of present nodes, level by level: level l holds exactly its
 * present nodes as (index, value) pairs, indices ascending, packed from the level's first slot; every slot past
 * count[l] is zero (keys and values).  This canonical form makes buffers comparable bit for bit, and for any present set
 * a p252_smtree of the same (arity, height) can hold, level l is the list of that tree's present slots of level l.
 * The root is values[level_offset[height]], 0 for the empty tree.  Struct and buffers belong to the caller; an
 * all-zero buffer set is the empty tree.  DEVICE buffers: values 16-byte aligned, keys / count / positions 8-byte
 * aligned.  An update reads and writes every present node of every level (about 80 B per present node per level) and
 * hashes only the dirty paths; its stream-ordered temporaries take about 48 B per max_leaves plus 250 B per item. */
typedef struct p252_ctree {
    uint32_t struct_size; /* sizeof(p252_ctree)                                                          */
    int32_t arity;        /* 2 or 4                                                                       */
    int32_t height;       /* 1..64, and arity^height <= 2^64 (arity 4: height <= 32)                      */
    int32_t reserved;
    uint64_t max_leaves;  /* bound on present positions the buffers are laid out for, 1 .. 2^31 - 1       */
    uint64_t* keys;       /* total_slots: per level the sorted node indices, level l at level_offset[l]   */
    p252_fr* values;      /* total_slots: the matching node values                                        */
    uint64_t* count;      /* height + 1 entries: present nodes of level l (count[0] = number of leaves)   */
} p252_ctree;
/* Level l has min(max_leaves, arity^(height - l)) slots (level height: 1), starting at level_offset[l] (height + 1
 * entries, optional); *total_slots (optional) is their sum.  Pure host arithmetic. */
int p252_ctree_layout(int arity, int height, uint64_t max_leaves, uint64_t* total_slots, uint64_t* level_offset);
/* One batch of operations (pos[i], op[i], values[i]) with the semantics of p252_smtree_update: op 0 inserts or
 * overwrites, op 1 removes (values[i] not read), op = NULL means all inserts; the result equals applying them in batch
 * order.  There is no separate build: inserting n leaves into the empty tree is the build (about n x height
 * permutations).  pos / op / values live in the tree's memory space (values required for n > 0); n < 2^31.
 *   HOST: a position >= arity^height or an op other than 0/1 is P252_ERR_INVALID_ARGUMENT and nothing is modified; so is a
 *   batch that would leave more than max_leaves present positions.  HOST trees are staged to the device and copied back.
 *   DEVICE: an invalid item is skipped on the device and counted into *n_rejected (optional HOST pointer, 0 for HOST
 *   calls; lifetime as for p252_mtree_update).  A batch that would leave more than max_leaves present positions is
 *   refused on the device without a host synchronisation: the tree is unchanged and *n_rejected = n.
 * After a CUDA failure the tree's contents are unspecified. */
int p252_ctree_update(p252_ctx* ctx, p252_ctree* tree, const uint64_t* pos, const uint8_t* op, const p252_fr* values,
                      size_t n, size_t* n_rejected, int flags);
/* Openings of positions pos[0..n) in the format of p252_mtree_open_batch (n x height x arity, absent slots 0); they
 * verify with p252_merkle_verify_batch, depth = height.  An absent position is P252_ERR_INVALID_ARGUMENT for HOST
 * buffers and an all-zero opening for DEVICE buffers. */
int p252_ctree_open_batch(p252_ctx* ctx, const p252_ctree* tree, const uint64_t* pos, size_t n, p252_fr* paths_out,
                          int flags);

/* ---- multi-GPU tree build: one process per GPU, one NCCL all-gather per level ---------------- */
#define P252_NCCL_UNIQUE_ID_BYTES 128
/* rank 0 creates the id and ships it to the other ranks by any means (torch.distributed / MPI) */
int p252_dist_unique_id(uint8_t id[P252_NCCL_UNIQUE_ID_BYTES]);
int p252_dist_init(p252_ctx* ctx, const uint8_t id[P252_NCCL_UNIQUE_ID_BYTES], int rank, int nranks);
int p252_dist_finalize(p252_ctx* ctx);
/* The partition p252_merkle4_build_dist follows (pure host arithmetic, no GPU needed): for every internal
 * level, bottom-up, where it lives in nodes_out, which slice this rank computes, and whether the level is
 * all-gathered (sharded = 1) or computed redundantly by every rank (levels with fewer nodes than ranks). */
typedef struct p252_level_plan {
    uint64_t level_offset; /* first node of the level inside nodes_out            */
    uint64_t level_size;   /* nodes in the level                                   */
    uint64_t my_offset;    /* first node (within the level) this rank computes     */
    uint64_t my_count;     /* how many it computes                                 */
    int32_t sharded;       /* 1: slices + all-gather; 0: every rank computes all   */
    int32_t reserved;
} p252_level_plan;
int p252_merkle4_shard_plan(size_t n_leaves_total, int nranks, int rank, p252_level_plan* levels, int capacity,
                            int* n_levels);
/* leaves_shard: this rank's contiguous n_leaves_total/nranks leaves (DEVICE or HOST per flags).
 * Every level's output is sharded contiguously across ranks, computed, then all-gathered so that
 * each rank ends with the complete level (levels smaller than nranks are computed redundantly).
 * nodes_out (same space as leaves_shard): all internal levels as in p252_merkle4_build. */
int p252_merkle4_build_dist(p252_ctx* ctx, const p252_fr* leaves_shard, size_t n_leaves_total, p252_fr* nodes_out,
                            int flags);
/* Per-level device times of the last p252_merkle4_build_dist(... | P252_TIMING) on this context (synchronises
 * the context first): kernel_ms on the compute stream, gather_ms / gather_bytes of that level's all-gather on the
 * communication stream (0 for levels computed redundantly), and total_ms from the first kernel to the last event. */
typedef struct p252_level_timing {
    uint64_t nodes;        /* nodes of the level                      */
    uint64_t my_nodes;     /* nodes this rank hashed                  */
    uint64_t gather_bytes; /* bytes this rank received + kept (level) */
    float kernel_ms;
    float gather_ms;
} p252_level_timing;
int p252_tree_level_timings(p252_ctx* ctx, p252_level_timing* levels, int capacity, int* n_levels, float* total_ms);

#ifdef __cplusplus
}
#endif
#endif /* POSEIDON252_B200_H */
