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
// Merkle openings over the leaves + bottom-up internal-level layout of p252_merkle_build (arity 2 or 4)
cudaError_t launch_merkle_open(const void* leaves, const void* nodes, const uint64_t* leaf_idx, size_t n, int arity,
                               uint32_t depth, uint64_t n_leaves, void* paths, cudaStream_t st);
cudaError_t launch_merkle_verify(const uint64_t tag[4], const uint64_t root[4], const void* leaf_items,
                                 const uint64_t* leaf_idx, const void* paths, size_t n, int arity, uint32_t depth,
                                 uint8_t* ok, unsigned long long* n_failed, cudaStream_t st);
void kernel_launch_shape(int* threads_per_block, int* min_blocks_per_sm);
size_t coop_max_items(int sm_count);   // default small-batch threshold (P252_COOP_MAX or derived from the SM count)
// 32x32->64-bit multiply instructions (IMAD.WIDE / IMAD.HI class) and DFMA per Hades permutation, counted from
// the generated PTX (fr_ptx.cuh) and the round structure of hades_permute()
uint32_t wide_mul_per_permutation();
uint32_t dfma_per_permutation();

}  // namespace p252
