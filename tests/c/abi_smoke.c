/* Plain-C consumer of include/poseidon252_b200.h that calls EXACTLY the entry points the Rust crate binds
 * (the `extern "C"` block of bindings/rust/src/lib.rs; tests/test_abi.py asserts the two lists are identical).
 * The Rust source cannot be compiled in this image, so this program is the mechanical check that the signatures
 * the binding assumes link and behave: compiled as C (not C++) against the header, linked with the library.
 *   without a GPU : p252_create must fail with P252_ERR_NO_DEVICE (no CPU fallback)       -> prints ABI_SMOKE_NO_DEVICE
 *   with an H100  : every call runs on small host buffers and the results are cross-checked -> prints ABI_SMOKE_OK   */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/poseidon252_b200.h"

#define CHECK(call)                                                                 \
    do {                                                                            \
        int rc__ = (call);                                                          \
        if (rc__ != P252_OK) {                                                      \
            fprintf(stderr, "%s -> %d (%s)\n", #call, rc__, p252_strerror(rc__));   \
            return 1;                                                               \
        }                                                                           \
    } while (0)

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("ABI_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        /* the host-only entry point of the set still works */
        size_t ni = 0;
        int lv = 0;
        if (p252_merkle_tree_nodes(4, 64, &ni, &lv) != P252_OK || ni != 21 || lv != 3) return 1;
        return 0;
    }
    if (rc != P252_OK) {
        fprintf(stderr, "p252_create -> %d (%s)\n", rc, p252_strerror(rc));
        return 1;
    }
    enum { N = 64, L = 2 };
    static p252_fr leaves[N], states[N / 4 * 5], digest[N / 4], trunc[N / 4], msg[N * L], uv[N * 2], nonce[N], cipher[N * (L + 1)],
        back[N * L], nodes[21], paths[8 * 3 * 4];
    static uint8_t ok[N];
    for (int i = 0; i < N; ++i) {                      /* small canonical values are valid BlsScalar.0 limbs (< p) */
        leaves[i].l[0] = 1000u + (uint64_t)i;
        nonce[i].l[0] = 7u * (uint64_t)i + 1;
        uv[2 * i].l[0] = (uint64_t)i + 3, uv[2 * i + 1].l[1] = (uint64_t)i + 5;
        for (int k = 0; k < L; ++k) msg[i * L + k].l[2] = (uint64_t)(i * L + k + 11);
    }
    memcpy(states, leaves, sizeof(p252_fr) * 20);
    CHECK(p252_permute_batch(ctx, states, N / 4, P252_MEM_HOST));
    CHECK(p252_hash_batch(ctx, P252_DOMAIN_MERKLE4, leaves, N / 4, 4, digest, 1, P252_MEM_HOST));
    CHECK(p252_hash_batch_truncated(ctx, P252_DOMAIN_MERKLE4, leaves, N / 4, 4, trunc, 1, P252_MEM_HOST));
    if (trunc[0].l[3] >> 58) return 2;                 /* 250-bit mask */
    CHECK(p252_encrypt_batch(ctx, msg, N, L, uv, nonce, cipher, P252_MEM_HOST));
    size_t failed = 99;
    cipher[5 * (L + 1) + L].l[0] ^= 1;                 /* tamper one authentication scalar */
    CHECK(p252_decrypt_batch(ctx, cipher, N, L, uv, nonce, back, ok, &failed, P252_MEM_HOST));
    if (failed != 1 || ok[5] != 0 || ok[6] != 1 || memcmp(&back[6 * L], &msg[6 * L], sizeof(p252_fr) * L)) return 3;
    size_t ni = 0;
    int depth = 0;
    CHECK(p252_merkle_tree_nodes(4, N, &ni, &depth));
    if (ni != 21 || depth != 3) return 4;
    CHECK(p252_merkle_build(ctx, 4, leaves, N, nodes, P252_MEM_HOST));
    if (memcmp(nodes, digest, sizeof(p252_fr) * (N / 4))) return 5;   /* level 0 of the tree = the Merkle4 digests */
    uint64_t idx[8] = {0, 1, 17, 63, 42, 5, 33, 16};
    p252_fr items[8];
    for (int i = 0; i < 8; ++i) items[i] = leaves[idx[i]];
    CHECK(p252_merkle_open_batch(ctx, 4, leaves, N, nodes, idx, 8, paths, P252_MEM_HOST));
    CHECK(p252_merkle_verify_batch(ctx, 4, depth, items, idx, paths, &nodes[20], 8, ok, &failed, P252_MEM_HOST));
    if (failed != 0) return 6;
    items[3].l[0] ^= 1;
    CHECK(p252_merkle_verify_batch(ctx, 4, depth, items, idx, paths, &nodes[20], 8, ok, &failed, P252_MEM_HOST));
    if (failed != 1 || ok[3] != 0 || ok[2] != 1) return 7;
    p252_destroy(ctx);
    printf("ABI_SMOKE_OK\n");
    return 0;
}
