/* Plain-C consumer of the mixed digest batch: calls EXACTLY the function of the `extern "C"` block of
 * bindings/rust/src/hash_mixed.rs, plus functions from the first block of lib.rs (tests/test_hash_mixed_cpu.py asserts
 * both).
 *   without a GPU : p252_create fails                                          -> prints HASH_MIXED_SMOKE_NO_DEVICE
 *   with an H100  : a Merkle4 node, a truncated Other digest of 3 scalars and an Other digest of 5 scalars with 2
 *                   outputs, in one call from a slice of larger CSR arrays (offsets[0], out_offsets[0] != 0), equal the
 *                   fixed-length p252_hash_batch / p252_hash_batch_truncated rows; an unknown mode bit and a Merkle
 *                   arity violation are refused with their statuses and nothing written
 *                                                                              -> prints HASH_MIXED_SMOKE_OK         */
#include <stdio.h>
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
        printf("HASH_MIXED_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    static p252_fr in[2 + 4 + 3 + 5];                  /* 2 scalars of another item first */
    for (size_t i = 0; i < sizeof in / sizeof in[0]; ++i)
        for (int k = 0; k < 4; ++k) in[i].l[k] = (uint64_t)(i * 4 + k + 1) * 0x9e3779b97f4a7c15ULL >> 3;   /* < p */
    const uint8_t mode[3] = {P252_DOMAIN_MERKLE4, P252_DOMAIN_OTHER | P252_MIXED_TRUNCATED, P252_DOMAIN_OTHER};
    const uint64_t offsets[4] = {2, 6, 9, 14};
    const uint64_t out_offsets[4] = {1, 2, 3, 5};
    static p252_fr out[5], want[5];
    size_t rejected = 9;
    CHECK(p252_hash_batch_mixed(ctx, mode, in, 14, offsets, 3, 5, out, 5, out_offsets, 2, &rejected, P252_MEM_HOST));
    CHECK(p252_hash_batch(ctx, P252_DOMAIN_MERKLE4, in + 2, 1, 4, want + 1, 1, P252_MEM_HOST));
    CHECK(p252_hash_batch_truncated(ctx, P252_DOMAIN_OTHER, in + 6, 1, 3, want + 2, 1, P252_MEM_HOST));
    CHECK(p252_hash_batch(ctx, P252_DOMAIN_OTHER, in + 9, 1, 5, want + 3, 2, P252_MEM_HOST));
    if (rejected != 0 || memcmp(out + 1, want + 1, 4 * sizeof(p252_fr))) return 2;
    if (want[2].l[3] >> 58) return 3;                 /* a truncated row is below 2^250 */
    static p252_fr sentinel[5];
    memset(out, 0xab, sizeof out);
    memcpy(sentinel, out, sizeof out);
    const uint8_t bad_bit[3] = {P252_DOMAIN_MERKLE4, P252_DOMAIN_OTHER | 0x04, P252_DOMAIN_OTHER};
    if (p252_hash_batch_mixed(ctx, bad_bit, in, 14, offsets, 3, 5, out, 5, out_offsets, 2, NULL, P252_MEM_HOST) !=
        P252_ERR_INVALID_ARGUMENT)
        return 4;
    const uint8_t bad_arity[3] = {P252_DOMAIN_MERKLE4, P252_DOMAIN_MERKLE2, P252_DOMAIN_OTHER};   /* Merkle2 of 3 */
    if (p252_hash_batch_mixed(ctx, bad_arity, in, 14, offsets, 3, 5, out, 5, out_offsets, 2, NULL, P252_MEM_HOST) !=
        P252_ERR_IO_PATTERN_VIOLATION)
        return 5;
    if (memcmp(out, sentinel, sizeof out)) return 6;   /* nothing written */
    p252_destroy(ctx);
    printf("HASH_MIXED_SMOKE_OK\n");
    return 0;
}
