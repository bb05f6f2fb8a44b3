/* Plain-C consumer of the batched BlsScalar::hash_to_scalar: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/hash_to_scalar.rs, plus functions from the first block of lib.rs (tests/test_hash_to_scalar_cpu.py
 * asserts both).
 *   without a GPU : p252_create fails                                          -> prints HASH_TO_SCALAR_SMOKE_NO_DEVICE
 *   with an H100  : the empty string, "abc" and a 200-byte message (two blocks) hash to their known scalars, from a
 *                   slice of a larger CSR array (offsets[0] != 0); 64 bytes of 0xff reduce to 2^512 - 1 mod p; a
 *                   decreasing offset and a max_len above P252_HASH_TO_SCALAR_MAX_LEN are refused with nothing written
 *                                                                              -> prints HASH_TO_SCALAR_SMOKE_OK     */
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

/* BlsScalar::hash_to_scalar of "", "abc" and bytes (7 i + 3) mod 256, i < 200, Montgomery limbs */
static const p252_fr WANT[3] = {
    {{0x54d4e1b7597843a5ULL, 0x8dda227ddb51e12fULL, 0x4600ae6ae56ce286ULL, 0x288d1fcd836322f9ULL}},
    {{0xeac3cf87a028522bULL, 0x8054d6ae5d6a9f49ULL, 0xf9d82ad1e858f016ULL, 0x304f42a5fc2b35a4ULL}},
    {{0x169d28fb8a9f9a01ULL, 0x87c02b152c5d0d70ULL, 0xeef94790bf83dbdcULL, 0x35a6e46568fec2ebULL}}};
/* BlsScalar::from_bytes_wide of 64 bytes of 0xff: (2^512 - 1) mod p, Montgomery limbs */
static const p252_fr WIDE_FF = {{0xc62c1805439b73b1ULL, 0xc2b9551e8ced218eULL, 0xda44ec81daf9a422ULL, 0x5605aa601c162e79ULL}};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("HASH_TO_SCALAR_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    static uint8_t bytes[5 + 3 + 200];
    memcpy(bytes, "xxxxxabc", 8);                      /* 5 bytes of another item first */
    for (int i = 0; i < 200; ++i) bytes[8 + i] = (uint8_t)(7 * i + 3);
    const uint64_t offsets[4] = {5, 5, 8, 208};
    static p252_fr out[3], wide[1];
    static const p252_fr zero[3];
    size_t rejected = 9;
    CHECK(p252_hash_to_scalar_batch(ctx, bytes, sizeof bytes, offsets, 3, 200, out, &rejected, P252_MEM_HOST));
    if (rejected != 0 || memcmp(out, WANT, sizeof WANT)) return 2;
    static uint8_t ff[64];
    memset(ff, 0xff, sizeof ff);
    CHECK(p252_scalars_from_bytes_wide(ctx, ff, 1, wide, P252_MEM_HOST));
    if (memcmp(wide, &WIDE_FF, sizeof WIDE_FF)) return 3;
    memset(out, 0, sizeof out);
    const uint64_t bad[4] = {5, 8, 6, 208};            /* item 1 decreases */
    if (p252_hash_to_scalar_batch(ctx, bytes, sizeof bytes, bad, 3, 200, out, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 4;
    if (p252_hash_to_scalar_batch(ctx, bytes, sizeof bytes, offsets, 3, P252_HASH_TO_SCALAR_MAX_LEN + 1, out, NULL,
                                  P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 5;
    if (memcmp(out, zero, sizeof zero)) return 6;      /* nothing written */
    p252_destroy(ctx);
    printf("HASH_TO_SCALAR_SMOKE_OK\n");
    return 0;
}
