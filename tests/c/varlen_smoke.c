/* Plain-C consumer of the variable-length digest batch: calls EXACTLY the function of the third `extern "C"` block of
 * bindings/rust/src/lib.rs, plus context handling from the first block (tests/test_varlen_bindings.py asserts both).
 *   without a GPU : p252_create fails                                               -> prints VARLEN_SMOKE_NO_DEVICE
 *   with an H100  : a ragged batch on host buffers equals per-length p252_hash_batch; a Merkle4 batch with one item of
 *                   the wrong length is refused and leaves out untouched            -> prints VARLEN_SMOKE_OK   */
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
        printf("VARLEN_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    /* five items of lengths 1, 4, 5, 9, 2 (a slice of a CSR array whose first offset is 3), two output scalars */
    static p252_fr data[3 + 21], out[5 * 2], want[2];
    const uint64_t offsets[6] = {3, 4, 8, 13, 22, 24};
    for (int i = 0; i < 24; ++i) data[i].l[0] = 1000u + (uint64_t)i, data[i].l[1] = (uint64_t)i;
    size_t rejected = 7;
    CHECK(p252_hash_batch_varlen(ctx, P252_DOMAIN_OTHER, data, 24, offsets, 5, 9, out, 2, &rejected, P252_MEM_HOST));
    if (rejected != 0) return 2;
    for (int i = 0; i < 5; ++i) {
        CHECK(p252_hash_batch(ctx, P252_DOMAIN_OTHER, data + offsets[i], 1, offsets[i + 1] - offsets[i], want, 2, P252_MEM_HOST));
        if (memcmp(want, out + 2 * i, sizeof want)) return 3;
    }
    /* Merkle4: items 0 and 2 have four children, item 1 has three -> IOPatternViolation, nothing written */
    const uint64_t moff[4] = {0, 4, 7, 11};
    memset(out, 0xab, sizeof out);
    if (p252_hash_batch_varlen(ctx, P252_DOMAIN_MERKLE4, data, 11, moff, 3, 4, out, 1, NULL, P252_MEM_HOST) !=
        P252_ERR_IO_PATTERN_VIOLATION)
        return 4;
    for (size_t b = 0; b < sizeof out; ++b)
        if (((const unsigned char*)out)[b] != 0xab) return 5;
    p252_destroy(ctx);
    printf("VARLEN_SMOKE_OK\n");
    return 0;
}
