/* Plain-C consumer of the variable-length encrypt / decrypt batches: calls EXACTLY the functions of the `extern "C"` block
 * of bindings/rust/src/crypt_varlen.rs, plus functions from the first block of lib.rs (tests/test_crypt_varlen_bindings.py
 * asserts both).
 *   without a GPU : p252_create fails                                                   -> prints CRYPT_VARLEN_SMOKE_NO_DEVICE
 *   with an H100  : a ragged batch on host buffers equals per-item p252_encrypt_batch, decrypts back with every ok set,
 *                   a tampered cipher fails alone, and an empty message is refused with out untouched
 *                                                                                       -> prints CRYPT_VARLEN_SMOKE_OK   */
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
        printf("CRYPT_VARLEN_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    /* five messages of lengths 1, 4, 5, 9, 2 (a slice of a CSR array whose first offset is 3) */
    enum { N = 5, NS = 24, NC = 21 + N };
    static p252_fr data[NS], uv[2 * N], nonce[N], cipher[NC], msg[21], want[10];
    const uint64_t offsets[N + 1] = {3, 4, 8, 13, 22, 24};
    uint64_t coff[N + 1];
    uint8_t ok[N];
    for (int i = 0; i < NS; ++i) data[i].l[0] = 1000u + (uint64_t)i, data[i].l[1] = (uint64_t)i;
    for (int i = 0; i < N; ++i) {
        uv[2 * i].l[0] = 7u + (uint64_t)i, uv[2 * i + 1].l[0] = 70u + (uint64_t)i, nonce[i].l[0] = 700u + (uint64_t)i;
        coff[i] = offsets[i] - offsets[0] + (uint64_t)i;
    }
    coff[N] = offsets[N] - offsets[0] + N;
    size_t rejected = 7, failed = 7;
    CHECK(p252_encrypt_batch_varlen(ctx, data, NS, offsets, N, 9, uv, nonce, cipher, &rejected, P252_MEM_HOST));
    if (rejected != 0) return 2;
    for (int i = 0; i < N; ++i) {
        const size_t L = offsets[i + 1] - offsets[i];
        CHECK(p252_encrypt_batch(ctx, data + offsets[i], 1, L, uv + 2 * i, nonce + i, want, P252_MEM_HOST));
        if (memcmp(want, cipher + coff[i], (L + 1) * sizeof(p252_fr))) return 3;
    }
    /* the cipher CSR decrypts straight back; then item 3's authentication scalar is tampered with */
    for (int round = 0; round < 2; ++round) {
        CHECK(p252_decrypt_batch_varlen(ctx, cipher, NC, coff, N, 9, uv, nonce, msg, ok, &failed, &rejected, P252_MEM_HOST));
        for (int i = 0; i < N; ++i) {
            const size_t L = offsets[i + 1] - offsets[i];
            const int bad = round == 1 && i == 3;
            if (ok[i] != (bad ? 0 : 1)) return 4;
            if (!bad && memcmp(msg + (offsets[i] - offsets[0]), data + offsets[i], L * sizeof(p252_fr))) return 5;
        }
        if (failed != (size_t)round || rejected != 0) return 6;
        cipher[coff[4] - 1].l[2] ^= 1;                       /* the last scalar of cipher 3 */
    }
    /* an empty message: InvalidIOPattern, nothing written */
    const uint64_t bad_off[3] = {0, 2, 2};
    memset(cipher, 0xab, sizeof cipher);
    if (p252_encrypt_batch_varlen(ctx, data, NS, bad_off, 2, 9, uv, nonce, cipher, NULL, P252_MEM_HOST) !=
        P252_ERR_INVALID_IO_PATTERN)
        return 7;
    for (size_t b = 0; b < sizeof cipher; ++b)
        if (((const unsigned char*)cipher)[b] != 0xab) return 8;
    p252_destroy(ctx);
    printf("CRYPT_VARLEN_SMOKE_OK\n");
    return 0;
}
