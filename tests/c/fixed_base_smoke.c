/* Plain-C consumer of the fixed-base scalar multiplication: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/fixed_base.rs, plus functions from the first block of lib.rs (tests/test_fixed_base_cpu.py asserts
 * both).
 *   without a GPU : p252_create fails                                                 -> prints FIXED_BASE_SMOKE_NO_DEVICE
 *   with an H100  : pk = [a] G, the sender's fused call makes R_i = [r_i] G and the ciphers to pk, R_i equals the
 *                   fixed-base batch, an r >= r_J is zeroed and counted, and an off-curve base is refused with nothing
 *                   written                                                           -> prints FIXED_BASE_SMOKE_OK   */
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

/* the generator used by the tests (u, v = 18), Montgomery limbs */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("FIXED_BASE_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 6, L = 2 };
    static p252_jscalar a[1], r[N];
    static p252_fr pk[2], R[2 * N], R2[2 * N], msg[N * L], cipher[N * (L + 1)], nonce[N];
    uint8_t ok[N];
    size_t bad = 9;
    a[0].l[0] = 0x1234567890abcdefULL, a[0].l[1] = 42, a[0].l[3] = 0x0e7db4ea6533afa8ULL;    /* < r_J */
    for (int i = 0; i < N; ++i) {
        r[i].l[0] = 1000u + (uint64_t)i, r[i].l[2] = (uint64_t)i << 40;
        nonce[i].l[0] = 77u + (uint64_t)i;
        for (int k = 0; k < L; ++k) msg[i * L + k].l[0] = 100u * (uint64_t)i + (uint64_t)k, msg[i * L + k].l[1] = 5;
    }
    r[3].l[3] = 0x0e7db4ea6533afaaULL;                          /* item 3: r >= r_J */
    CHECK(p252_fixed_base_batch(ctx, G, a, 1, pk, ok, &bad, P252_MEM_HOST));
    if (!ok[0] || bad != 0) return 2;
    CHECK(p252_fixed_base_batch(ctx, G, r, N, R, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || ok[3]) return 3;
    CHECK(p252_encrypt_batch_ephemeral(ctx, msg, N, L, r, G, pk, 1, nonce, cipher, R2, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || memcmp(R, R2, sizeof R)) return 4;
    for (int i = 0; i < N; ++i) {
        if (ok[i] != (i == 3 ? 0 : 1)) return 5;
        static const p252_fr zero[L + 1];
        if ((i == 3) != (memcmp(cipher + i * (L + 1), zero, sizeof zero) == 0)) return 6;
    }
    /* batch checks: an off-curve base writes nothing */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    memset(R2, 0xA5, sizeof R2);
    if (p252_fixed_base_batch(ctx, off, r, N, R2, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_POINT) return 7;
    if (R2[0].l[0] != 0xA5A5A5A5A5A5A5A5ULL) return 8;
    if (p252_encrypt_batch_ephemeral(ctx, msg, N, 0, r, G, pk, 1, nonce, cipher, R2, ok, NULL, P252_MEM_HOST) !=
        P252_ERR_INVALID_IO_PATTERN)
        return 9;
    p252_destroy(ctx);
    printf("FIXED_BASE_SMOKE_OK\n");
    return 0;
}
