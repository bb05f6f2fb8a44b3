/* Plain-C consumer of the JubJub key exchange: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/dhke.rs, plus functions from the first block of lib.rs (tests/test_jubjub_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                       -> prints DHKE_SMOKE_NO_DEVICE
 *   with an H100  : a sender derives R_i = [r_i] G and encrypts to pk = [a] G with the fused call, the receiver decrypts
 *                   with the view key a in the (1, n) shape, [a] R_i == [r_i] pk, a tampered cipher and an off-curve
 *                   key fail alone                                                          -> prints DHKE_SMOKE_OK   */
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
        printf("DHKE_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 6, L = 3 };
    static p252_jscalar a[1], r[N];
    static p252_fr pk[2], R[2 * N], s1[2 * N], s2[2 * N], msg[N * L], cipher[N * (L + 1)], back[N * L], nonce[N];
    uint8_t ok[N];
    size_t bad = 9;
    a[0].l[0] = 0x1234567890abcdefULL, a[0].l[1] = 42, a[0].l[3] = 0x0e7db4ea6533afa8ULL;    /* < r_J */
    for (int i = 0; i < N; ++i) {
        r[i].l[0] = 1000u + (uint64_t)i, r[i].l[2] = (uint64_t)i << 40;
        nonce[i].l[0] = 77u + (uint64_t)i;
        for (int k = 0; k < L; ++k) msg[i * L + k].l[0] = 100u * (uint64_t)i + (uint64_t)k, msg[i * L + k].l[1] = 5;
    }
    /* pk = [a] G, R_i = [r_i] G (the (n, 1) shape) */
    CHECK(p252_dhke_batch(ctx, a, 1, G, 1, 1, pk, ok, &bad, P252_MEM_HOST));
    if (!ok[0] || bad != 0) return 2;
    CHECK(p252_dhke_batch(ctx, r, N, G, 1, N, R, ok, &bad, P252_MEM_HOST));
    /* [a] R_i == [r_i] pk */
    CHECK(p252_dhke_batch(ctx, a, 1, R, N, N, s1, ok, &bad, P252_MEM_HOST));
    CHECK(p252_dhke_batch(ctx, r, N, pk, 1, N, s2, ok, &bad, P252_MEM_HOST));
    if (memcmp(s1, s2, sizeof s1) || bad != 0) return 3;
    /* sender: fused encrypt to pk; receiver: fused decrypt with the view key in the (1, n) shape */
    CHECK(p252_encrypt_batch_dhke(ctx, msg, N, L, r, N, pk, 1, nonce, cipher, ok, &bad, P252_MEM_HOST));
    for (int i = 0; i < N; ++i)
        if (!ok[i]) return 4;
    cipher[2 * (L + 1) + L].l[1] ^= 1;                          /* item 2's authentication scalar */
    R[2 * 4].l[0] ^= 1;                                         /* item 4's key is no longer on the curve */
    CHECK(p252_decrypt_batch_dhke(ctx, cipher, N, L, a, 1, R, N, nonce, back, ok, &bad, P252_MEM_HOST));
    for (int i = 0; i < N; ++i) {
        const int fail = i == 2 || i == 4;
        if (ok[i] != (fail ? 0 : 1)) return 5;
        if (!fail && memcmp(back + i * L, msg + i * L, L * sizeof(p252_fr))) return 6;
    }
    if (bad != 2) return 7;
    /* batch checks */
    if (p252_dhke_batch(ctx, r, 2, G, 1, N, s1, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 8;
    if (p252_decrypt_batch_dhke(ctx, cipher, N, 0, a, 1, R, N, nonce, back, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_IO_PATTERN)
        return 9;
    p252_destroy(ctx);
    printf("DHKE_SMOKE_OK\n");
    return 0;
}
