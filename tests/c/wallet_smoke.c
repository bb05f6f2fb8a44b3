/* Plain-C consumer of the wallet scan: calls EXACTLY the function of the `extern "C"` block of
 * bindings/rust/src/wallet.rs, plus functions from the first block of lib.rs (tests/test_wallet_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                 -> prints WALLET_SMOKE_NO_DEVICE
 *   with an H100  : two keys, one of them bad (a = r_J), scan three notes that neither owns, one with R off the curve:
 *                   every owner is -1, every row and total zero, one invalid note and one bad key counted; n_keys = 0
 *                   and an off-curve G' (also for n == 0) are refused with nothing written
 *                                                                                     -> prints WALLET_SMOKE_OK   */
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

/* a generator of the prime-order subgroup (u, v = 18), Montgomery limbs */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("WALLET_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 3, K = 2 };
    static p252_jscalar a[K], b[K], blinder[N], zs;
    static p252_fr R[2 * N], pk[2 * N], C[2 * N], nonce[N], cipher[3 * N], nul[N], zf;
    uint64_t pos[N] = {0, 1, 2}, value[N], totals[4 * K];
    int32_t owner[N];
    uint8_t opened[N];
    size_t bad = 9, inval = 9;
    a[0].l[0] = 1, b[0].l[0] = 1;
    a[1].l[0] = 0xd0970e5ed6f72cb7ULL, a[1].l[1] = 0xa6682093ccc81082ULL;   /* a = r_J: a bad key */
    a[1].l[2] = 0x06673b0101343b00ULL, a[1].l[3] = 0x0e7db4ea6533afa9ULL;
    for (int i = 0; i < N; ++i) R[2 * i] = G[0], R[2 * i + 1] = G[1], pk[2 * i] = G[0], pk[2 * i + 1] = G[1];
    R[5].l[0] ^= 1;                                                       /* note 2: R off the curve */
    memset(value, 0xA5, sizeof value);
    memset(totals, 0xA5, sizeof totals);
    CHECK(p252_wallet_scan_batch(ctx, a, b, K, R, pk, pos, nonce, cipher, C, N, G, G, owner, nul, value, blinder, opened, totals,
                                 &inval, &bad, P252_MEM_HOST));
    if (inval != 1 || bad != 1) return 2;
    for (int i = 0; i < N; ++i)
        if (owner[i] != -1 || opened[i] || value[i] || memcmp(&nul[i], &zf, sizeof zf) || memcmp(&blinder[i], &zs, sizeof zs))
            return 3;
    for (int j = 0; j < 4 * K; ++j)
        if (totals[j]) return 4;
    /* refused calls write nothing: n_keys = 0, an off-curve G' (also for n == 0) */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    owner[0] = 77;
    bad = 9;
    if (p252_wallet_scan_batch(ctx, a, b, 0, R, pk, pos, nonce, cipher, C, N, G, G, owner, nul, value, blinder, opened, totals,
                               &inval, &bad, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT ||
        p252_wallet_scan_batch(ctx, a, b, K, R, pk, pos, nonce, cipher, C, 0, G, off, owner, nul, value, blinder, opened, totals,
                               &inval, &bad, P252_MEM_HOST) != P252_ERR_INVALID_POINT)
        return 5;
    if (owner[0] != 77 || bad != 9) return 6;
    p252_destroy(ctx);
    printf("WALLET_SMOKE_OK\n");
    return 0;
}
