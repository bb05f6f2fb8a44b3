/* Plain-C consumer of the Schnorr signatures: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/schnorr.rs, plus functions from the first block of lib.rs (tests/test_schnorr_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                  -> prints SCHNORR_SMOKE_NO_DEVICE
 *   with an H100  : the public key PK = [sk] G comes from a signing call itself (sk = 0 makes u = r and R = [r] G);
 *                   signatures by sk verify under PK and not under another key or for another message, an r >= r_J is
 *                   zeroed and counted, its zeroed signature is not verified, and an off-curve G is refused with
 *                   nothing written                                                   -> prints SCHNORR_SMOKE_OK   */
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
        printf("SCHNORR_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 7 };
    static p252_jscalar zero_sk[1], keys[2], key_u[2], r[N], u[N];
    static p252_fr key_pk[4], msg[N], R[2 * N], zero_msg[2];
    uint8_t ok[N], verified[N];
    size_t bad = 9, good = 9;
    keys[0].l[0] = 0x1234567890abcdefULL, keys[0].l[1] = 42, keys[0].l[3] = 0x0e7db4ea6533afa8ULL;   /* sk < r_J */
    keys[1].l[0] = 0xfeedfacecafebeefULL, keys[1].l[2] = 7;                                         /* another key */
    for (int i = 0; i < N; ++i) {
        r[i].l[0] = 1000u + (uint64_t)i, r[i].l[2] = (uint64_t)i << 40;
        msg[i].l[0] = 77u * (uint64_t)i + 5u, msg[i].l[3] = (uint64_t)i;
    }
    r[3].l[3] = 0x0e7db4ea6533afaaULL;                          /* item 3: r >= r_J */
    /* PK = [sk] G for both keys: the R rows of a signing call with sk = 0 and r = the keys */
    CHECK(p252_schnorr_sign_batch(ctx, zero_sk, 1, keys, zero_msg, 2, G, key_u, key_pk, ok, &bad, P252_MEM_HOST));
    if (!ok[0] || !ok[1] || bad != 0 || memcmp(&key_u[0], &keys[0], sizeof keys[0])) return 2;
    CHECK(p252_schnorr_sign_batch(ctx, keys, 1, r, msg, N, G, u, R, ok, &bad, P252_MEM_HOST));
    if (bad != 1) return 3;
    for (int i = 0; i < N; ++i) {
        static const p252_fr zero[2];
        static const p252_jscalar zs;
        const int zeroed = memcmp(R + 2 * i, zero, sizeof zero) == 0 && memcmp(&u[i], &zs, sizeof zs) == 0;
        if (ok[i] != (i == 3 ? 0 : 1) || (i == 3) != zeroed) return 4;
    }
    CHECK(p252_schnorr_verify_batch(ctx, key_pk, 1, u, R, msg, N, G, verified, &good, &bad, P252_MEM_HOST));
    if (good != N - 1 || bad != 0) return 5;   /* the zeroed signature 3: R = (0, 0) is canonical, not verified */
    for (int i = 0; i < N; ++i)
        if (verified[i] != (i == 3 ? 0 : 1)) return 6;
    CHECK(p252_schnorr_verify_batch(ctx, key_pk + 2, 1, u, R, msg, N, G, verified, &good, &bad, P252_MEM_HOST));
    if (good != 0 || bad != 0) return 7;
    msg[0].l[0] ^= 1;                                           /* another message */
    CHECK(p252_schnorr_verify_batch(ctx, key_pk, 1, u, R, msg, 1, G, verified, &good, NULL, P252_MEM_HOST));
    if (good != 0 || verified[0] != 0) return 8;
    /* batch checks: an off-curve G writes nothing */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    memset(verified, 0xA5, sizeof verified);
    good = 9;
    if (p252_schnorr_verify_batch(ctx, key_pk, 1, u, R, msg, N, off, verified, &good, NULL, P252_MEM_HOST) !=
        P252_ERR_INVALID_POINT)
        return 9;
    if (verified[0] != 0xA5 || good != 9) return 10;
    if (p252_schnorr_sign_batch(ctx, keys, 2, r, msg, N, G, u, R, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 11;
    p252_destroy(ctx);
    printf("SCHNORR_SMOKE_OK\n");
    return 0;
}
