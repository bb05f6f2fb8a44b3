/* Plain-C consumer of the double-key Schnorr signatures: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/schnorr_double.rs, plus functions from the first block of lib.rs (tests/test_schnorr_double_cpu.py
 * asserts both).
 *   without a GPU : p252_create fails                                                  -> prints SCHNORR_DOUBLE_SMOKE_NO_DEVICE
 *   with an H100  : G' = -G, so R' = [r] G' = -R and the note key pair is (PK, PK') = (-pk', pk') with pk' from the
 *                   note signer.  The note signatures verify under that pair, a tampered u does not, an a >= r_J is
 *                   zeroed and counted, sk = 0 signs with u = r, an off-curve G' is refused with nothing written, and
 *                   n_secret not 1 or n is refused                                     -> prints SCHNORR_DOUBLE_SMOKE_OK   */
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

/* a generator of the prime-order subgroup (u, v = 18), Montgomery limbs, and the field modulus p */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const uint64_t PM[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};

/* -x mod p on Montgomery limbs (the Montgomery image of -x) */
static p252_fr neg(p252_fr x) {
    p252_fr r;
    uint64_t borrow = 0, any = x.l[0] | x.l[1] | x.l[2] | x.l[3];
    for (int k = 0; k < 4; ++k) {
        const uint64_t d = PM[k] - x.l[k] - borrow;
        borrow = (PM[k] < x.l[k]) || (PM[k] - x.l[k] < borrow);
        r.l[k] = any ? d : 0;
    }
    return r;
}

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("SCHNORR_DOUBLE_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 3 };
    p252_fr Gp[2];
    Gp[0] = neg(G[0]), Gp[1] = G[1];
    static p252_fr note_R[2 * N], msg[N], R[2 * N], Rp[2 * N], pkp[2 * N], PK[2 * N], zero;
    static p252_jscalar a[N], b[N], r[N], u[N];
    uint8_t ok[N], ver[N];
    size_t bad = 9, nver = 9;
    for (int i = 0; i < N; ++i) {
        note_R[2 * i] = G[0], note_R[2 * i + 1] = G[1];
        a[i].l[0] = 0x1234567890abcdefULL + (uint64_t)i, a[i].l[2] = 77;
        b[i].l[0] = 0xfedcba9876543210ULL, b[i].l[1] = (uint64_t)i;
        r[i].l[0] = 1000 + (uint64_t)i, r[i].l[3] = 0x0123456789abcdefULL;
        msg[i].l[0] = (uint64_t)i;
    }
    a[2].l[3] = 0x0e7db4ea6533afaaULL;                              /* item 2: a >= r_J */
    CHECK(p252_note_sign_double_batch(ctx, a, b, N, note_R, r, msg, N, G, Gp, u, R, Rp, pkp, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || !ok[0] || !ok[1] || ok[2]) return 2;
    static const p252_jscalar zs;
    if (memcmp(&u[2], &zs, sizeof zs)) return 3;
    for (int k = 4; k < 6; ++k)                                     /* item 2's rows are zeroed */
        if (memcmp(&R[k], &zero, sizeof zero) || memcmp(&Rp[k], &zero, sizeof zero) || memcmp(&pkp[k], &zero, sizeof zero))
            return 3;
    for (int i = 0; i < 2; ++i) {                                   /* R' = [r] (-G) = -R */
        const p252_fr nu = neg(R[2 * i]);
        if (memcmp(&Rp[2 * i], &nu, sizeof nu) || memcmp(&Rp[2 * i + 1], &R[2 * i + 1], sizeof nu)) return 4;
        PK[2 * i] = neg(pkp[2 * i]), PK[2 * i + 1] = pkp[2 * i + 1];  /* [note_sk] G = -[note_sk] G' */
    }
    CHECK(p252_schnorr_verify_double_batch(ctx, PK, pkp, 2, u, R, Rp, msg, 2, G, Gp, ver, &nver, &bad, P252_MEM_HOST));
    if (nver != 2 || bad != 0 || !ver[0] || !ver[1]) return 5;
    u[0].l[0] ^= 1;                                                 /* a tampered u */
    CHECK(p252_schnorr_verify_double_batch(ctx, PK, pkp, 2, u, R, Rp, msg, 2, G, Gp, ver, &nver, &bad, P252_MEM_HOST));
    if (nver != 1 || bad != 0 || ver[0] || !ver[1]) return 6;
    /* sk = 0 for the batch (n_secret = 1): u = r, and it verifies under the identity pair */
    static p252_jscalar sk0;
    CHECK(p252_schnorr_sign_double_batch(ctx, &sk0, 1, r, msg, N, G, Gp, u, R, Rp, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || memcmp(u, r, sizeof u)) return 7;
    /* batch checks: an off-curve G' writes nothing, also for n == 0; n_secret must be 1 or n */
    p252_fr off[2];
    memcpy(off, Gp, sizeof off);
    off[1].l[0] ^= 1;
    memset(ok, 0xA5, sizeof ok);
    bad = 9;
    if (p252_schnorr_sign_double_batch(ctx, &sk0, 1, r, msg, N, G, off, u, R, Rp, ok, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT ||
        p252_note_sign_double_batch(ctx, a, b, 1, note_R, r, msg, 0, G, off, u, R, Rp, pkp, ok, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT)
        return 8;
    if (ok[0] != 0xA5 || bad != 9) return 9;
    if (p252_schnorr_sign_double_batch(ctx, a, 2, r, msg, N, G, Gp, u, R, Rp, ok, NULL, P252_MEM_HOST) !=
        P252_ERR_INVALID_ARGUMENT)
        return 10;
    p252_destroy(ctx);
    printf("SCHNORR_DOUBLE_SMOKE_OK\n");
    return 0;
}
