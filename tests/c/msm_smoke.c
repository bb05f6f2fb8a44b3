/* Plain-C consumer of the multi-scalar multiplication and all-or-nothing verification: calls EXACTLY the functions of the
 * `extern "C"` block of bindings/rust/src/msm.rs, plus functions from the first block of lib.rs (tests/test_msm_cpu.py
 * asserts both).
 *   without a GPU : p252_create fails                                                      -> prints MSM_SMOKE_NO_DEVICE
 *   with an H100  : [a] G + [b] G == [a + b] G, [s] P + [s] (-P) is the identity (0, 1), n == 0 gives the identity, a
 *                   scalar >= r_J is skipped and counted; signatures under the identity key PK = (0, 1) (sk = 0, so
 *                   u = r and R = [r] G for any challenge) pass verify_all, a changed u fails it, a u >= r_J is counted
 *                   and fails it, n == 0 passes, and an off-curve G is refused with nothing written -> prints MSM_SMOKE_OK */
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
/* the identity (0, 1): 1 in Montgomery form */
static const p252_fr IDENT[2] = {{{0, 0, 0, 0}},
                                 {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}}};
static const uint64_t P[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
static const p252_jscalar R_J = {{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};

/* x = p - x for 0 < x < p (the negation of a Montgomery image) */
static void negate(p252_fr* x) {
    unsigned borrow = 0;
    for (int k = 0; k < 4; ++k) {
        const uint64_t a = P[k], b = x->l[k];
        const uint64_t d = a - b - borrow;
        borrow = (a < b) || (a - b < borrow);
        x->l[k] = d;
    }
}

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("MSM_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 6 };
    static p252_jscalar s[N], u[N], w[N];
    static p252_fr pts[2 * N], R[2 * N], msg[N], out[2], want[2];
    size_t bad = 9;
    /* [a] G + [b] G == [a + b] G */
    s[0].l[0] = 0x1234567890abcdefULL, s[0].l[2] = 5;
    s[1].l[0] = 0x0000000011111111ULL, s[1].l[1] = 3;
    memcpy(pts, G, sizeof G);
    memcpy(pts + 2, G, sizeof G);
    CHECK(p252_jubjub_msm(ctx, s, pts, 2, out, &bad, P252_MEM_HOST));
    if (bad != 0) return 2;
    p252_jscalar ab = {{s[0].l[0] + s[1].l[0], s[0].l[1] + s[1].l[1], s[0].l[2], 0}};   /* no carries */
    CHECK(p252_jubjub_msm(ctx, &ab, G, 1, want, NULL, P252_MEM_HOST));
    if (memcmp(out, want, sizeof out)) return 3;
    /* [s] P + [s] (-P) == identity, with P = out */
    memcpy(pts, out, sizeof out);
    memcpy(pts + 2, out, sizeof out);
    negate(&pts[2]);
    s[1] = s[0];
    CHECK(p252_jubjub_msm(ctx, s, pts, 2, out, NULL, P252_MEM_HOST));
    if (memcmp(out, IDENT, sizeof out)) return 4;
    CHECK(p252_jubjub_msm(ctx, NULL, NULL, 0, out, &bad, P252_MEM_HOST));
    if (memcmp(out, IDENT, sizeof out) || bad != 0) return 5;
    /* a scalar >= r_J is skipped and counted */
    s[1] = R_J;
    memcpy(pts + 2, G, sizeof G);
    CHECK(p252_jubjub_msm(ctx, s, pts, 2, out, &bad, P252_MEM_HOST));
    CHECK(p252_jubjub_msm(ctx, s, pts, 1, want, NULL, P252_MEM_HOST));
    if (bad != 1 || memcmp(out, want, sizeof out)) return 6;
    /* signatures of sk = 0 under PK = (0, 1): u = r, R = [r] G */
    for (int i = 0; i < N; ++i) {
        u[i].l[0] = 1000u + 17u * (uint64_t)i, u[i].l[2] = (uint64_t)i << 30;
        w[i].l[0] = 0x9e3779b97f4a7c15ULL * (uint64_t)(i + 1), w[i].l[1] = 0x632be59bd9b4e019ULL + (uint64_t)i;
        msg[i].l[0] = 77u * (uint64_t)i + 5u;
        CHECK(p252_jubjub_msm(ctx, &u[i], G, 1, R + 2 * i, NULL, P252_MEM_HOST));
    }
    uint8_t all = 9;
    CHECK(p252_schnorr_verify_all(ctx, IDENT, 1, u, R, msg, w, N, G, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 7;
    u[4].l[0] ^= 1;                                             /* a changed u */
    CHECK(p252_schnorr_verify_all(ctx, IDENT, 1, u, R, msg, w, N, G, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 0) return 8;
    u[4] = R_J;                                                 /* an invalid item */
    CHECK(p252_schnorr_verify_all(ctx, IDENT, 1, u, R, msg, w, N, G, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 1) return 9;
    all = 9;
    CHECK(p252_schnorr_verify_all(ctx, IDENT, 1, NULL, NULL, NULL, NULL, 0, G, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 10;
    /* batch checks: an off-curve G writes nothing; a NULL answer is refused */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    all = 9;
    if (p252_schnorr_verify_all(ctx, IDENT, 1, u, R, msg, w, N, off, &all, NULL, P252_MEM_HOST) != P252_ERR_INVALID_POINT)
        return 11;
    if (all != 9) return 12;
    if (p252_schnorr_verify_all(ctx, IDENT, 1, u, R, msg, w, N, G, NULL, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 13;
    p252_destroy(ctx);
    printf("MSM_SMOKE_OK\n");
    return 0;
}
