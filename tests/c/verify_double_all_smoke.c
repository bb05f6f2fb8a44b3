/* Plain-C consumer of the all-or-nothing verification of double-key signatures: calls EXACTLY the function of the
 * `extern "C"` block of bindings/rust/src/verify_double_all.rs, plus functions from the first block of lib.rs
 * (tests/test_verify_double_all_cpu.py asserts both).
 *   without a GPU : p252_create fails                                            -> prints VERIFY_DOUBLE_ALL_SMOKE_NO_DEVICE
 *   with an H100  : G' = -G and the key pair (PK, PK') is the identity (0, 1) twice (sk = 0), so (u, R, R') = (1, G, G')
 *                   and (0, O, O) are signatures of every message.  They pass under one key pair and under one pair per
 *                   item; a changed u fails; a u or a weight_p >= r_J is counted and fails; R = D, R' = -D with u = 0
 *                   (the two equations off by -D and +D) passes with weight_p == weight and fails with independent
 *                   weights; an R of order 2 passes (the check is cofactored); n == 0 passes; an off-curve G' is refused
 *                   with nothing written, also for n == 0; a NULL answer and n_public not 1 or n are refused
 *                                                                                  -> prints VERIFY_DOUBLE_ALL_SMOKE_OK */
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

/* a generator of the prime-order subgroup (u, v = 18), Montgomery limbs; 1 in Montgomery form; p; r_J */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const p252_fr ONE = {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
static const uint64_t PM[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
static const p252_jscalar R_J = {{0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}};

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

static void set_pt(p252_fr* dst, p252_fr u, p252_fr v) { dst[0] = u, dst[1] = v; }

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("VERIFY_DOUBLE_ALL_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 5 };
    static const p252_fr zero;
    p252_fr Gp[2], ident[2];
    set_pt(Gp, neg(G[0]), G[1]);
    set_pt(ident, zero, ONE);
    static p252_fr PK[2 * N], R[2 * N], Rp[2 * N], msg[N];
    static p252_jscalar u[N], w[N], wp[N];
    for (int i = 0; i < N; ++i) {
        set_pt(PK + 2 * i, zero, ONE);
        if (i % 2 == 0) {                                           /* (1, G, G') */
            u[i].l[0] = 1;
            set_pt(R + 2 * i, G[0], G[1]);
            set_pt(Rp + 2 * i, Gp[0], Gp[1]);
        } else {                                                    /* (0, O, O) */
            set_pt(R + 2 * i, zero, ONE);
            set_pt(Rp + 2 * i, zero, ONE);
        }
        msg[i].l[0] = 31u * (uint64_t)i + 7u;
        w[i].l[0] = 0x9e3779b97f4a7c15ULL * (uint64_t)(i + 1), w[i].l[1] = 0x632be59bd9b4e019ULL + (uint64_t)i;
        wp[i].l[0] = 0xbf58476d1ce4e5b9ULL * (uint64_t)(i + 3), wp[i].l[1] = 0x94d049bb133111ebULL ^ (uint64_t)i;
    }
    uint8_t all = 9;
    size_t bad = 9;
    CHECK(p252_schnorr_verify_double_all(ctx, ident, ident, 1, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 2;
    all = 9;
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 3;
    u[2].l[0] = 2;                                                  /* a changed u */
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 0) return 4;
    u[2] = R_J;                                                     /* an invalid item */
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 1) return 5;
    u[2].l[0] = 1, u[2].l[1] = u[2].l[2] = u[2].l[3] = 0;
    wp[3] = R_J;                                                    /* an invalid weight_p */
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 1) return 6;
    wp[3].l[0] = 5, wp[3].l[1] = wp[3].l[2] = wp[3].l[3] = 0;
    /* item 1: u = 0, R = D, R' = -D with D = G (-D = G'): [0] G - R = -D and [0] G' - R' = +D cancel under equal
     * weights only */
    set_pt(R + 2, G[0], G[1]);
    set_pt(Rp + 2, Gp[0], Gp[1]);
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, w, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 7;
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 0 || bad != 0) return 8;
    /* item 1: R = (0, -1), of order 2, u = 0, R' = O: [8] (-R) is the identity */
    set_pt(R + 2, zero, neg(ONE));
    set_pt(Rp + 2, zero, ONE);
    CHECK(p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, &all, &bad, P252_MEM_HOST));
    if (all != 1 || bad != 0) return 9;
    all = 9;
    CHECK(p252_schnorr_verify_double_all(ctx, ident, ident, 1, NULL, NULL, NULL, NULL, NULL, NULL, 0, G, Gp, &all, &bad,
                                         P252_MEM_HOST));
    if (all != 1 || bad != 0) return 10;
    /* batch checks: an off-curve G' writes nothing, also for n == 0; a NULL answer; n_public not 1 or n */
    p252_fr off[2];
    memcpy(off, Gp, sizeof off);
    off[1].l[0] ^= 1;
    all = 9, bad = 9;
    if (p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, off, &all, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT ||
        p252_schnorr_verify_double_all(ctx, ident, ident, 1, u, R, Rp, msg, w, wp, 0, off, Gp, &all, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT)
        return 11;
    if (all != 9 || bad != 9) return 12;
    if (p252_schnorr_verify_double_all(ctx, PK, PK, N, u, R, Rp, msg, w, wp, N, G, Gp, NULL, NULL, P252_MEM_HOST) !=
            P252_ERR_INVALID_ARGUMENT ||
        p252_schnorr_verify_double_all(ctx, PK, PK, 2, u, R, Rp, msg, w, wp, N, G, Gp, &all, NULL, P252_MEM_HOST) !=
            P252_ERR_INVALID_ARGUMENT)
        return 13;
    p252_destroy(ctx);
    printf("VERIFY_DOUBLE_ALL_SMOKE_OK\n");
    return 0;
}
