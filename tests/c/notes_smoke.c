/* Plain-C consumer of the note value calls: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/notes.rs, plus functions from the first block of lib.rs (tests/test_notes_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                  -> prints NOTES_SMOKE_NO_DEVICE
 *   with an H100  : G' = -G, so commit(v, v) is the identity.  Notes created for the receiver (A, B) = (G, G) (view key
 *                   a = 1) carry the same commitments as p252_value_commit_batch, open under a = 1 with their (v,
 *                   blinder), and do not open under a = 2; a blinder >= r_J is zeroed and counted, an off-curve G' is
 *                   refused with nothing written (also for n == 0), and n_public not 1 or n is refused
 *                                                                                      -> prints NOTES_SMOKE_OK   */
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

/* a generator of the prime-order subgroup (u, v = 18), Montgomery limbs, the field modulus p and 1 (Montgomery) */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const uint64_t PM[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
static const p252_fr ONE = {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};

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
        printf("NOTES_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 3 };
    p252_fr Gp[2];
    Gp[0] = neg(G[0]), Gp[1] = G[1];
    static p252_fr nonce[N], R[2 * N], pk[2 * N], C[2 * N], C2[2 * N], cipher[3 * N], zero;
    static p252_jscalar r[N], blinder[N], b_out[N], a;
    uint64_t value[N] = {0, 1234567, 0xffffffffffffffffULL}, v_out[N];
    uint8_t ok[N];
    size_t bad = 9;
    for (int i = 0; i < N; ++i) {
        r[i].l[0] = 1000 + (uint64_t)i, r[i].l[3] = 0x0123456789abcdefULL;
        blinder[i].l[0] = 0xfedcba9876543210ULL, blinder[i].l[1] = (uint64_t)i;
        nonce[i].l[0] = 77 + (uint64_t)i;
    }
    /* commit(v, v) with G' = -G is the identity (0, 1) */
    static p252_jscalar vb[1];
    vb[0].l[0] = 1234567;
    CHECK(p252_value_commit_batch(ctx, &value[1], vb, 1, G, Gp, C, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || !ok[0] || memcmp(&C[0], &zero, sizeof zero) || memcmp(&C[1], &ONE, sizeof ONE)) return 2;
    CHECK(p252_value_commit_batch(ctx, value, blinder, N, G, Gp, C2, ok, &bad, P252_MEM_HOST));
    if (bad != 0) return 3;
    CHECK(p252_note_create_batch(ctx, r, value, blinder, nonce, N, G, Gp, G, G, 1, R, pk, C, cipher, ok, &bad,
                                 P252_MEM_HOST));
    if (bad != 0 || !ok[0] || !ok[1] || !ok[2] || memcmp(C, C2, sizeof C)) return 4;
    a.l[0] = 1;                                                     /* the receiver's view key: A = [1] G */
    CHECK(p252_note_open_batch(ctx, &a, 1, R, nonce, cipher, C, N, G, Gp, v_out, b_out, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || memcmp(v_out, value, sizeof value) || memcmp(b_out, blinder, sizeof b_out)) return 5;
    a.l[0] = 2;                                                     /* another view key opens nothing */
    CHECK(p252_note_open_batch(ctx, &a, 1, R, nonce, cipher, C, N, G, Gp, v_out, b_out, ok, &bad, P252_MEM_HOST));
    if (bad != N || ok[0] || ok[1] || ok[2] || v_out[2] != 0) return 6;
    /* item 1: blinder >= r_J -> every row zeroed, counted once */
    blinder[1].l[3] = 0x0e7db4ea6533afaaULL;
    CHECK(p252_note_create_batch(ctx, r, value, blinder, nonce, N, G, Gp, G, G, 1, R, pk, C, cipher, ok, &bad,
                                 P252_MEM_HOST));
    if (bad != 1 || !ok[0] || ok[1] || !ok[2]) return 7;
    for (int k = 0; k < 3; ++k)
        if (memcmp(&cipher[3 + k], &zero, sizeof zero) || (k < 2 && (memcmp(&R[2 + k], &zero, sizeof zero) ||
                                                                      memcmp(&pk[2 + k], &zero, sizeof zero) ||
                                                                      memcmp(&C[2 + k], &zero, sizeof zero))))
            return 8;
    /* batch checks: an off-curve G' writes nothing, also for n == 0; n_public must be 1 or n */
    p252_fr off[2];
    memcpy(off, Gp, sizeof off);
    off[1].l[0] ^= 1;
    memset(ok, 0xA5, sizeof ok);
    bad = 9;
    if (p252_value_commit_batch(ctx, value, blinder, N, G, off, C, ok, &bad, P252_MEM_HOST) != P252_ERR_INVALID_POINT ||
        p252_note_open_batch(ctx, &a, 1, R, nonce, cipher, C, 0, off, Gp, v_out, b_out, ok, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT)
        return 9;
    if (ok[0] != 0xA5 || bad != 9) return 10;
    if (p252_note_create_batch(ctx, r, value, blinder, nonce, N, G, Gp, G, G, 2, R, pk, C, cipher, ok, NULL,
                               P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 11;
    p252_destroy(ctx);
    printf("NOTES_SMOKE_OK\n");
    return 0;
}
