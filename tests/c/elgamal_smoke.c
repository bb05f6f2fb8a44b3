/* Plain-C consumer of JubJub ElGamal and the encrypted note sender: calls EXACTLY the functions of the `extern "C"` block
 * of bindings/rust/src/elgamal.rs, plus functions from the first block of lib.rs (tests/test_elgamal_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                    -> prints ELGAMAL_SMOKE_NO_DEVICE
 *   with an H100  : M = G encrypted under PK = G (sk = 1) decrypts to G, and with r = 0 gives (identity, M); an r >= r_J
 *                   is zeroed and counted.  The sender (A, B) = (G, identity) of a note with R = the identity and
 *                   b = r_J - hash(identity) + 1 (so note_sk = 1 and note_pk = G is owned) comes back; the same note with
 *                   another note_pk is not owned.  An off-curve G is refused with nothing written, also for n == 0
 *                                                                                        -> prints ELGAMAL_SMOKE_OK   */
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

/* a generator of the prime-order subgroup (u, v = 18), Montgomery limbs; ONE is 1 */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const p252_fr ONE = {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
static const uint64_t R_J[4] = {0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("ELGAMAL_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 3 };
    static p252_fr ident[2], M[2 * N], c1[2 * N], c2[2 * N], out[2 * N], h;
    static p252_jscalar r[N], sk[1];
    static const p252_fr zero[2];
    uint8_t ok[N];
    size_t bad = 9;
    ident[1] = ONE;
    for (int i = 0; i < N; ++i) M[2 * i] = G[0], M[2 * i + 1] = G[1];
    r[0].l[0] = 5, r[1].l[0] = 0;
    memcpy(r[2].l, R_J, sizeof R_J);                                   /* item 2: r = r_J */
    sk[0].l[0] = 1;
    CHECK(p252_elgamal_encrypt_batch(ctx, G, 1, M, r, N, G, c1, c2, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || !ok[0] || !ok[1] || ok[2]) return 2;
    if (memcmp(&c1[2], ident, sizeof ident) || memcmp(&c2[2], G, sizeof G)) return 3;           /* r = 0 */
    if (memcmp(&c1[4], zero, sizeof zero) || memcmp(&c2[4], zero, sizeof zero)) return 4;      /* zeroed */
    CHECK(p252_elgamal_decrypt_batch(ctx, sk, 1, c1, c2, 2, out, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || memcmp(&out[0], G, sizeof G) || memcmp(&out[2], G, sizeof G)) return 5;
    /* the sender: note_sk = hash(identity) + b = 1 */
    static p252_fr R[2], note_pk[2], A[2], B[2], enc[8], gotA[2], gotB[2];
    static p252_jscalar a[1], b[1], blinder[2];
    CHECK(p252_hash_batch_truncated(ctx, P252_DOMAIN_OTHER, ident, 1, 2, &h, 1, P252_MEM_HOST));
    uint64_t borrow = 0, carry = 1;
    for (int k = 0; k < 4; ++k) {
        const uint64_t d = R_J[k] - h.l[k] - borrow;
        borrow = (R_J[k] < h.l[k]) || (R_J[k] - h.l[k] < borrow);
        b[0].l[k] = d + carry;
        carry = carry && b[0].l[k] == 0;
    }
    a[0].l[0] = 0x1234567890abcdefULL;
    R[0] = ident[0], R[1] = ident[1];
    note_pk[0] = G[0], note_pk[1] = G[1];
    A[0] = G[0], A[1] = G[1], B[0] = ident[0], B[1] = ident[1];
    blinder[0].l[0] = 7, blinder[1].l[0] = 11;
    CHECK(p252_note_sender_encrypt_batch(ctx, note_pk, A, B, 1, blinder, 1, G, enc, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || !ok[0]) return 6;
    CHECK(p252_note_sender_decrypt_batch(ctx, a, b, 1, R, note_pk, enc, 1, G, gotA, gotB, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || !ok[0] || memcmp(gotA, A, sizeof A) || memcmp(gotB, B, sizeof B)) return 7;
    CHECK(p252_note_sender_decrypt_batch(ctx, a, b, 1, R, &c1[0], enc, 1, G, gotA, gotB, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || ok[0] || memcmp(gotA, zero, sizeof zero) || memcmp(gotB, zero, sizeof zero)) return 8;
    /* batch checks: an off-curve G writes nothing, also for n == 0 */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    memset(ok, 0xA5, sizeof ok);
    bad = 9;
    if (p252_elgamal_encrypt_batch(ctx, G, 1, M, r, N, off, c1, c2, ok, &bad, P252_MEM_HOST) != P252_ERR_INVALID_POINT ||
        p252_note_sender_encrypt_batch(ctx, note_pk, A, B, 1, blinder, 0, off, enc, ok, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT ||
        p252_note_sender_decrypt_batch(ctx, a, b, 1, R, note_pk, enc, 1, off, gotA, gotB, ok, &bad, P252_MEM_HOST) !=
            P252_ERR_INVALID_POINT)
        return 9;
    if (ok[0] != 0xA5 || bad != 9) return 10;
    p252_destroy(ctx);
    printf("ELGAMAL_SMOKE_OK\n");
    return 0;
}
