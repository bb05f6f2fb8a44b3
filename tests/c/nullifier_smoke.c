/* Plain-C consumer of the note nullifiers: calls EXACTLY the function of the `extern "C"` block of
 * bindings/rust/src/nullifier.rs, plus functions from the first block of lib.rs (tests/test_nullifier_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                  -> prints NULLIFIER_SMOKE_NO_DEVICE
 *   with an H100  : for notes with R = the identity, [a] R is the identity, so h = hash(identity) comes from
 *                   p252_hash_batch_truncated and b = r_J - h makes note_sk = 0 and pk' = the identity: the nullifiers
 *                   at positions 0 and 1 equal p252_hash_batch(Other, [0, 1, pos]).  An a >= r_J is zeroed and counted,
 *                   an off-curve G' is refused with nothing written, and n_secret not 1 or n is refused
 *                                                                                      -> prints NULLIFIER_SMOKE_OK   */
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

/* a generator of the prime-order subgroup (u, v = 18) and the identity (0, 1), Montgomery limbs; ONE is 1 */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const p252_fr ONE = {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}};
static const uint64_t R_J[4] = {0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("NULLIFIER_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 3 };
    static p252_fr ident[2], R[2 * N], rows[3 * 2], want[2], h, nul[N];
    static p252_jscalar a[N], b[N];
    uint8_t ok[N];
    size_t bad = 9;
    ident[1] = ONE;
    /* h = hash(identity), canonical and < 2^250; b = r_J - h */
    CHECK(p252_hash_batch_truncated(ctx, P252_DOMAIN_OTHER, ident, 1, 2, &h, 1, P252_MEM_HOST));
    uint64_t borrow = 0;
    for (int k = 0; k < 4; ++k) {
        const uint64_t d = R_J[k] - h.l[k] - borrow;
        borrow = (R_J[k] < h.l[k]) || (R_J[k] - h.l[k] < borrow);
        b[0].l[k] = d;
    }
    for (int i = 0; i < N; ++i) R[2 * i] = ident[0], R[2 * i + 1] = ident[1], a[i].l[0] = 0x1234567890abcdefULL + (uint64_t)i,
        b[i] = b[0];
    a[2].l[3] = 0x0e7db4ea6533afaaULL;                              /* item 2: a >= r_J */
    const uint64_t pos[N] = {0, 1, 1};
    /* the digest rows [0, 1, pos] of pk' = the identity: pos 0 is the zero scalar, pos 1 is ONE */
    memset(rows, 0, sizeof rows);
    rows[1] = ONE, rows[4] = ONE, rows[5] = ONE;
    CHECK(p252_hash_batch(ctx, P252_DOMAIN_OTHER, rows, 2, 3, want, 1, P252_MEM_HOST));
    CHECK(p252_nullifier_batch(ctx, a, b, N, G, R, pos, N, nul, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || !ok[0] || !ok[1] || ok[2]) return 2;
    if (memcmp(&nul[0], &want[0], sizeof(p252_fr)) || memcmp(&nul[1], &want[1], sizeof(p252_fr))) return 3;
    static const p252_fr zero;
    if (memcmp(&nul[2], &zero, sizeof zero)) return 4;
    /* one key for the batch (n_secret = 1) */
    CHECK(p252_nullifier_batch(ctx, a, b, 1, G, R, pos, N, nul, ok, &bad, P252_MEM_HOST));
    if (bad != 0 || memcmp(&nul[2], &want[1], sizeof(p252_fr))) return 5;
    /* batch checks: an off-curve G' writes nothing, also for n == 0; n_secret must be 1 or n */
    p252_fr off[2];
    memcpy(off, G, sizeof off);
    off[1].l[0] ^= 1;
    memset(ok, 0xA5, sizeof ok);
    bad = 9;
    if (p252_nullifier_batch(ctx, a, b, 1, off, R, pos, N, nul, ok, &bad, P252_MEM_HOST) != P252_ERR_INVALID_POINT ||
        p252_nullifier_batch(ctx, a, b, 1, off, R, pos, 0, nul, ok, &bad, P252_MEM_HOST) != P252_ERR_INVALID_POINT)
        return 6;
    if (ok[0] != 0xA5 || bad != 9) return 7;
    if (p252_nullifier_batch(ctx, a, b, 2, G, R, pos, N, nul, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 8;
    p252_destroy(ctx);
    printf("NULLIFIER_SMOKE_OK\n");
    return 0;
}
