/* Plain-C consumer of the stealth addresses: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/stealth.rs, plus functions from the first block of lib.rs (tests/test_stealth_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                  -> prints STEALTH_SMOKE_NO_DEVICE
 *   with an H100  : the receiver's keys A = [a] G and B = [b] G come from the sender call itself (A = B = the identity
 *                   makes R = [r] G); notes to (A, B) are owned by (a, B) and by no other view key, an r >= r_J is
 *                   zeroed and counted, its note is invalid in the scan, and an off-curve spend key is refused with
 *                   nothing written                                                    -> prints STEALTH_SMOKE_OK   */
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

/* the generator used by the tests (u, v = 18) and the identity (0, 1), Montgomery limbs */
static const p252_fr G[2] = {{{0xc8cd898c547c71aaULL, 0x1e77bad0b3564650ULL, 0x0b5183a649031ebeULL, 0x4f54a483a3031a2cULL}},
                             {{0x00000026ffffffd9ULL, 0x3e1c038b003ffc27ULL, 0x323016c688581730ULL, 0x56cb8254a901ea00ULL}}};
static const p252_fr O[2] = {{{0, 0, 0, 0}},
                             {{0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL}}};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("STEALTH_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 7 };
    static p252_jscalar keys[2], r[N], other[1];
    static p252_fr key_uv[4], key_pk[4], R[2 * N], pk[2 * N];
    uint8_t ok[N], owned[N];
    size_t bad = 9, mine = 9;
    keys[0].l[0] = 0x1234567890abcdefULL, keys[0].l[1] = 42, keys[0].l[3] = 0x0e7db4ea6533afa8ULL;   /* a < r_J */
    keys[1].l[0] = 0xfeedfacecafebeefULL, keys[1].l[2] = 7;                                         /* b */
    other[0] = keys[0];
    other[0].l[0] ^= 1;
    for (int i = 0; i < N; ++i) r[i].l[0] = 1000u + (uint64_t)i, r[i].l[2] = (uint64_t)i << 40;
    r[3].l[3] = 0x0e7db4ea6533afaaULL;                          /* item 3: r >= r_J */
    /* (A, B) = ([a] G, [b] G): the R rows of a sender call to the identity */
    CHECK(p252_stealth_address_batch(ctx, keys, 2, G, O, O, 1, key_uv, key_pk, ok, &bad, P252_MEM_HOST));
    if (!ok[0] || !ok[1] || bad != 0) return 2;
    const p252_fr* A = key_uv;
    const p252_fr* B = key_uv + 2;
    CHECK(p252_stealth_address_batch(ctx, r, N, G, A, B, 1, R, pk, ok, &bad, P252_MEM_HOST));
    if (bad != 1) return 3;
    for (int i = 0; i < N; ++i) {
        static const p252_fr zero[2];
        if (ok[i] != (i == 3 ? 0 : 1)) return 4;
        if ((i == 3) != (memcmp(pk + 2 * i, zero, sizeof zero) == 0 && memcmp(R + 2 * i, zero, sizeof zero) == 0)) return 5;
    }
    CHECK(p252_stealth_owns_batch(ctx, keys, B, G, R, pk, N, owned, &mine, &bad, P252_MEM_HOST));
    if (mine != N - 1 || bad != 1) return 6;   /* the zeroed note 3: R = (0, 0) is not a curve point */
    for (int i = 0; i < N; ++i)
        if (owned[i] != (i == 3 ? 0 : 1)) return 7;
    CHECK(p252_stealth_owns_batch(ctx, other, B, G, R, pk, N, owned, &mine, &bad, P252_MEM_HOST));
    if (mine != 0 || bad != 1) return 8;
    /* batch checks: an off-curve spend key writes nothing */
    p252_fr off[2];
    memcpy(off, B, sizeof off);
    off[1].l[0] ^= 1;
    memset(owned, 0xA5, sizeof owned);
    mine = 9;
    if (p252_stealth_owns_batch(ctx, keys, off, G, R, pk, N, owned, &mine, NULL, P252_MEM_HOST) != P252_ERR_INVALID_POINT)
        return 9;
    if (owned[0] != 0xA5 || mine != 9) return 10;
    if (p252_stealth_address_batch(ctx, r, N, G, A, B, 2, R, pk, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT)
        return 11;
    p252_destroy(ctx);
    printf("STEALTH_SMOKE_OK\n");
    return 0;
}
