/* Plain-C consumer of the point compression: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/points.rs, plus functions from the first block of lib.rs (tests/test_points_cpu.py asserts both).
 *   without a GPU : p252_create fails                                                  -> prints POINTS_SMOKE_NO_DEVICE
 *   with an H100  : G and -G encode with the same v and opposite sign bits and decode back; 32 zero bytes decode (v = 0);
 *                   an off-curve point encodes to 32 bytes of 0xff, which do not decode, and both are counted; a NULL
 *                   buffer is refused                                                  -> prints POINTS_SMOKE_OK   */
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
/* p, the field modulus */
static const uint64_t P[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};

int main(void) {
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("POINTS_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    enum { N = 4 };
    p252_fr pts[2 * N], back[2 * N];
    uint8_t bytes[32 * N], ok[N];
    size_t bad = 9;
    /* 0: G, 1: -G (u -> p - u, which in Montgomery form is also p - limbs), 2: (0, 0) off the curve, 3: G */
    memcpy(pts, G, sizeof G);
    pts[2] = G[0], pts[3] = G[1];
    unsigned __int128 borrow = 0;
    for (int k = 0; k < 4; ++k) {
        const unsigned __int128 d = (unsigned __int128)P[k] - G[0].l[k] - borrow;
        pts[2].l[k] = (uint64_t)d;
        borrow = (d >> 64) ? 1 : 0;
    }
    memset(&pts[4], 0, 2 * sizeof(p252_fr));
    memcpy(&pts[6], G, sizeof G);
    CHECK(p252_points_to_bytes(ctx, pts, N, bytes, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || !ok[0] || !ok[1] || ok[2] || !ok[3]) return 2;
    if (memcmp(bytes, bytes + 32, 31) || ((bytes[31] ^ bytes[63]) != 0x80)) return 3;   /* same v, opposite sign */
    for (int j = 0; j < 32; ++j)
        if (bytes[64 + j] != 0xff) return 4;
    CHECK(p252_points_from_bytes(ctx, bytes, N, back, ok, &bad, P252_MEM_HOST));
    if (bad != 1 || !ok[0] || !ok[1] || ok[2] || !ok[3]) return 5;
    if (memcmp(back, pts, 2 * sizeof(p252_fr)) || memcmp(back + 2, pts + 2, 2 * sizeof(p252_fr))) return 6;
    static const p252_fr zero_row[2];
    if (memcmp(back + 4, zero_row, sizeof zero_row)) return 7;                 /* the rejected row is (0, 0) */
    /* 32 zero bytes: v = 0, the order-4 point (sqrt(-1), 0) */
    memset(bytes, 0, 32);
    CHECK(p252_points_from_bytes(ctx, bytes, 1, back, ok, NULL, P252_MEM_HOST));
    if (!ok[0] || memcmp(&back[1], &zero_row[0], sizeof(p252_fr)) != 0 || memcmp(&back[0], &zero_row[0], sizeof(p252_fr)) == 0)
        return 8;
    /* batch checks */
    if (p252_points_from_bytes(ctx, NULL, 1, back, ok, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 9;
    if (p252_points_to_bytes(ctx, pts, 1, bytes, NULL, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 10;
    p252_destroy(ctx);
    printf("POINTS_SMOKE_OK\n");
    return 0;
}
