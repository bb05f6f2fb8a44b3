/* Plain-C consumer of the compact sparse-tree entry points: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/ctree.rs, plus context handling from the first block of lib.rs (tests/test_ctree_bindings.py
 * asserts both and checks them against the header).
 *   without a GPU : layout arithmetic and argument checks that need no device, p252_create fails -> CTREE_SMOKE_NO_DEVICE
 *   with an H100  : inserts / removals / open / refusals on host buffers at arity 2, height 64   -> CTREE_SMOKE_OK   */
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

/* arity 2, height 64, max_leaves 8: levels 0..61 have 8 slots, levels 62, 63, 64 have 4, 2, 1 */
enum { H = 64, ML = 8, TOTAL = 62 * 8 + 4 + 2 + 1 };

int main(void) {
    static uint64_t keys[TOTAL], keys2[TOTAL], count[H + 1], off[H + 1];
    static p252_fr values[TOTAL], vals[8], paths[H * 2];
    uint64_t total = 0;
    p252_ctree t = {sizeof(p252_ctree), 2, H, 0, ML, keys, values, count};
    /* layout: pure arithmetic, 2^64 positions, refusals */
    CHECK(p252_ctree_layout(2, H, ML, &total, off));
    if (total != TOTAL || off[1] != 8 || off[62] != 62 * 8 || off[63] != 62 * 8 + 4 || off[64] != TOTAL - 1) return 2;
    if (p252_ctree_layout(4, 33, ML, &total, off) != P252_ERR_INVALID_ARGUMENT) return 3;   /* 4^33 > 2^64 */
    if (p252_ctree_layout(2, H, 0, &total, off) != P252_ERR_INVALID_ARGUMENT) return 4;
    /* a missing context is refused before anything else */
    uint64_t pos[6] = {0, UINT64_MAX, 1, 5, 0, 0};
    size_t rejected = 9;
    if (p252_ctree_update(NULL, &t, pos, NULL, vals, 4, &rejected, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 5;
    if (p252_ctree_open_batch(NULL, &t, pos, 1, paths, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 6;
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("CTREE_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    for (int i = 0; i < 8; ++i) vals[i].l[0] = 700u + (uint64_t)i, vals[i].l[3] = (uint64_t)i;
    CHECK(p252_ctree_update(ctx, &t, pos, NULL, vals, 4, &rejected, P252_MEM_HOST));   /* insert 0, 2^64-1, 1, 5 */
    uint64_t gone = 1;
    uint8_t op = 1;
    CHECK(p252_ctree_update(ctx, &t, &gone, &op, vals, 1, &rejected, P252_MEM_HOST));   /* remove 1 */
    if (rejected != 0 || count[0] != 3 || keys[0] != 0 || keys[1] != 5 || keys[2] != UINT64_MAX || keys[3] != 0) return 7;
    if (values[1].l[0] != 703 || values[2].l[0] != 701 || values[3].l[0] != 0) return 8;
    if (count[H] != 1 || !(values[TOTAL - 1].l[0] | values[TOTAL - 1].l[1] | values[TOTAL - 1].l[2] | values[TOTAL - 1].l[3]))
        return 9;
    /* level 1: parents 0 (of 0), 2 (of 5) and 2^63 - 1 (of 2^64 - 1) */
    if (count[1] != 3 || keys[off[1]] != 0 || keys[off[1] + 1] != 2 || keys[off[1] + 2] != UINT64_MAX / 2) return 10;
    /* the opening of 2^64 - 1: its level-0 group is (absent 2^64 - 2, the value) */
    uint64_t top = UINT64_MAX;
    CHECK(p252_ctree_open_batch(ctx, &t, &top, 1, paths, P252_MEM_HOST));
    if (paths[0].l[0] || memcmp(&paths[1], &values[2], sizeof(p252_fr))) return 11;
    /* refusals leave the tree as it is: an absent position, and a batch beyond max_leaves */
    if (p252_ctree_open_batch(ctx, &t, &gone, 1, paths, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 12;
    memcpy(keys2, keys, sizeof keys);
    uint64_t many[6] = {10, 11, 12, 13, 14, 15};
    if (p252_ctree_update(ctx, &t, many, NULL, vals, 6, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 13;
    if (memcmp(keys, keys2, sizeof keys) || count[0] != 3) return 14;
    p252_destroy(ctx);
    printf("CTREE_SMOKE_OK\n");
    return 0;
}
