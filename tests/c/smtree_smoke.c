/* Plain-C consumer of the sparse-tree entry points: calls EXACTLY the functions of the `extern "C"` block of
 * bindings/rust/src/smtree.rs, plus context handling from the first block of lib.rs (tests/test_smtree_bindings.py
 * asserts both and checks them against the header).
 *   without a GPU : argument checks that need no device, p252_create fails         -> prints SMTREE_SMOKE_NO_DEVICE
 *   with an H100  : inserts / removals / build / len / open on host buffers         -> prints SMTREE_SMOKE_OK   */
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

/* arity 4, height 3, capacity 37: 40 leaf slots, 17 node slots (levels 1..3 at 0, 12, 16) */
enum { LS = 40, NS = 17 };

int main(void) {
    static p252_fr leaves[LS], nodes[NS], leaves2[LS], nodes2[NS], paths[3 * 4], vals[4];
    static uint8_t present[LS + NS], present2[LS + NS];
    p252_smtree t = {sizeof(p252_smtree), 4, 3, 0, 37, leaves, nodes, present};
    uint64_t pos[4] = {3, 17, 36, 0}, cnt = 0;
    uint8_t op[4] = {0, 0, 0, 0};
    size_t rejected = 9;
    /* a missing context is refused before anything else */
    if (p252_smtree_build(NULL, &t, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 2;
    if (p252_smtree_update(NULL, &t, pos, op, vals, 4, &rejected, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 3;
    if (p252_smtree_len(NULL, &t, &cnt, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 4;
    if (p252_smtree_open_batch(NULL, &t, pos, 1, paths, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 5;
    p252_ctx* ctx = NULL;
    int rc = p252_create(0, &ctx);
    if (rc == P252_ERR_NO_DEVICE) {
        printf("SMTREE_SMOKE_NO_DEVICE %s\n", p252_strerror(rc));
        return 0;
    }
    CHECK(rc);
    for (int i = 0; i < 4; ++i) vals[i].l[0] = 900u + (uint64_t)i, vals[i].l[2] = (uint64_t)i;
    CHECK(p252_smtree_update(ctx, &t, pos, NULL, vals, 3, &rejected, P252_MEM_HOST));   /* insert 3, 17, 36 */
    /* remove 3, then insert it again: the later operation wins; remove 17; insert 0 */
    uint64_t pos2[4] = {3, 3, 17, 0};
    uint8_t op2[4] = {1, 0, 1, 0};
    CHECK(p252_smtree_update(ctx, &t, pos2, op2, vals, 4, &rejected, P252_MEM_HOST));
    CHECK(p252_smtree_len(ctx, &t, &cnt, P252_MEM_HOST));
    if (cnt != 3 || rejected != 0 || !present[0] || !present[3] || present[17] || !present[36]) return 6;
    if (leaves[3].l[0] != 901 || leaves[17].l[0] != 0) return 7;
    /* the same leaves built from scratch, with garbage in the nodes */
    memcpy(leaves2, leaves, sizeof leaves);
    memcpy(present2, present, LS);
    memset(nodes2, 0x5a, sizeof nodes2);
    memset(present2 + LS, 7, NS);
    p252_smtree u = {sizeof(p252_smtree), 4, 3, 0, 37, leaves2, nodes2, present2};
    CHECK(p252_smtree_build(ctx, &u, P252_MEM_HOST));
    if (memcmp(nodes, nodes2, sizeof nodes) || memcmp(present, present2, sizeof present)) return 8;
    /* level-1 groups: 0 (leaves 0..3) and 9 (36..39) present, the rest absent; level 2 node 1 (level-1 4..7) absent */
    if (!present[LS + 0] || present[LS + 4] || !present[LS + 9] || present[LS + 12 + 1] || !present[LS + 16]) return 9;
    if (nodes[4].l[0] || nodes[4].l[1] || nodes[4].l[2] || nodes[4].l[3]) return 10;
    /* refusals leave the tree as it is */
    uint64_t bad = 37;
    if (p252_smtree_update(ctx, &t, &bad, NULL, vals, 1, NULL, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 11;
    bad = 17;
    if (p252_smtree_open_batch(ctx, &t, &bad, 1, paths, P252_MEM_HOST) != P252_ERR_INVALID_ARGUMENT) return 12;
    if (memcmp(nodes, nodes2, sizeof nodes)) return 13;
    uint64_t p36 = 36;
    CHECK(p252_smtree_open_batch(ctx, &t, &p36, 1, paths, P252_MEM_HOST));
    if (memcmp(&paths[0], &leaves[36], sizeof(p252_fr)) || paths[1].l[0] || memcmp(&paths[4], &nodes[8], 4 * sizeof(p252_fr)))
        return 14;
    p252_destroy(ctx);
    printf("SMTREE_SMOKE_OK\n");
    return 0;
}
