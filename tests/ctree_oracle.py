"""Oracle of the compact sparse tree (p252_ctree), restated from {position: value} level by level.

Presence and node values are those of the sparse tree (tests/smtree_oracle.py): a node is present iff one of its arity
children is present; a present node is Hash::digest(Domain::Merkle{A}, its child slots) with absent children reading as
0; an absent node is 0 and is never hashed (src/hash.rs:24-26).  Here only the present nodes exist: level l is a dict
{index: value}, so any height up to 64 (arity 2) or 32 (arity 4) works.  `hash_groups` is one of mtree_oracle's
(pure-Python or the C restatement); every level is one call, so heights 32 and 64 stay fast.

`buffers_of` lays the levels out as p252_ctree holds them (p252_ctree_layout): per level the sorted keys and their
values packed from the level's first slot, zeros after, and the per-level counts."""
import numpy as np

from mtree_oracle import py_hash_groups


def compact_levels(arity, height, items, hash_groups=None):
    """items: {position: (4,) uint64 value} -> [ {index: (4,) uint64} ] for levels 0..height (level height: {0: root}
    or {} for the empty tree)."""
    hash_groups = hash_groups or py_hash_groups(arity)
    cur = {int(k): np.asarray(v, dtype=np.uint64) for k, v in items.items()}
    assert all(0 <= k < arity ** height for k in cur)
    levels = [cur]
    for _ in range(height):
        parents = sorted({k // arity for k in cur})
        groups = np.zeros((len(parents), arity, 4), dtype=np.uint64)
        row = {g: r for r, g in enumerate(parents)}
        for k, v in cur.items():
            groups[row[k // arity], k % arity] = v
        digests = hash_groups(groups) if parents else np.zeros((0, 4), dtype=np.uint64)
        cur = {g: digests[r] for r, g in enumerate(parents)}
        levels.append(cur)
    return levels


def root_of(levels):
    return levels[-1].get(0, np.zeros(4, dtype=np.uint64))


def buffers_of(levels, arity, height, max_leaves):
    """(keys (total,), values (total, 4), count (height + 1,)) exactly as p252_ctree holds them."""
    from poseidon252_b200.engine import ctree_layout
    total, off = ctree_layout(arity, height, max_leaves)
    keys = np.zeros(total, dtype=np.uint64)
    values = np.zeros((total, 4), dtype=np.uint64)
    count = np.zeros(height + 1, dtype=np.uint64)
    for l, lv in enumerate(levels):
        ks = sorted(lv)
        assert len(ks) <= (off[l + 1] if l < height else total) - off[l]
        count[l] = len(ks)
        for j, k in enumerate(ks):
            keys[off[l] + j] = k
            values[off[l] + j] = lv[k]
    return keys, values, count


def paths(levels, arity, pos):
    """Openings (len(pos), height, arity, 4): per level the full sibling group, absent slots 0."""
    height = len(levels) - 1
    out = np.zeros((len(pos), height, arity, 4), dtype=np.uint64)
    for n, i in enumerate(pos):
        i = int(i)
        for l in range(height):
            g = i // arity
            for q in range(arity):
                v = levels[l].get(g * arity + q)
                if v is not None:
                    out[n, l, q] = v
            i = g
    return out
