"""Oracle of the sparse fixed-height tree (p252_smtree), restated from the node hash and the empty-slot rule.

Each position in [0, capacity) is present (holds a value) or absent.  Level-0 slot j holds the leaf value if j is
present and 0 otherwise.  A node of level l >= 1 is present iff one of its arity children is present; a present node is
Hash::digest(Domain::Merkle{A}, its children's slots) with absent children reading as 0, an absent node IS 0 and is
never hashed (src/hash.rs:24-26).  So presence is stored beside the values: a present leaf of value zero makes its
parent H(0, ..), an absent one leaves it 0.

`sparse_tree` returns every level over its full slot range (p252_mtree_layout) as (values (slots, 4), present (slots,)),
leaves first; `hash_groups` is one of mtree_oracle's (pure-Python or the C restatement)."""
import numpy as np

from mtree_oracle import py_hash_groups


def sparse_tree(arity, height, capacity, items, hash_groups=None):
    """items: {position: (4,) uint64 value} of the present positions -> [(values, present)] for levels 0..height."""
    from poseidon252_b200.engine import mtree_layout
    hash_groups = hash_groups or py_hash_groups(arity)
    leaf_slots, node_slots, off = mtree_layout(arity, height, capacity)
    vals = np.zeros((leaf_slots, 4), dtype=np.uint64)
    pres = np.zeros(leaf_slots, dtype=bool)
    for j, v in items.items():
        assert 0 <= j < capacity
        vals[j] = v
        pres[j] = True
    levels = [(vals, pres)]
    for l in range(1, height + 1):
        slots = (off[l + 1] if l < height else node_slots) - off[l]
        groups = vals.reshape(-1, arity, 4)
        gp = pres.reshape(-1, arity).any(axis=1)
        nv = np.zeros((slots, 4), dtype=np.uint64)
        npres = np.zeros(slots, dtype=bool)
        if gp.any():
            nv[:gp.shape[0]][gp] = hash_groups(np.ascontiguousarray(groups[gp]))
        npres[:gp.shape[0]] = gp
        vals, pres = nv, npres
        levels.append((vals, pres))
    return levels


def root_of(levels):
    return levels[-1][0][0]


def buffers_of(levels):
    """(leaves, nodes, present) exactly as p252_smtree holds them: nodes levels 1..H bottom-up, presence bytes of the
    leaves then of the nodes."""
    leaves = levels[0][0]
    nodes = np.concatenate([v for v, _ in levels[1:]])
    present = np.concatenate([p for _, p in levels]).astype(np.uint8)
    return leaves, nodes, present


def paths(levels, arity, pos):
    """Openings (len(pos), height, arity, 4): per level the full sibling group (absent slots are 0 in the levels)."""
    height = len(levels) - 1
    out = np.zeros((len(pos), height, arity, 4), dtype=np.uint64)
    for k, i in enumerate(pos):
        i = int(i)
        for l in range(height):
            g = i // arity
            out[k, l] = levels[l][0][g * arity:(g + 1) * arity]
            i = g
    return out


def apply(items, pos, op, values):
    """The batch applied one operation after another: op 0 inserts / overwrites, op 1 removes."""
    items = dict(items)
    for k, p in enumerate(pos):
        p = int(p)
        if op is None or int(op[k]) == 0:
            items[p] = np.asarray(values[k], dtype=np.uint64).copy()
        else:
            items.pop(p, None)
    return items
