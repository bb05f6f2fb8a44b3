"""CPU: the sparse-tree oracle (tests/smtree_oracle.py) against the prefix-tree oracle and the rules that make presence
different from a zero value, plus the sparse-tree refusals that need no device."""
import ctypes

import numpy as np
import pytest

import mtree_oracle as mo
import smtree_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.engine import mtree_layout
from poseidon252_b200.scalar import random_scalars


@pytest.mark.parametrize("arity,height,capacity,n", [(4, 3, 64, 64), (4, 3, 37, 21), (4, 3, 37, 0), (2, 6, 50, 33),
                                                     (2, 5, 32, 1), (4, 1, 4, 3)])
def test_prefix_present_set_equals_fixed_tree(arity, height, capacity, n):
    leaves = random_scalars(np.random.default_rng(n + capacity), n) if n else np.zeros((0, 4), dtype=np.uint64)
    levels = so.sparse_tree(arity, height, capacity, {j: leaves[j] for j in range(n)})
    want_leaves, want_nodes = mo.layout_of(mo.fixed_tree(arity, height, leaves), arity, height, capacity)
    got_leaves, got_nodes, present = so.buffers_of(levels)
    assert np.array_equal(got_leaves, want_leaves) and np.array_equal(got_nodes, want_nodes)
    ls, ns, _ = mtree_layout(arity, height, capacity)
    assert present.shape == (ls + ns,) and int(present[:ls].sum()) == n
    # a node is present iff its slot lies inside the prefix of its level
    m = n
    off = ls
    for l in range(1, height + 1):
        m = -(-m // arity)
        slots = levels[l][1].shape[0]
        assert list(present[off:off + slots]) == [1] * m + [0] * (slots - m)
        off += slots


def test_present_zero_leaf_differs_from_absent():
    arity, height, capacity = 4, 3, 40
    v = random_scalars(np.random.default_rng(1), 2)
    zero = np.zeros(4, dtype=np.uint64)
    absent = so.sparse_tree(arity, height, capacity, {5: v[0], 30: v[1]})
    present = so.sparse_tree(arity, height, capacity, {5: v[0], 30: v[1], 17: zero})
    assert not np.array_equal(so.root_of(absent), so.root_of(present))
    assert np.array_equal(absent[0][0], present[0][0])        # the leaf values themselves are equal
    assert not absent[1][1][4] and present[1][1][4]           # the parent of leaf 17 is absent vs H(0, 0, 0, 0)
    assert not absent[1][0][4].any() and present[1][0][4].any()
    # a tree whose only present leaf is zero has a non-zero root
    assert so.root_of(so.sparse_tree(arity, height, capacity, {0: zero})).any()


def test_removing_every_leaf_gives_zero_buffers():
    arity, height, capacity = 2, 6, 50
    rng = np.random.default_rng(2)
    pos = rng.choice(capacity, 30, replace=False)
    items = so.apply({}, pos, None, random_scalars(rng, 30))
    assert len(items) == 30 and so.root_of(so.sparse_tree(arity, height, capacity, items)).any()
    items = so.apply(items, rng.permutation(pos), np.ones(30, dtype=np.uint8), np.zeros((30, 4), dtype=np.uint64))
    leaves, nodes, present = so.buffers_of(so.sparse_tree(arity, height, capacity, items))
    assert items == {} and not leaves.any() and not nodes.any() and not present.any()


def test_batch_order_semantics():
    v = random_scalars(np.random.default_rng(3), 4)
    items = so.apply({}, [3, 3, 7, 9, 9], [0, 1, 0, 1, 0], [v[0], v[0], v[1], v[2], v[3]])
    assert sorted(items) == [7, 9] and np.array_equal(items[7], v[1]) and np.array_equal(items[9], v[3])
    after = so.apply(items, [4], [1], [v[0]])                 # removing an absent position does nothing
    assert sorted(after) == [7, 9] and all(np.array_equal(after[k], items[k]) for k in after)


def test_refusals_without_a_device():
    lib = _native.lib()
    ls, ns, _ = mtree_layout(4, 3, 37)
    leaves, nodes = np.zeros((ls, 4), dtype=np.uint64), np.zeros((ns, 4), dtype=np.uint64)
    present = np.zeros(ls + ns, dtype=np.uint8)
    t = _native.SMTree(ctypes.sizeof(_native.SMTree), 4, 3, 0, 37, leaves.ctypes.data, nodes.ctypes.data, present.ctypes.data)
    n = ctypes.c_uint64(0)
    assert lib.p252_smtree_len(None, ctypes.byref(t), ctypes.byref(n), 0) == -1
    assert lib.p252_smtree_build(None, ctypes.byref(t), 0) == -1
    assert lib.p252_smtree_update(None, ctypes.byref(t), None, None, None, 0, None, 0) == -1
    assert lib.p252_smtree_open_batch(None, ctypes.byref(t), None, 0, None, 0) == -1
