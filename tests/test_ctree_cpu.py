"""CPU: the compact-tree oracle (tests/ctree_oracle.py) against the sparse-tree oracle, the p252_ctree_layout arithmetic,
and the compact-tree refusals that need no device."""
import ctypes

import numpy as np
import pytest

import ctree_oracle as co
import smtree_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.engine import ctree_layout
from poseidon252_b200.errors import EngineError
from poseidon252_b200.scalar import random_scalars


@pytest.mark.parametrize("arity,height,n", [(4, 3, 20), (4, 3, 64), (2, 6, 33), (2, 5, 1), (4, 1, 3), (2, 4, 0)])
def test_oracle_equals_sparse_tree_present_slots(arity, height, n):
    rng = np.random.default_rng(arity * 100 + height * 10 + n)
    cap = arity ** height
    pos = rng.choice(cap, n, replace=False)
    vals = random_scalars(rng, n) if n else np.zeros((0, 4), dtype=np.uint64)
    items = {int(p): vals[k] for k, p in enumerate(pos)}
    sparse = so.sparse_tree(arity, height, cap, items)
    compact = co.compact_levels(arity, height, items)
    for l in range(height + 1):
        values, present = sparse[l]
        idx = np.flatnonzero(present)
        assert sorted(compact[l]) == [int(i) for i in idx]
        for i in idx:
            assert np.array_equal(compact[l][int(i)], values[i])
    assert np.array_equal(co.root_of(compact), so.root_of(sparse))
    # openings equal the sparse tree's
    if n:
        assert np.array_equal(co.paths(compact, arity, pos[:5]), so.paths(sparse, arity, pos[:5]))


def test_buffers_are_canonical():
    arity, height, max_leaves = 2, 5, 10
    v = random_scalars(np.random.default_rng(4), 3)
    keys, values, count = co.buffers_of(co.compact_levels(arity, height, {31: v[0], 0: v[1], 30: v[2]}), arity, height,
                                        max_leaves)
    total, off = ctree_layout(arity, height, max_leaves)
    assert total == 10 + 10 + 8 + 4 + 2 + 1 and off == [0, 10, 20, 28, 32, 34]
    assert list(count) == [3, 2, 2, 2, 2, 1]
    assert list(keys[:4]) == [0, 30, 31, 0] and list(keys[off[1]:off[1] + 3]) == [0, 15, 0]
    assert not values[3:off[1]].any() and not keys[3:off[1]].any()


def test_empty_tree_is_all_zero():
    keys, values, count = co.buffers_of(co.compact_levels(4, 6, {}), 4, 6, 16)
    assert not keys.any() and not values.any() and not count.any()


def test_present_zero_leaf_differs_from_absent():
    v = random_scalars(np.random.default_rng(5), 1)[0]
    zero = np.zeros(4, dtype=np.uint64)
    a = co.compact_levels(2, 64, {7: v})
    b = co.compact_levels(2, 64, {7: v, 2 ** 64 - 1: zero})
    assert not np.array_equal(co.root_of(a), co.root_of(b))
    assert co.root_of(co.compact_levels(2, 64, {0: zero})).any()


@pytest.mark.parametrize("arity,height", [(2, 64), (4, 32), (2, 1), (4, 1), (2, 63), (4, 31)])
def test_layout_arithmetic(arity, height):
    for max_leaves in (1, 5, 2 ** 20, 2 ** 31 - 1):
        total, off = ctree_layout(arity, height, max_leaves)
        slots = [min(max_leaves, arity ** (height - l)) for l in range(height + 1)]
        assert off == [sum(slots[:l]) for l in range(height + 1)] and total == sum(slots)
        assert slots[height] == 1


@pytest.mark.parametrize("arity,height,max_leaves", [(4, 33, 8), (2, 65, 8), (2, 0, 8), (3, 4, 8), (2, 8, 0),
                                                     (4, 8, 2 ** 31), (2, 64, 2 ** 40)])
def test_layout_refusals(arity, height, max_leaves):
    with pytest.raises(EngineError):
        ctree_layout(arity, height, max_leaves)
    lib = _native.lib()
    total = ctypes.c_uint64(7)
    assert lib.p252_ctree_layout(arity, height, max_leaves, ctypes.byref(total), None) == -1
    assert total.value == 7


def test_refusals_without_a_device():
    lib = _native.lib()
    total, _ = ctree_layout(4, 32, 16)
    keys, values, count = np.zeros(total, dtype=np.uint64), np.zeros((total, 4), dtype=np.uint64), np.zeros(33, dtype=np.uint64)
    t = _native.CTree(ctypes.sizeof(_native.CTree), 4, 32, 0, 16, keys.ctypes.data, values.ctypes.data, count.ctypes.data)
    assert ctypes.sizeof(_native.CTree) == 48
    assert lib.p252_ctree_update(None, ctypes.byref(t), None, None, None, 0, None, 0) == -1
    assert lib.p252_ctree_open_batch(None, ctypes.byref(t), None, 0, None, 0) == -1
