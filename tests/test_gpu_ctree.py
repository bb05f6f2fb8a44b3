"""GPU (-m gpu): compact sparse trees (p252_ctree) against a full-capacity p252_smtree fed the same batches and against
the oracle restatement (tests/ctree_oracle.py) at heights where every u64 is a position -- mixed batches, duplicates,
absent removals, emptying the tree, present zero leaves, one batch versus several, host versus device buffers,
rejections with canaries, capacity refusals, openings and asynchronous updates.  Both digest kernels (the two-parameter
`engine` fixture)."""
import numpy as np
import pytest

import ctree_oracle as co
import mtree_oracle as mo
import smtree_oracle as so
import poseidon252_b200 as pb
from poseidon252_b200 import merkle
from poseidon252_b200.scalar import random_scalars

pytestmark = pytest.mark.gpu

MEMS = ["host", "device"]
U64 = (1 << 64) - 1


def host(x):
    if hasattr(x, "is_cuda"):
        a = x.cpu().numpy()
        return a if a.dtype == np.uint8 else a.view(np.uint64)
    return np.asarray(x)


def dev(a, like):
    """numpy array (uint64 scalars / positions, or uint8 ops) -> the memory space of `like`"""
    a = np.ascontiguousarray(a)
    if hasattr(like, "is_cuda"):
        import torch
        t = torch.from_numpy(a if a.dtype == np.uint8 else a.astype(np.uint64).view(np.int64))
        return t.to(like.device)
    return a if a.dtype == np.uint8 else a.astype(np.uint64)


def new_tree(engine, arity, height, max_leaves, mem):
    return merkle.CompactTree(arity, height, max_leaves, engine=engine, device=None if mem == "host" else engine.device)


def buffers(tree):
    return host(tree.keys).copy(), host(tree.values).copy(), host(tree.count).copy()


def assert_tree_is(tree, items):
    levels = co.compact_levels(tree.arity, tree.height, items, mo.c_hash_groups(tree.arity))
    want = co.buffers_of(levels, tree.arity, tree.height, tree.max_leaves)
    got = buffers(tree)
    for g, w, name in zip(got, want, ("keys", "values", "count")):
        assert np.array_equal(g, w), name
    assert len(tree) == len(items)
    assert np.array_equal(host(tree.root), co.root_of(levels))
    return levels


def run(tree, pos, op, vals, async_=False):
    pos = np.asarray(pos, dtype=np.uint64)
    like = tree.values
    if op is None:
        tree.insert(dev(pos, like), dev(vals, like), async_=async_)
    else:
        tree.apply(dev(pos, like), dev(np.asarray(op, dtype=np.uint8), like), dev(vals, like), async_=async_)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height", [(4, 8), (2, 14)])
def test_matches_full_capacity_sparse_tree(engine, mem, arity, height):
    rng = np.random.default_rng(arity * 100 + height)
    cap = arity ** height
    tree = new_tree(engine, arity, height, 3000, mem)
    sparse = merkle.SparseTree(arity, height, cap, engine=engine, device=None if mem == "host" else engine.device)
    for k, n in enumerate((1500, 700, 900, 1, 400)):
        pos = rng.integers(0, cap, n).astype(np.uint64)
        pos[: n // 4] = rng.integers(0, 64, n // 4)               # clusters: shared groups and duplicates
        op = (rng.random(n) < (0.1 if k == 0 else 0.4)).astype(np.uint8)
        vals = random_scalars(rng, n)
        run(tree, pos, op, vals)
        sparse.apply(dev(pos, sparse.leaves), dev(op, sparse.present), dev(vals, sparse.leaves))
        assert engine.last_ctree_rejected() == 0
        keys, values, count = buffers(tree)
        svals = [host(sparse.leaves)] + [host(sparse.nodes)[sparse.level_offset[l]:] for l in range(1, height + 1)]
        spres = host(sparse.present)
        ls = host(sparse.leaves).shape[0]
        sp = [spres[:ls]] + [spres[ls + sparse.level_offset[l]:] for l in range(1, height + 1)]
        for l in range(height + 1):
            width = arity ** (height - l)
            idx = np.flatnonzero(sp[l][:width])
            o, c = tree.level_offset[l], int(count[l])
            assert c == len(idx), (k, l)
            assert np.array_equal(keys[o:o + c], idx.astype(np.uint64)), (k, l)
            assert np.array_equal(values[o:o + c], svals[l][idx]), (k, l)
            end = tree.level_offset[l + 1] if l < height else keys.shape[0]
            assert not keys[o + c:end].any() and not values[o + c:end].any()
        assert np.array_equal(host(tree.root), host(sparse.root))


def edge_positions(arity, height, rng):
    top = arity ** (height - 1)                                   # pairs that share nothing but the root
    return np.array([0, U64, U64 - 1, 1, 2, 3, 4, top, top - 1, (arity - 1) * top, 12345, 12346] +
                    [int(x) for x in rng.integers(0, 1 << 63, 60, dtype=np.uint64) * 2 + 1], dtype=np.uint64)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height", [(4, 32), (2, 64)])
def test_full_position_space_against_oracle(engine, mem, arity, height):
    rng = np.random.default_rng(height)
    tree = new_tree(engine, arity, height, 200, mem)
    items = {}

    def step(pos, op, async_=False):
        nonlocal items
        pos = np.asarray(pos, dtype=np.uint64)
        vals = random_scalars(rng, len(pos)) if len(pos) else np.zeros((0, 4), dtype=np.uint64)
        items = so.apply(items, pos, op, vals)
        run(tree, pos, op, vals, async_=async_)
        if async_:
            engine.sync()
        assert engine.last_ctree_rejected() == 0
        return assert_tree_is(tree, items)

    edge = edge_positions(arity, height, rng)
    step(edge, None)
    step([U64, U64, 0, 0, 7, 7, 7], [0, 1, 1, 0, 0, 0, 0])        # duplicates: the last operation wins
    absent = [p for p in (5, 6, 8, 1 << 40) if p not in items]
    before = buffers(tree)
    step(absent, np.ones(len(absent)))                            # removing absent positions does nothing
    assert all(np.array_equal(a, b) for a, b in zip(before, buffers(tree)))
    step(rng.choice(edge, 40), rng.integers(0, 2, 40), async_=True)
    step([], None)
    levels = step(list(items), np.ones(len(items)))               # remove everything: all-zero buffers
    assert items == {} and not any(b.any() for b in buffers(tree)) and not co.root_of(levels).any()
    step([U64, 0], None)                                          # and back


@pytest.mark.parametrize("mem", MEMS)
def test_present_zero_leaf_is_not_absent(engine, mem):
    rng = np.random.default_rng(3)
    tree = new_tree(engine, 2, 64, 8, mem)
    v = random_scalars(rng, 1)
    run(tree, [9], None, v)
    r1 = host(tree.root).copy()
    run(tree, [U64], None, np.zeros((1, 4), dtype=np.uint64))
    assert len(tree) == 2 and not np.array_equal(host(tree.root), r1)
    assert_tree_is(tree, {9: v[0], U64: np.zeros(4, dtype=np.uint64)})
    run(tree, [U64], [1], np.zeros((1, 4), dtype=np.uint64))
    assert np.array_equal(host(tree.root), r1)


@pytest.mark.parametrize("mem", MEMS)
def test_one_batch_equals_several(engine, mem):
    rng = np.random.default_rng(4)
    pos = rng.integers(0, 1 << 62, 3000, dtype=np.uint64) * 4 + rng.integers(0, 4, 3000, dtype=np.uint64)
    pos[-400:] = pos[:400]                                        # repeats across the chunks
    vals = random_scalars(rng, len(pos))
    one = new_tree(engine, 4, 32, 4000, mem)
    run(one, pos, None, vals)
    many = new_tree(engine, 4, 32, 4000, mem)
    for a in range(0, len(pos), 700):
        run(many, pos[a:a + 700], None, vals[a:a + 700])
    assert all(np.array_equal(a, b) for a, b in zip(buffers(one), buffers(many)))
    assert_tree_is(one, so.apply({}, pos, None, vals))


def test_host_and_device_trees_agree(engine):
    rng = np.random.default_rng(5)
    h = new_tree(engine, 2, 64, 1500, "host")
    d = new_tree(engine, 2, 64, 1500, "device")
    for n in (1000, 500, 800):
        pos = rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2
        pos[: n // 2] = rng.choice(host(h.keys)[: max(len(h), 1)], n // 2)
        op = (rng.random(n) < 0.5).astype(np.uint8)
        vals = random_scalars(rng, n)
        run(h, pos, op, vals)
        run(d, pos, op, vals)
        assert all(np.array_equal(a, b) for a, b in zip(buffers(h), buffers(d)))


@pytest.mark.parametrize("mem", MEMS)
def test_rejections(engine, mem):
    import torch
    rng = np.random.default_rng(6)
    arity, height, ml = 4, 20, 600                                # 4^20 = 2^40 positions: some u64 are out of range
    tree = new_tree(engine, arity, height, ml, mem)
    pad = 64
    if mem == "device":                                           # canaries around every buffer
        for name in ("keys", "values", "count"):
            b = getattr(tree, name)
            big = torch.full((b.shape[0] + 2 * pad,) + tuple(b.shape[1:]), 0x5A5A, dtype=torch.int64, device=b.device)
            big[pad:pad + b.shape[0]] = b
            setattr(tree, "_big_" + name, big)
            setattr(tree, name, big[pad:pad + b.shape[0]])
    pos = rng.integers(0, 1 << 40, 300, dtype=np.uint64)
    vals = random_scalars(rng, 300)
    run(tree, pos, None, vals)
    items = so.apply({}, pos, None, vals)
    before = buffers(tree)
    bad_pos = np.array([3, 1 << 40, (1 << 40) - 1, U64, 7, 1 << 41, 12], dtype=np.uint64)
    bad_op = np.array([0, 0, 1, 1, 2, 0, 0], dtype=np.uint8)
    bvals = random_scalars(rng, len(bad_pos))
    if mem == "host":
        for p_, o_ in ((bad_pos, None), (bad_pos[[0, 4]], bad_op[[0, 4]])):
            with pytest.raises(pb.EngineError):                   # nothing modified
                run(tree, p_, o_, bvals[:len(p_)])
            assert all(np.array_equal(a, b) for a, b in zip(buffers(tree), before))
        return
    run(tree, bad_pos, bad_op, bvals)                             # skipped and counted
    assert engine.last_ctree_rejected() == 4
    keep = [k for k in range(len(bad_pos)) if int(bad_pos[k]) < 1 << 40 and bad_op[k] <= 1]
    items = so.apply(items, bad_pos[keep], bad_op[keep], bvals[keep])
    assert_tree_is(tree, items)
    run(tree, bad_pos, None, bvals, async_=True)                  # no op array: only the positions
    engine.sync()
    assert engine.last_ctree_rejected() == 3
    items = so.apply(items, bad_pos[[0, 2, 4, 6]], None, bvals[[0, 2, 4, 6]])
    assert_tree_is(tree, items)
    for name in ("keys", "values", "count"):
        big = getattr(tree, "_big_" + name)
        assert (big[:pad] == 0x5A5A).all() and (big[-pad:] == 0x5A5A).all(), name


@pytest.mark.parametrize("mem", MEMS)
def test_capacity_overflow_is_refused(engine, mem):
    rng = np.random.default_rng(7)
    tree = new_tree(engine, 2, 64, 100, mem)
    pos = rng.integers(0, 1 << 63, 90, dtype=np.uint64)
    vals = random_scalars(rng, 90)
    run(tree, pos, None, vals)
    items = so.apply({}, pos, None, vals)
    before = buffers(tree)
    more = rng.integers(0, 1 << 63, 11, dtype=np.uint64) | np.uint64(1 << 63)   # 101 present positions
    mvals = random_scalars(rng, 11)
    if mem == "host":
        with pytest.raises(pb.EngineError):
            run(tree, more, None, mvals)
    else:
        run(tree, more, None, mvals)
        assert engine.last_ctree_rejected() == 11                 # the whole batch: the tree is unchanged
    assert all(np.array_equal(a, b) for a, b in zip(buffers(tree), before))
    # removing one first makes the same inserts fit exactly
    run(tree, np.concatenate([pos[:1], more]), np.array([1] + [0] * 11), np.concatenate([vals[:1], mvals]))
    assert engine.last_ctree_rejected() == 0
    items = so.apply(items, np.concatenate([pos[:1], more]), [1] + [0] * 11, np.concatenate([vals[:1], mvals]))
    assert len(items) == 100
    assert_tree_is(tree, items)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height", [(4, 32), (2, 64), (4, 6)])
def test_openings_verify(engine, mem, arity, height):
    rng = np.random.default_rng(8 + height)
    tree = new_tree(engine, arity, height, 1000, mem)
    pos = np.unique(np.concatenate([edge_positions(arity, height, rng) % np.uint64(arity ** height if height < 32 else 1 << 63),
                                    rng.integers(0, min(arity ** height, 1 << 63), 300, dtype=np.uint64)]))
    if height >= 32:
        pos = np.unique(np.concatenate([pos, np.array([U64], dtype=np.uint64)]))
    vals = random_scalars(rng, len(pos))
    vals[0] = 0                                                   # a present zero leaf opens and verifies too
    run(tree, pos, None, vals)
    items = so.apply({}, pos, None, vals)
    levels = co.compact_levels(arity, height, items, mo.c_hash_groups(arity))
    idx = np.concatenate([pos[:5], pos[-3:], rng.choice(pos, 100)]).astype(np.uint64)
    want = co.paths(levels, arity, idx)
    got = tree.open(dev(idx, tree.values))
    assert np.array_equal(host(got), want)
    root = host(tree.root)
    leaf_items = np.stack([items[int(i)] for i in idx])
    ok = engine.merkle_verify_batch(leaf_items, idx, want, root, arity=arity)
    assert ok.all() and engine.last_verify_failures() == 0
    bad_p, bad_i = want.copy(), leaf_items.copy()
    expect = np.ones(len(idx), dtype=bool)
    for t in range(0, len(idx), 4):                               # a sibling slot (absent ones too) at a random level
        lvl = int(rng.integers(0, height))
        p = (int(idx[t]) // arity ** lvl) % arity
        bad_p[t, lvl, (p + 1) % arity, 2] ^= np.uint64(1)
        expect[t] = False
    for t in range(1, len(idx), 4):                               # the leaf item
        bad_i[t, 1] ^= np.uint64(2)
        expect[t] = False
    ok = engine.merkle_verify_batch(bad_i, idx, bad_p, root, arity=arity)
    assert np.array_equal(ok.astype(bool), expect)
    op = tree.opening(int(pos[3]))
    assert op.verify(items[int(pos[3])], engine=engine) and not op.verify(items[int(pos[4])], engine=engine)
    cands = [int(p) ^ 1 for p in pos[5:]] + list(range(1 << 10))  # a sibling of a present leaf first
    absent = np.array([c for c in cands if c not in items][:2], dtype=np.uint64)
    if mem == "host":
        for a in absent:
            with pytest.raises(pb.EngineError):
                tree.open(np.array([a], dtype=np.uint64))
    else:
        both = np.concatenate([absent, idx[:2]])
        got = host(tree.open(dev(both, tree.values)))
        assert not got[:2].any() and np.array_equal(got[2:], want[:2])
    assert tree.contains(int(pos[7])) and not tree.contains(int(absent[0]))


def test_async_update_is_valid_after_sync(engine):
    rng = np.random.default_rng(9)
    tree = new_tree(engine, 4, 32, 5000, "device")
    pos = rng.integers(0, 1 << 63, 4000, dtype=np.uint64)
    vals = random_scalars(rng, 4000)
    run(tree, pos, None, vals, async_=True)
    tree.remove(dev(pos[:100], tree.values), async_=True)
    engine.sync()
    assert engine.last_ctree_rejected() == 0
    assert_tree_is(tree, so.apply(so.apply({}, pos, None, vals), pos[:100], np.ones(100), vals[:100]))


def test_python_front_end(engine):
    rng = np.random.default_rng(10)
    t = pb.CompactTree(2, 64, 400, engine=engine)
    pos = rng.integers(0, 1 << 63, 300, dtype=np.uint64) * 2 + 1
    vals = random_scalars(rng, 300)
    t.insert(pos, vals)
    t.remove(pos[::3])
    assert len(t) == t.len() == 200 and t.contains(int(pos[1])) and not t.contains(int(pos[0]))
    assert not t.contains(-1) and not t.contains(1 << 64)
    keys, values = t.level(0)
    assert np.array_equal(keys, np.sort(np.delete(pos, np.arange(0, 300, 3))))
