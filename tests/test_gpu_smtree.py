"""GPU (-m gpu): sparse fixed-height trees with inserts and removals at any position (p252_smtree) against the oracle
restatement (tests/smtree_oracle.py) -- builds from garbage, seeded operation sequences, duplicates within a batch,
emptying subtrees and the whole tree, the prefix cross-check against p252_mtree, the untouched-node check, rejections,
openings, the Python / C++ front ends and a full-size tree.  Host and device buffers, both digest kernels (the
two-parameter `engine` fixture)."""
import os
import subprocess

import numpy as np
import pytest

import mtree_oracle as mo
import smtree_oracle as so
import poseidon252_b200 as pb
from poseidon252_b200 import merkle
from poseidon252_b200.scalar import random_scalars

pytestmark = pytest.mark.gpu

MEMS = ["host", "device"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def host(x):
    if hasattr(x, "is_cuda"):
        a = x.cpu().numpy()
        return a if a.dtype == np.uint8 else a.view(np.uint64)
    return np.asarray(x)


def dev(a, like):
    """numpy array (uint64 scalars / indices, or uint8 bytes) -> the memory space of `like`"""
    a = np.ascontiguousarray(a)
    if hasattr(like, "is_cuda"):
        import torch
        t = torch.from_numpy(a if a.dtype == np.uint8 else a.astype(np.uint64).view(np.int64))
        return t.to(like.device)
    return a if a.dtype == np.uint8 else a.astype(np.uint64)


def new_tree(engine, arity, height, capacity, mem):
    return merkle.SparseTree(arity, height, capacity, engine=engine, device=None if mem == "host" else engine.device)


def assert_tree_is(tree, items, engine):
    """leaves, nodes, presence bytes and len equal the oracle over `items`, and a fresh build over the same leaves"""
    levels = so.sparse_tree(tree.arity, tree.height, tree.capacity, items, mo.c_hash_groups(tree.arity))
    leaves, nodes, present = so.buffers_of(levels)
    assert np.array_equal(host(tree.leaves), leaves)
    assert np.array_equal(host(tree.present), present)
    assert np.array_equal(host(tree.nodes), nodes)
    assert len(tree) == len(items)
    assert np.array_equal(host(tree.root), so.root_of(levels))
    fresh = new_tree(engine, tree.arity, tree.height, tree.capacity, "host" if not hasattr(tree.leaves, "is_cuda") else "device")
    fresh.leaves[:] = tree.leaves
    fresh.leaf_present[:] = tree.leaf_present
    fresh.build()
    assert np.array_equal(host(fresh.nodes), nodes) and np.array_equal(host(fresh.present), present)
    return levels


BUILD_CASES = [(4, 1, 4, k) for k in (0, 1, 4)] + [(4, 3, 37, k) for k in (0, 1, 9, 37)] + \
              [(4, 6, 4096, k) for k in (1, 300, 4096)] + [(4, 17, 8300, k) for k in (3, 2000)] + \
              [(2, 12, 4096, k) for k in (1, 777, 4096)]


@pytest.mark.parametrize("mem", MEMS)
def test_build_matches_oracle(engine, mem):
    rng = np.random.default_rng(21)
    for arity, height, capacity, k in BUILD_CASES:
        tree = new_tree(engine, arity, height, capacity, mem)
        pos = rng.choice(capacity, k, replace=False) if k else np.zeros(0, dtype=np.int64)
        vals = random_scalars(rng, tree.leaves.shape[0])
        vals[pos[:1]] = 0                                          # a present leaf of value zero
        flags = np.zeros(tree.leaves.shape[0], dtype=np.uint8)
        flags[pos] = rng.integers(1, 256, k)                      # any non-zero byte is present
        flags[capacity:] = rng.integers(1, 256, tree.leaves.shape[0] - capacity)   # beyond capacity: library-owned
        tree.leaves[:] = dev(vals, tree.leaves)                   # garbage values at absent positions
        tree.leaf_present[:] = dev(flags, tree.present)
        tree.nodes[:] = dev(random_scalars(rng, tree.nodes.shape[0]), tree.nodes)
        tree.node_present[:] = dev(rng.integers(0, 256, tree.nodes.shape[0]).astype(np.uint8), tree.present)
        tree.build()
        assert_tree_is(tree, {int(j): vals[j] for j in pos}, engine)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height,capacity", [(4, 7, 3000), (2, 12, 2500)])
def test_operation_sequence_matches_oracle(engine, mem, arity, height, capacity):
    rng = np.random.default_rng(arity * 1000 + capacity)
    tree = new_tree(engine, arity, height, capacity, mem)
    items = {}

    def step(pos, op, async_=False):
        nonlocal items
        pos = np.asarray(pos, dtype=np.uint64)
        op = None if op is None else np.asarray(op, dtype=np.uint8)
        vals = random_scalars(rng, len(pos)) if len(pos) else np.zeros((0, 4), dtype=np.uint64)
        items = so.apply(items, pos, op, vals)
        if op is None:
            tree.insert(dev(pos, tree.leaves), dev(vals, tree.leaves), async_=async_)
        else:
            tree.apply(dev(pos, tree.leaves), dev(op, tree.present), dev(vals, tree.leaves), async_=async_)
        if async_:
            engine.sync()
        assert engine.last_smtree_rejected() == 0
        assert_tree_is(tree, items, engine)

    step(rng.choice(capacity, 200, replace=False), None)          # inserts only, scattered
    step(rng.integers(0, capacity, 300), rng.integers(0, 2, 300))  # mixed, with overwrites and absent removals
    p = [5, 5, 9, 9, 11, 11, 11, 13, 13]                          # insert->remove, remove->insert, repeated inserts
    step(p, [0, 1, 1, 0, 0, 0, 0, 1, 1])
    absent = [j for j in range(capacity) if j not in items][:50]
    step(absent, np.ones(50))                                     # removals of absent positions: nothing changes
    step(rng.integers(0, capacity, 500), rng.integers(0, 2, 500), async_=True)
    step([], None)
    sub = arity ** 3                                              # empty the whole level-3 subtree 1
    step(range(sub, 2 * sub), [0] * (sub // 2) + [1] * (sub - sub // 2))
    step(range(sub, 2 * sub), np.ones(sub))
    assert not any(sub <= j < 2 * sub for j in items)
    step(sorted(items), np.ones(len(items)))                      # the whole tree
    assert items == {} and not host(tree.nodes).any() and not host(tree.present).any() and not host(tree.leaves).any()
    step([capacity - 1, 0], None)                                 # and back


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height,capacity,n", [(4, 6, 3000, 1000), (2, 12, 4096, 777)])
def test_prefix_equals_mtree(engine, mem, arity, height, capacity, n):
    rng = np.random.default_rng(22 + n)
    leaves = random_scalars(rng, n + 300)
    dense = merkle.Tree(arity, height, capacity, engine=engine, device=None if mem == "host" else engine.device)
    dense.extend(dev(leaves[:n], dense.leaves))
    tree = new_tree(engine, arity, height, capacity, mem)
    tree.leaves[:n] = dev(leaves[:n], tree.leaves)
    tree.leaf_present[:n] = 1
    tree.build()
    assert np.array_equal(host(tree.leaves), host(dense.leaves)) and np.array_equal(host(tree.nodes), host(dense.nodes))
    idx = rng.integers(0, n, 200)
    vals = random_scalars(rng, 200)
    dense.update(dev(idx, dense.leaves), dev(vals, dense.leaves))
    dense.extend(dev(leaves[n:], dense.leaves))
    tree.insert(dev(np.concatenate([idx, np.arange(n, n + 300)]), tree.leaves), dev(np.concatenate([vals, leaves[n:]]), tree.leaves))
    assert np.array_equal(host(tree.leaves), host(dense.leaves)) and np.array_equal(host(tree.nodes), host(dense.nodes))
    assert len(tree) == n + 300


def test_only_touched_paths_are_rewritten(engine):
    import torch
    rng = np.random.default_rng(23)
    arity, height, capacity = 4, 6, 4096
    tree = new_tree(engine, arity, height, capacity, "device")
    pos = rng.choice(capacity, 2000, replace=False)
    vals = random_scalars(rng, 2000)
    tree.insert(dev(pos, tree.leaves), dev(vals, tree.leaves))
    items = so.apply({}, pos, None, vals)
    off = tree.level_offset
    far = off[2] + 150                                            # level-2 node 150 (leaves 2400..2415): off every path
    sentinel = torch.full((4,), 0x1234, dtype=torch.int64, device=tree.nodes.device)
    saved = tree.nodes[far].clone()
    tree.nodes[far] = sentinel
    ops_pos = np.array([5, 700, 701, 2999, 4095, 64], dtype=np.uint64)
    ops = np.array([0, 1, 0, 1, 0, 1], dtype=np.uint8)
    vals2 = random_scalars(rng, len(ops_pos))
    tree.apply(dev(ops_pos, tree.leaves), dev(ops, tree.present), dev(vals2, tree.leaves))
    items = so.apply(items, ops_pos, ops, vals2)
    assert torch.equal(tree.nodes[far], sentinel)                 # no full rebuild, no over-wide dirty set
    tree.nodes[far] = saved
    assert_tree_is(tree, items, engine)


@pytest.mark.parametrize("mem", MEMS)
def test_rejections(engine, mem):
    rng = np.random.default_rng(24)
    tree = new_tree(engine, 4, 6, 600, mem)
    pos = rng.choice(600, 300, replace=False)
    vals = random_scalars(rng, 300)
    tree.insert(dev(pos, tree.leaves), dev(vals, tree.leaves))
    items = so.apply({}, pos, None, vals)
    before = [host(b).copy() for b in (tree.leaves, tree.nodes, tree.present)]
    bad_pos = np.array([3, 600, 599, 10 ** 12, 7, 640, 12], dtype=np.uint64)
    bad_op = np.array([0, 0, 1, 1, 2, 0, 0], dtype=np.uint8)        # positions >= capacity, an op of 2
    vals = random_scalars(rng, len(bad_pos))
    if mem == "host":
        for p_, o_ in ((bad_pos, None), (bad_pos[[0, 4]], bad_op[[0, 4]])):
            with pytest.raises(pb.EngineError):                   # nothing modified
                tree.apply(p_, o_, vals[:len(p_)]) if o_ is not None else tree.insert(p_, vals[:len(p_)])
            assert all(np.array_equal(host(b), c) for b, c in zip((tree.leaves, tree.nodes, tree.present), before))
        return
    tree.apply(dev(bad_pos, tree.leaves), dev(bad_op, tree.present), dev(vals, tree.leaves))   # skipped and counted
    assert engine.last_smtree_rejected() == 4
    keep = [k for k in range(len(bad_pos)) if int(bad_pos[k]) < 600 and bad_op[k] <= 1]
    items = so.apply(items, bad_pos[keep], bad_op[keep], vals[keep])
    assert_tree_is(tree, items, engine)
    tree.apply(dev(bad_pos, tree.leaves), dev(bad_op, tree.present), dev(vals, tree.leaves), async_=True)
    engine.sync()
    assert engine.last_smtree_rejected() == 4
    tree.insert(dev(bad_pos, tree.leaves), dev(vals, tree.leaves), async_=True)   # no op array: only the positions
    engine.sync()
    assert engine.last_smtree_rejected() == 3
    assert_tree_is(tree, so.apply(items, bad_pos[[0, 2, 4, 6]], None, vals[[0, 2, 4, 6]]), engine)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity,height,capacity,k", [(4, 6, 4096, 1000), (2, 12, 4096, 300), (4, 9, 5000, 4000)])
def test_openings_verify(engine, mem, arity, height, capacity, k):
    rng = np.random.default_rng(25 + k)
    tree = new_tree(engine, arity, height, capacity, mem)
    pos = rng.choice(capacity, k, replace=False)
    vals = random_scalars(rng, k)
    vals[0] = 0                                                   # a present zero leaf opens and verifies too
    tree.insert(dev(pos, tree.leaves), dev(vals, tree.leaves))
    items = so.apply({}, pos, None, vals)
    levels = so.sparse_tree(arity, height, capacity, items, mo.c_hash_groups(arity))
    idx = np.concatenate([pos[:5], rng.choice(pos, 120)]).astype(np.uint64)
    want = so.paths(levels, arity, idx)
    got = tree.open(dev(idx, tree.leaves))
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
    absent = np.array([next(j for j in range(capacity) if j not in items), capacity, capacity + 7], dtype=np.uint64)
    if mem == "host":
        for a in absent:
            with pytest.raises(pb.EngineError):
                tree.open(np.array([a], dtype=np.uint64))
    else:
        both = np.concatenate([absent, idx[:2]])
        got = host(tree.open(dev(both, tree.leaves)))
        assert not got[:3].any() and np.array_equal(got[3:], want[:2])


def test_python_and_cpp_front_ends(engine):
    rng = np.random.default_rng(26)
    vals = random_scalars(rng, 300)
    t = pb.SparseTree(4, 8, 5000, engine=engine)
    pos = np.arange(300, dtype=np.uint64) * 7 + 3
    t.insert(pos, vals)
    t.remove(pos[::3])
    items = so.apply({}, pos[1::3], None, vals[1::3])
    items.update(so.apply({}, pos[2::3], None, vals[2::3]))
    assert_tree_is(t, items, engine)
    assert len(t) == t.len() == 200 and t.contains(10) and not t.contains(3) and not t.contains(10 ** 9)
    # the C++ SparseTree (include/poseidon252_b200.hpp) on the same values: it prints its root
    libdir = os.path.join(ROOT, "poseidon252_b200", "lib")
    exe = os.path.join(ROOT, "tests", "cpp", "smtree_mirror_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "smtree_mirror_test.cpp"), "-o", exe,
                           "-L", libdir, "-lposeidon252_b200", "-Wl,-rpath," + libdir])
    inp = "\n".join(" ".join(str(int(v)) for v in row) for row in vals)
    res = subprocess.run([exe], input=inp, capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    got = np.array([int(v) for v in res.stdout.split("root")[1].split()[:4]], dtype=np.uint64)
    assert np.array_equal(got, t.root)


def test_full_size_device_update(engine):
    """capacity 2^22, height 17, 2^20 random present positions; 2^16 mixed operations in one call == a fresh build
    (compared on the device), the touched leaves follow the last operation, and 64 dirty leaf-to-root paths are
    recomputed with the C oracle."""
    import torch
    arity, height, capacity, n = 4, 17, 1 << 22, 1 << 20
    rng = np.random.default_rng(27)
    g = torch.Generator(device="cuda")
    g.manual_seed(27)

    def scalars(k):
        a = torch.randint(-(1 << 63), (1 << 63) - 1, (k, 4), dtype=torch.int64, device="cuda", generator=g)
        a[:, 3] = torch.randint(0, 0x73EDA753299D7D48, (k,), dtype=torch.int64, device="cuda", generator=g)
        return a

    tree = new_tree(engine, arity, height, capacity, "device")
    present = rng.choice(capacity, n, replace=False)
    pt = torch.from_numpy(present).cuda()
    tree.leaves[pt] = scalars(n)
    tree.leaf_present[pt] = 1
    tree.build()
    assert len(tree) == n
    n_ops = 1 << 16
    pos = np.where(rng.random(n_ops) < 0.5, rng.choice(present, n_ops), rng.integers(0, capacity, n_ops)).astype(np.int64)
    op = (rng.random(n_ops) < 0.4).astype(np.uint8)
    vals = scalars(n_ops)
    tree.apply(torch.from_numpy(pos).cuda(), torch.from_numpy(op).cuda(), vals)
    assert engine.last_smtree_rejected() == 0
    fresh = new_tree(engine, arity, height, capacity, "device")
    fresh.leaves.copy_(tree.leaves)
    fresh.leaf_present.copy_(tree.leaf_present)
    fresh.build()
    assert torch.equal(fresh.nodes, tree.nodes) and torch.equal(fresh.present, tree.present)
    assert torch.equal(fresh.leaves, tree.leaves)
    last = {}
    for k, p in enumerate(pos):
        last[int(p)] = k
    keys = np.array(sorted(last), dtype=np.int64)
    lk = np.array([last[int(p)] for p in keys])
    ins = op[lk] == 0
    kt = torch.from_numpy(keys).cuda()
    assert np.array_equal(host(tree.leaf_present[kt]), ins.astype(np.uint8))
    want = vals[torch.from_numpy(lk).cuda()].clone()
    want[torch.from_numpy(~ins).cuda()] = 0
    assert torch.equal(tree.leaves[kt], want)
    pres_model = np.zeros(capacity, dtype=bool)
    pres_model[present] = True
    pres_model[keys] = ins
    assert len(tree) == int(pres_model.sum())
    hg = mo.c_hash_groups(arity)
    off = tree.level_offset
    below, below_p = tree.leaves, tree.leaf_present
    node_p = tree.node_present
    cur = rng.choice(keys, 64)
    for l in range(1, height + 1):
        grp_i = cur // arity
        slots = torch.from_numpy((grp_i[:, None] * arity + np.arange(arity)[None, :]).reshape(-1)).cuda()
        grp = host(below[slots]).reshape(-1, arity, 4)
        gp = host(below_p[slots]).reshape(-1, arity).any(axis=1)
        gt = torch.from_numpy(grp_i).cuda()
        got = host(tree.nodes[off[l]:][gt])
        got_p = host(node_p[off[l]:][gt])
        assert np.array_equal(got_p, gp.astype(np.uint8)), l
        assert not got[~gp].any(), l
        if gp.any():
            assert np.array_equal(hg(np.ascontiguousarray(grp[gp])), got[gp]), l
        below, below_p, cur = tree.nodes[off[l]:], node_p[off[l]:], grp_i
