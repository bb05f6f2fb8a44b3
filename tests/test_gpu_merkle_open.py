"""GPU (-m gpu): Merkle openings and batch verification (SURVEY.md 8 row f1, second half) against an oracle
recomputation -- arity 4 (4^6 leaves) and arity 2 (2^10 leaves), host and device buffers, tampered siblings,
wrong leaf, wrong index, wrong root.  Node hash = Hash::digest(Domain::Merkle4|Merkle2, children),
src/hash.rs:22-31; opening semantics = poseidon-merkle `Opening` (AGENTS.md:62-66)."""
import numpy as np
import pytest

import poseidon252_b200 as pb
from conftest import mont
from poseidon252_b200 import merkle
from poseidon252_b200.scalar import random_scalars

pytestmark = pytest.mark.gpu


def oracle_tree(coracle, oracle, leaves, arity):
    dom = oracle.Domain.Merkle4 if arity == 4 else oracle.Domain.Merkle2
    tag = mont(oracle.hash_to_scalar(oracle.tag_input([oracle.Absorb(arity), oracle.Squeeze(1)], dom)))
    levels, cur = [leaves], leaves
    while cur.shape[0] > 1:
        cur = coracle.digest(tag, cur.reshape(-1, arity, 4), arity, 1).reshape(-1, 4)
        levels.append(cur)
    return levels                      # levels[0] = leaves, levels[-1] = [root]


def oracle_paths(levels, idx, arity):
    depth = len(levels) - 1
    out = np.zeros((len(idx), depth, arity, 4), dtype=np.uint64)
    for k, i in enumerate(idx):
        i = int(i)
        for l in range(depth):
            g = i // arity
            out[k, l] = levels[l][g * arity:(g + 1) * arity]
            i = g
    return out


def oracle_verify(coracle, oracle, item, idx, path, root, arity):
    dom = oracle.Domain.Merkle4 if arity == 4 else oracle.Domain.Merkle2
    tag = mont(oracle.hash_to_scalar(oracle.tag_input([oracle.Absorb(arity), oracle.Squeeze(1)], dom)))
    cur, i = item, int(idx)
    for l in range(path.shape[0]):
        if not np.array_equal(path[l, i % arity], cur):
            return False
        cur = coracle.digest(tag, path[l].reshape(1, arity, 4), arity, 1).reshape(4)
        i //= arity
    return bool(np.array_equal(cur, root)) and i == 0


@pytest.mark.parametrize("arity,k", [(4, 6), (2, 10)])
def test_open_and_verify_vs_oracle(engine, coracle, oracle, arity, k):
    rng = np.random.default_rng(arity * 100 + k)
    n_leaves = arity ** k
    leaves = random_scalars(rng, n_leaves)
    leaves[5] = 0                                               # an "empty slot" is the zero scalar (src/hash.rs:22-31)
    levels = oracle_tree(coracle, oracle, leaves, arity)
    nodes = engine.merkle_build(leaves, arity=arity)
    assert np.array_equal(nodes, np.concatenate(levels[1:], axis=0))
    root = nodes[-1]
    idx = np.concatenate([np.array([0, 1, 5, n_leaves - 1, n_leaves // 2], dtype=np.uint64),
                          rng.integers(0, n_leaves, size=200, dtype=np.uint64)])
    want = oracle_paths(levels, idx, arity)
    got = engine.merkle_open_batch(leaves, nodes, idx, arity=arity)            # host gather
    assert got.shape == (len(idx), k, arity, 4) and np.array_equal(got, want)
    ok = engine.merkle_verify_batch(leaves[idx.astype(np.int64)], idx, got, root, arity=arity)
    assert ok.dtype == np.uint8 and ok.all() and engine.last_verify_failures() == 0

    # tampering: every kind must be caught, and only on the tampered items
    n = len(idx)
    bad_paths, bad_items, bad_idx = got.copy(), leaves[idx.astype(np.int64)].copy(), idx.copy()
    expect = np.ones(n, dtype=bool)
    for t in range(0, n, 7):                                    # a sibling that is NOT the path node, at a random level
        lvl = int(rng.integers(0, k))
        pos = (int(idx[t]) // arity ** lvl) % arity
        bad_paths[t, lvl, (pos + 1) % arity, 0] ^= np.uint64(1)
        expect[t] = False
    for t in range(1, n, 7):                                    # the path node itself at an upper level
        lvl = int(rng.integers(1, k))
        pos = (int(idx[t]) // arity ** lvl) % arity
        bad_paths[t, lvl, pos, 3] ^= np.uint64(1 << 40)
        expect[t] = False
    for t in range(2, n, 7):                                    # wrong leaf value
        bad_items[t, 1] ^= np.uint64(2)
        expect[t] = False
    for t in range(3, n, 7):                                    # index pointing at a sibling with a different value
        j = int(idx[t]) ^ 1
        if not np.array_equal(leaves[j], leaves[int(idx[t])]):
            bad_idx[t] = j
            expect[t] = False
    ok = engine.merkle_verify_batch(bad_items, bad_idx, bad_paths, root, arity=arity)
    assert np.array_equal(ok.astype(bool), expect)
    assert engine.last_verify_failures() == int((~expect).sum())
    for t in range(0, n, 11):                                   # spot-check the verdicts against the oracle's verify
        assert oracle_verify(coracle, oracle, bad_items[t], bad_idx[t], bad_paths[t], root, arity) == bool(ok[t])
    wrong_root = root.copy()
    wrong_root[0] ^= np.uint64(1)
    assert not engine.merkle_verify_batch(leaves[idx.astype(np.int64)], idx, got, wrong_root, arity=arity).any()
    # index beyond the tree: the residual index is non-zero after `depth` levels
    far = idx.copy()
    far[0] = idx[0] + np.uint64(n_leaves)
    assert not engine.merkle_verify_batch(leaves[idx.astype(np.int64)], far, got, root, arity=arity)[0]


@pytest.mark.parametrize("arity,k", [(4, 5), (2, 9)])
def test_open_verify_device_tensors(engine, arity, k):
    import torch
    rng = np.random.default_rng(77 + arity)
    n_leaves = arity ** k
    leaves = random_scalars(rng, n_leaves)
    nodes = engine.merkle_build(leaves, arity=arity)
    idx = rng.integers(0, n_leaves, size=1000, dtype=np.uint64)
    host_paths = engine.merkle_open_batch(leaves, nodes, idx, arity=arity)
    d_leaves = torch.from_numpy(leaves.view(np.int64)).cuda()
    d_nodes = torch.from_numpy(nodes.view(np.int64)).cuda()
    d_idx = torch.from_numpy(idx.view(np.int64)).cuda()
    d_paths = engine.merkle_open_batch(d_leaves, d_nodes, d_idx, arity=arity)      # k_merkle_open
    assert d_paths.is_cuda and np.array_equal(d_paths.cpu().numpy().view(np.uint64), host_paths)
    d_items = d_leaves[d_idx]
    ok = engine.merkle_verify_batch(d_items, d_idx, d_paths, nodes[-1], arity=arity)
    assert ok.is_cuda and bool(ok.all()) and engine.last_verify_failures() == 0
    # a device index outside the tree: all-zero opening, verification fails
    far = d_idx.clone()
    far[0] = n_leaves + 5
    z = engine.merkle_open_batch(d_leaves, d_nodes, far, arity=arity)
    assert not bool(z[0].any()) and torch.equal(z[1:], d_paths[1:])
    assert not bool(engine.merkle_verify_batch(d_items, far, z, nodes[-1], arity=arity)[0])
    d_paths[3, 1, 0, 0] ^= 1
    d_paths[999, 0, arity - 1, 2] ^= 4
    ok = engine.merkle_verify_batch(d_items, d_idx, d_paths, nodes[-1], arity=arity).cpu().numpy()
    assert not ok[3] and not ok[999] and ok.sum() == 998
    assert engine.last_verify_failures() == 2                   # counted on the device (atomic per warp)


def test_opening_mirror_and_errors(engine):
    rng = np.random.default_rng(5)
    leaves = random_scalars(rng, 64)
    nodes = merkle.merkle4_build(leaves, engine=engine)
    paths = merkle.open_batch(leaves, nodes, np.array([37], dtype=np.uint64), engine=engine)
    op = merkle.Opening(nodes[-1], paths[0], 37)
    assert op.positions == [37 % 4, (37 // 4) % 4, (37 // 16) % 4]
    assert op.verify(leaves[37], engine=engine) and not op.verify(leaves[36], engine=engine)
    with pytest.raises(pb.EngineError):                          # leaf index outside the tree (host buffers are checked)
        engine.merkle_open_batch(leaves, nodes, np.array([64], dtype=np.uint64))
    with pytest.raises(pb.Error):                                # 48 leaves: not a power of the arity
        engine.merkle_open_batch(leaves[:48], nodes, np.array([1], dtype=np.uint64))
    with pytest.raises(pb.EngineError):                          # node array of the wrong size
        engine.merkle_open_batch(leaves, nodes[:-1], np.array([1], dtype=np.uint64))
    assert engine.merkle_open_batch(leaves, nodes, np.zeros(0, dtype=np.uint64)).shape == (0, 3, 4, 4)


def test_merkle_golden(engine, golden):
    """tests/golden: trees + one opening each (oracle-derived, tests/golden/make_golden.py)"""
    from conftest import hx, unmont
    for t in golden["merkle"]:
        arity = t["arity"]
        leaves = mont([hx(v) for v in t["leaves"]])
        nodes = engine.merkle_build(leaves, arity=arity)
        assert ["0x%064x" % v for v in unmont(nodes)] == t["nodes"]
        i = t["opening_leaf"]
        paths = engine.merkle_open_batch(leaves, nodes, np.array([i], dtype=np.uint64), arity=arity)
        assert [["0x%064x" % v for v in unmont(row)] for row in paths[0]] == t["opening"]
        assert engine.merkle_verify_batch(leaves[i:i + 1], np.array([i], dtype=np.uint64), paths, nodes[-1], arity=arity)[0]


def test_verify_host_multi_chunk(engine):
    """80k host openings: several staged chunks (ramp-up sizes, then full chunks) through run_host_pipeline."""
    rng = np.random.default_rng(31)
    leaves = random_scalars(rng, 4 ** 5)
    nodes = engine.merkle_build(leaves, arity=4)
    idx = rng.integers(0, 4 ** 5, size=80_000, dtype=np.uint64)
    paths = engine.merkle_open_batch(leaves, nodes, idx)
    items = leaves[idx.astype(np.int64)]
    bad = rng.choice(80_000, size=300, replace=False)
    items = items.copy()
    items[bad, 0] ^= np.uint64(1)
    ok = engine.merkle_verify_batch(items, idx, paths, nodes[-1])
    expect = np.ones(80_000, dtype=np.uint8)
    expect[bad] = 0
    assert np.array_equal(ok, expect) and engine.last_verify_failures() == 300
