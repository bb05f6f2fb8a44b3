"""GPU (-m gpu): every entry point that runs the Hades permutation, on the constructed edge states of
tests/hades_edges.py, bit for bit against the C oracle.

The states drive the scaled-lazy formulation through stored u == p (a true zero), u = s + p, u = p - 1, true values
+-1 at every round and lane, the first add's conditional subtraction at exactly p, and a final value == p (an output
lane 0).  Random batches of any size never reach these sites (tests/test_hades_edges.py checks on the model that the
corpus does).  Both digest kernels run every test (the two-parameter `engine` fixture); raw permutes run on host and
device buffers, out of place and in place, with the dense formulation, and tiled to a batch that takes the 256 x 2
kernel."""
import numpy as np
import pytest

import c_oracle
import ctree_oracle as co
import hades_edges as he
import mtree_oracle as mo
import smtree_oracle as so
from conftest import mont
from poseidon252_b200 import merkle
from poseidon252_b200.scalar import random_limbs_fast
from test_gpu_device_path import (NONCANONICAL, SENTINEL, TH, WIDE, _np, assert_guards, assert_items_equal, guarded_in,
                                  guarded_out, truncated)

import poseidon252_b200 as pb

pytestmark = pytest.mark.gpu

MEMS = ["host", "device"]


def to_mem(a, mem):
    a = np.ascontiguousarray(a)
    if mem == "host":
        return a if a.dtype == np.uint8 else a.astype(np.uint64)
    import torch
    return torch.from_numpy(a if a.dtype == np.uint8 else a.astype(np.uint64).view(np.int64)).cuda()


def host(x):
    if hasattr(x, "is_cuda"):
        a = x.cpu().numpy()
        return a.view(np.uint64) if a.dtype == np.int64 else a
    return np.asarray(x)


def raw_states():
    return mont([c.x for c in he.raw_corpus()]).reshape(-1, 5, 4)


def raw_want():
    return c_oracle.permute(raw_states(), threads=TH)


# ---- raw permute ---------------------------------------------------------------------------------------------------------
def test_permute_host(engine):
    x, want = raw_states(), raw_want()
    for dense in (False, True):
        assert_items_equal(engine.permute_batch(x, dense=dense), want, "host permute (dense=%s)" % dense)
    y = x.copy()
    engine.permute_batch_inplace(y)
    assert_items_equal(y, want, "host in-place permute")


def test_permute_device(engine):
    x, want = raw_states(), raw_want()
    n = x.shape[0]
    xbuf, xd = guarded_in(x)
    for dense in (False, True):
        obuf, od = guarded_out((n, 5, 4))
        assert engine.permute_batch(xd, dense=dense, out=od) is od
        assert_items_equal(_np(od), want, "device permute (dense=%s)" % dense)
        assert_guards(obuf, n, SENTINEL)
    assert np.array_equal(_np(xd), x)
    engine.permute_batch_inplace(xd)
    assert_items_equal(_np(xd), want, "device in-place permute")
    assert_guards(xbuf, n, NONCANONICAL)


def test_permute_wide_tile(engine):
    """The corpus tiled to P252_WIDE_SHAPE_MIN + 289 states: the 256 x 2 kernel, ragged last block."""
    import torch
    x, want = raw_states(), raw_want()
    n = WIDE + 289
    d = torch.from_numpy(np.resize(x, (n, 5, 4)).view(np.int64)).cuda()
    got = _np(engine.permute_batch(d))
    assert_items_equal(got, np.resize(want, (n, 5, 4)), "256 x 2 permute of the tiled corpus")


# ---- digests -------------------------------------------------------------------------------------------------------------
SHAPES = ["%s-%d-%d" % s for s in he.DIGEST_SHAPES]


def corpus_of(shape):
    dom, a, b = shape.split("-")
    return he.digest_corpus(dom, int(a), int(b))


def digest_want(c):
    return c_oracle.digest(mont(c.tag), mont(c.data).reshape(-1, c.in_len, 4), c.in_len, c.out_len)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("shape", SHAPES)
def test_digest(engine, mem, shape):
    c = corpus_of(shape)
    x = mont(c.data).reshape(-1, c.in_len, 4)
    got = engine.hash_batch(getattr(pb.Domain, c.domain), to_mem(x, mem), c.out_len)
    assert_items_equal(host(got), digest_want(c), "%s digests (%s)" % (shape, mem))


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("shape", [s for s in SHAPES if s.startswith("Other")])
def test_digest_truncated(engine, mem, shape):
    c = corpus_of(shape)
    x = mont(c.data).reshape(-1, c.in_len, 4)
    got = engine.hash_batch_truncated(pb.Domain.Other, to_mem(x, mem), c.out_len)
    assert_items_equal(host(got), truncated(digest_want(c)), "%s truncated digests (%s)" % (shape, mem))


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("shape", ["Other-3-1", "Other-8-5"])
def test_digest_varlen(engine, mem, shape):
    """Crafted items of one length interleaved with random items of the other lengths 1..12."""
    c = corpus_of(shape)
    crafted = mont(c.data).reshape(-1, c.in_len, 4)
    rng = np.random.default_rng([c.in_len, c.out_len, 8])
    others = [L for L in range(1, 13) if L != c.in_len]
    items = []
    for k in range(crafted.shape[0]):
        items.append(random_limbs_fast(rng, others[k % len(others)]))
        items.append(crafted[k])
    lens = np.array([it.shape[0] for it in items])
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    data = np.concatenate(items)
    got = host(engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, mem), to_mem(offsets, mem), c.out_len))
    assert engine.last_varlen_rejected() == 0
    assert_items_equal(got[1::2], digest_want(c), "crafted varlen digests (%s)" % mem)
    for L in others:
        sel = [i for i in range(0, len(items), 2) if lens[i] == L]
        if sel:
            tag = mont(he.hash_tag(he.o.Domain.Other, L, c.out_len))
            want = c_oracle.digest(tag, np.stack([items[i] for i in sel]), L, c.out_len)
            assert_items_equal(got[sel], want, "random varlen digests of length %d (%s)" % (L, mem))


# ---- trees ---------------------------------------------------------------------------------------------------------------
def merkle_corpus(arity):
    return he.digest_corpus("Merkle%d" % arity, arity, 1)


def crafted_groups(arity):
    """(k, arity, 4) leaf groups whose node hash reaches the edges."""
    return mont(merkle_corpus(arity).data).reshape(-1, arity, 4)


def spread_groups(k, n_groups, rng):
    """k distinct group indices spread over [0, n_groups), sorted."""
    return np.sort(rng.choice(n_groups, size=k, replace=False))


def leaf_positions(groups, arity):
    return (groups.astype(np.int64)[:, None] * arity + np.arange(arity)).reshape(-1).astype(np.uint64)


def verify_openings(engine, leaves, pos, paths, root, arity, mem):
    """The openings verify, and with the leaf items rotated by one (every item the wrong leaf) none does."""
    ok = host(engine.merkle_verify_batch(to_mem(leaves, mem), to_mem(pos, mem), to_mem(paths, mem), root, arity=arity))
    assert ok.all(), "%d of %d openings of crafted leaves fail" % (int((ok == 0).sum()), ok.shape[0])
    bad = np.roll(leaves, 1, axis=0)
    same = (bad == leaves).all(axis=1)
    ok = host(engine.merkle_verify_batch(to_mem(bad, mem), to_mem(pos, mem), to_mem(paths, mem), root, arity=arity))
    assert not ok[~same].any()


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity", [2, 4])
def test_merkle_build_and_openings(engine, mem, arity):
    g = crafted_groups(arity)
    depth = 4 if arity == 4 else 6                             # 256 / 64 leaves
    n = arity ** depth
    rng = np.random.default_rng([arity, 11])
    leaves = random_limbs_fast(rng, n).reshape(n, 4)
    groups = spread_groups(g.shape[0], n // arity, rng)
    pos = leaf_positions(groups, arity)
    leaves[pos] = g.reshape(-1, 4)
    nodes = host(engine.merkle_build(to_mem(leaves, mem), arity=arity))
    levels = mo.fixed_tree(arity, depth, leaves, mo.c_hash_groups(arity))
    assert_items_equal(nodes, np.concatenate(levels[1:]), "tree nodes (%s)" % mem)
    want = c_oracle.digest(mont(merkle_corpus(arity).tag), g, arity, 1).reshape(-1, 4)
    assert_items_equal(nodes[groups], want, "crafted parents (%s)" % mem)
    paths = host(engine.merkle_open_batch(to_mem(leaves, mem), to_mem(nodes, mem), to_mem(pos, mem), arity=arity))
    assert_items_equal(paths, mo.paths(levels, arity, pos), "openings (%s)" % mem)
    verify_openings(engine, leaves[pos], pos, paths, nodes[-1], arity, mem)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity", [2, 4])
def test_mtree_update(engine, mem, arity):
    g = crafted_groups(arity)
    height, cap = (4, 200) if arity == 4 else (7, 100)
    rng = np.random.default_rng([arity, 12])
    tree = merkle.Tree(arity, height, cap, engine=engine, device=None if mem == "host" else engine.device)
    model = random_limbs_fast(rng, cap - 3).reshape(-1, 4)
    tree.extend(to_mem(model, mem))
    groups = spread_groups(g.shape[0], model.shape[0] // arity, rng)
    pos = leaf_positions(groups, arity)
    tree.update(to_mem(pos, mem), to_mem(g.reshape(-1, 4), mem))
    assert engine.last_update_rejected() == 0
    model[pos] = g.reshape(-1, 4)
    levels = mo.fixed_tree(arity, height, model, mo.c_hash_groups(arity))
    want_leaves, want_nodes = mo.layout_of(levels, arity, height, cap)
    assert tree.n_leaves == model.shape[0]
    assert np.array_equal(host(tree.leaves), want_leaves)
    assert_items_equal(host(tree.nodes), want_nodes, "mtree nodes (%s)" % mem)
    paths = host(tree.open(to_mem(pos, mem)))
    assert_items_equal(paths, mo.paths(levels, arity, pos), "mtree openings (%s)" % mem)
    verify_openings(engine, model[pos], pos, paths, mo.root_of(levels), arity, mem)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity", [2, 4])
def test_smtree_update(engine, mem, arity):
    g = crafted_groups(arity)
    height, cap = (4, 256) if arity == 4 else (8, 256)
    rng = np.random.default_rng([arity, 13])
    tree = merkle.SparseTree(arity, height, cap, engine=engine, device=None if mem == "host" else engine.device)
    groups = spread_groups(g.shape[0], cap // arity, rng)
    pos = leaf_positions(groups, arity)
    single = np.setdiff1d(rng.choice(cap, size=9, replace=False), pos)          # lone random leaves beside them
    all_pos = np.concatenate([pos, single.astype(np.uint64)])
    vals = np.concatenate([g.reshape(-1, 4), random_limbs_fast(rng, single.shape[0]).reshape(-1, 4)])
    tree.insert(to_mem(all_pos, mem), to_mem(vals, mem))
    assert engine.last_smtree_rejected() == 0
    items = {int(p): v for p, v in zip(all_pos, vals)}
    levels = so.sparse_tree(arity, height, cap, items, mo.c_hash_groups(arity))
    leaves, nodes, present = so.buffers_of(levels)
    assert np.array_equal(host(tree.leaves), leaves) and np.array_equal(host(tree.present), present)
    assert_items_equal(host(tree.nodes), nodes, "smtree nodes (%s)" % mem)
    paths = host(tree.open(to_mem(pos, mem)))
    assert_items_equal(paths, so.paths(levels, arity, pos), "smtree openings (%s)" % mem)
    verify_openings(engine, g.reshape(-1, 4), pos, paths, so.root_of(levels), arity, mem)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("arity", [2, 4])
def test_ctree_update(engine, mem, arity):
    g = crafted_groups(arity)
    height = 40 if arity == 2 else 20
    rng = np.random.default_rng([arity, 14])
    tree = merkle.CompactTree(arity, height, 256, engine=engine, device=None if mem == "host" else engine.device)
    groups = np.unique(rng.integers(0, arity ** (height - 1), size=g.shape[0], dtype=np.uint64))
    assert groups.shape[0] == g.shape[0]
    pos = leaf_positions(groups, arity)
    tree.insert(to_mem(pos, mem), to_mem(g.reshape(-1, 4), mem))
    assert engine.last_ctree_rejected() == 0
    items = {int(p): v for p, v in zip(pos, g.reshape(-1, 4))}
    levels = co.compact_levels(arity, height, items, mo.c_hash_groups(arity))
    keys, values, count = co.buffers_of(levels, arity, height, 256)
    assert np.array_equal(host(tree.keys), keys) and np.array_equal(host(tree.count), count)
    assert_items_equal(host(tree.values), values, "ctree values (%s)" % mem)
    paths = host(tree.open(to_mem(pos, mem)))
    assert_items_equal(paths, co.paths(levels, arity, pos), "ctree openings (%s)" % mem)
    verify_openings(engine, g.reshape(-1, 4), pos, paths, co.root_of(levels), arity, mem)


# ---- encryption ----------------------------------------------------------------------------------------------------------
def crypt_inputs(L):
    c = he.crypt_corpus(L)
    n = len(c.cases)
    msg = mont(c.messages).reshape(n, L, 4)
    uv = mont([k.data[:2] for k in c.cases]).reshape(n, 2, 4)
    nonce = mont([k.data[2] for k in c.cases]).reshape(n, 4)
    return c, msg, uv, nonce


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("L", [1, 3])
def test_crypt(engine, mem, L):
    c, msg, uv, nonce = crypt_inputs(L)
    want = c_oracle.encrypt(mont(c.tag), msg, L, uv, nonce)
    cipher = host(engine.encrypt_batch(to_mem(msg, mem), to_mem(uv, mem), to_mem(nonce, mem)))
    assert_items_equal(cipher, want, "ciphers (%s)" % mem)
    m, ok = engine.decrypt_batch(to_mem(cipher, mem), to_mem(uv, mem), to_mem(nonce, mem))
    assert host(ok).all() and np.array_equal(host(m), msg)
    bad = cipher.copy()
    bad[:, L] = np.roll(cipher[:, L], 1, axis=0)                   # every item carries another item's authentication
    m, ok = engine.decrypt_batch(to_mem(bad, mem), to_mem(uv, mem), to_mem(nonce, mem))
    assert not host(ok).any() and engine.last_decrypt_failures() == bad.shape[0]


@pytest.mark.parametrize("mem", MEMS)
def test_crypt_varlen(engine, mem):
    """The crafted L = 1 and L = 3 encryptions interleaved with random messages of lengths 2 and 4..9."""
    rng = np.random.default_rng(15)
    parts = []                                                     # (message (L, 4), uv (2, 4), nonce (4,))
    for L in (1, 3):
        c, msg, uv, nonce = crypt_inputs(L)
        for k in range(msg.shape[0]):
            r = [2, 4, 5, 6, 7, 8, 9][k % 7]
            parts.append((random_limbs_fast(rng, r), random_limbs_fast(rng, 2), random_limbs_fast(rng, 1)[0]))
            parts.append((msg[k], uv[k], nonce[k]))
    lens = np.array([p[0].shape[0] for p in parts])
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    data = np.concatenate([p[0] for p in parts])
    uv = np.stack([p[1] for p in parts])
    nonce = np.stack([p[2] for p in parts])
    cipher, coff = engine.encrypt_batch_varlen(to_mem(data, mem), to_mem(offsets, mem), to_mem(uv, mem), to_mem(nonce, mem))
    cipher, coff = host(cipher), host(coff).astype(np.int64)
    assert engine.last_crypt_rejected() == 0
    for L in np.unique(lens):
        sel = np.nonzero(lens == L)[0]
        want = c_oracle.encrypt(mont(he.crypt_tag(int(L))), np.stack([parts[i][0] for i in sel]), int(L), uv[sel],
                                nonce[sel])
        assert_items_equal(cipher[coff[sel][:, None] + np.arange(L + 1)], want, "varlen ciphers of length %d" % L)
    m, moff, ok = engine.decrypt_batch_varlen(to_mem(cipher, mem), to_mem(coff.astype(np.uint64), mem), to_mem(uv, mem),
                                              to_mem(nonce, mem))
    assert host(ok).all() and np.array_equal(host(m)[:data.shape[0]], data)
    bad = cipher.copy()
    last = coff[1:] - 1                                            # each item's authentication scalar
    bad[last] = np.roll(cipher[last], 1, axis=0)
    m, moff, ok = engine.decrypt_batch_varlen(to_mem(bad, mem), to_mem(coff.astype(np.uint64), mem), to_mem(uv, mem),
                                              to_mem(nonce, mem))
    assert not host(ok).any()
