"""Device buffers (CUDA tensors) on every digest / permute launch shape, against the C oracle.

A: the fixed-length entry points on device tensors at small and medium batch sizes (both the lane-split small-batch
   kernel and the 128 x 5 kernel, through the shared `engine` fixture).  Every output is a slice of a larger tensor
   whose guard rows hold a sentinel, and every input a slice whose guard rows hold non-canonical scalars, so a store
   past the batch, or a read outside it, is caught.
B: batches of at least P252_WIDE_SHAPE_MIN items on device tensors, which take the 256 x 2 digest and permute kernels
   (the shape `bench.py` times).  Host buffers never reach that shape (see C), so the host path is an independent
   second shape to compare every item with.
C: (CPU) the source constants that keep host chunks below the wide-shape threshold, so that B keeps comparing two
   different shapes."""
import ctypes
import functools
import os
import re

import c_oracle
import numpy as np
import pytest

import poseidon252_b200 as pb
from conftest import ROOT, edge_and_random_scalars, mont
from poseidon252_b200 import _native
from poseidon252_b200.scalar import from_mont, random_limbs_fast

KERNELS_CU = os.path.join(ROOT, "poseidon252_b200", "csrc", "kernels.cu")
CAPI_CU = os.path.join(ROOT, "poseidon252_b200", "csrc", "capi.cu")


def source_constant(path, name):
    """The value of `#define NAME expr` or `NAME = expr` in a C++ source, expr an integer literal or `a << b`."""
    with open(path) as f:
        src = f.read()
    pat = r"(?:#define\s+%s\s+|\b%s\s*=\s*)\(?\s*(\d+)[uUlL]*\s*(?:<<\s*(\d+))?\s*\)?" % (name, name)
    found = re.findall(pat, src)
    assert len(found) == 1, "expected one definition of %s in %s, found %d" % (name, path, len(found))
    base, shift = found[0]
    return int(base) << int(shift or 0)


WIDE = source_constant(KERNELS_CU, "P252_WIDE_SHAPE_MIN")   # digest / permute batches from here on run 256 x 2
TH = min(8, os.cpu_count() or 1)
G = 32                                    # guard rows on each side of every device batch
SENTINEL = 0x5A5A5A5A5A5A5A5A             # what output guard rows hold
OK_SENTINEL = 0x5A
NONCANONICAL = -1                         # every limb 0xFF..FF: what input guard rows hold
M64 = (1 << 64) - 1


# ---- helpers -------------------------------------------------------------------------------------------------------
def _tag(oracle, pattern, dom):
    return mont(oracle.hash_to_scalar(oracle.tag_input(pattern, dom)))


def _hash_tag(oracle, dom, in_len, out_len):
    return _tag(oracle, [oracle.Absorb(in_len), oracle.Squeeze(out_len)], getattr(oracle.Domain, dom))


def _crypt_tag(oracle, L):
    return _tag(oracle, [oracle.Absorb(2), oracle.Absorb(1), oracle.Squeeze(L), oracle.Absorb(L), oracle.Squeeze(1)],
                oracle.Domain.Encryption)


def _edge_scalars():
    import hades_oracle as o
    # the hand-picked values of edge_and_random_scalars (0, 1, p-1, p-2, R mod p, 2^254, ...) and the KAT inputs
    return edge_and_random_scalars(np.random.default_rng(0), 11 + len(o.kat_inputs()))


def edge_rows(n):
    """Item 0, the last item, and both sides of the last two 256-item block boundaries below n."""
    rows = {0, n - 1}
    last = (n - 1) // 256 * 256
    for b in (last, last - 256):
        if b > 0:
            rows |= {b - 1, b}
    return sorted(rows)


def plant_edges(a):
    """a (n, k, 4) uint64: every scalar of the rows edge_rows(n) becomes an edge value (each row a different rotation of
    the list).  Random batches never hold them: random_limbs_fast keeps the top limb below p's."""
    e = _edge_scalars()
    k = a.shape[1]
    for j, r in enumerate(edge_rows(a.shape[0])):
        a[r] = e[(j * k + np.arange(k)) % len(e)]
    return a


def _np(t):
    return t.cpu().numpy().view(np.uint64)


def guarded_in(host):
    """host (n, ...) uint64 -> (buffer, view): a CUDA buffer holding host in rows G..G+n and non-canonical scalars in
    the G rows on either side, and the contiguous view of the n batch rows."""
    import torch
    n = host.shape[0]
    buf = torch.full((n + 2 * G,) + host.shape[1:], NONCANONICAL, dtype=torch.int64, device="cuda")
    buf[G:G + n] = torch.from_numpy(np.ascontiguousarray(host).view(np.int64)).cuda()
    return buf, buf[G:G + n]


def guarded_out(shape, dtype=None):
    """-> (buffer, view): a CUDA buffer of shape[0] + 2G rows filled with the sentinel, and the view of the middle rows."""
    import torch
    dtype = torch.int64 if dtype is None else dtype
    fill = OK_SENTINEL if dtype == torch.uint8 else SENTINEL
    n = shape[0]
    buf = torch.full((n + 2 * G,) + tuple(shape[1:]), fill, dtype=dtype, device="cuda")
    return buf, buf[G:G + n]


def assert_guards(buf, n, fill):
    a = buf.cpu().numpy().reshape(buf.shape[0], -1)
    same = (a == fill).all(axis=1)
    bad = [int(r) - G for r in np.nonzero(~same)[0] if r < G or r >= G + n]
    assert not bad, "guard rows at %s (relative to item 0 of the %d-item batch) changed" % (bad[:8], n)


def assert_items_equal(got, want, what):
    if not np.array_equal(got, want):
        diff = np.nonzero((got != want).reshape(got.shape[0], -1).any(axis=1))[0]
        raise AssertionError("%s: %d of %d items differ, first at %s" % (what, diff.size, got.shape[0], diff[:8].tolist()))


def truncated(digests):
    """Hash::finalize_truncated of oracle digests: the canonical value masked to 250 bits, as raw u64 limbs."""
    vals = [int(v) & ((1 << 250) - 1) for v in from_mont(digests).reshape(-1)]
    return np.array([[(v >> (64 * k)) & M64 for k in range(4)] for v in vals], dtype=np.uint64).reshape(digests.shape)


def sample_rows(n):
    """The first 512 items, the last 1024 and a strided sample of 4096."""
    return np.unique(np.concatenate([np.arange(min(512, n)), np.arange(max(n - 1024, 0), n),
                                     np.linspace(0, n - 1, 4096).astype(np.int64)]))


# ---- A. fixed-length device path, small and medium batches ------------------------------------------------------------
# (domain, in_len, out_len): Merkle4 / Merkle2 / Other.  Batch sizes: the lane-split kernel packs 6 items per warp and 24
# per block; 3168 is the default small-batch threshold on a 132-SM H100, 3169 the first batch above it.
M4, M2 = ("Merkle4", 4, 1), ("Merkle2", 2, 1)
O11, O31, O52, O47, O95, O168 = (("Other", a, b) for a, b in ((1, 1), (3, 1), (5, 2), (4, 7), (9, 5), (16, 8)))
DIGEST_CASES = [
    (M4, 1), (M4, 3168), (M4, 3169), (M4, 4099), (M2, 5), (M2, 129), (M2, 3169), (O11, 6), (O11, 33), (O11, 4099),
    (O31, 7), (O31, 3168), (O52, 31), (O52, 3169), (O47, 32), (O47, 129), (O95, 33), (O95, 4099), (O168, 129),
    (O168, 3169),
]


def _digest_params():
    return [pytest.param(c, n, False, id="%s-%d-%d-n%d" % (c + (n,))) for c, n in DIGEST_CASES] + \
        [pytest.param(M4, 3169, True, id="Merkle4-4-1-n3169-async")]


@pytest.mark.gpu
@pytest.mark.parametrize("case,n,async_", _digest_params())
def test_device_digest_vs_oracle(engine, oracle, coracle, case, n, async_):
    dom, in_len, out_len = case
    x = plant_edges(random_limbs_fast(np.random.default_rng([in_len, out_len, n]), (n, in_len)))
    xbuf, xd = guarded_in(x)
    obuf, od = guarded_out((n, out_len, 4))
    res = pb.Hash.digest_batch(getattr(pb.Domain, dom), xd, out_len, engine=engine, out=od, async_=async_)
    if async_:
        engine.sync()
    assert res is od
    assert_items_equal(_np(od), coracle.digest(_hash_tag(oracle, dom, in_len, out_len), x, in_len, out_len, threads=TH),
                       "device digests vs oracle")
    assert_guards(obuf, n, SENTINEL)
    assert_guards(xbuf, n, NONCANONICAL)
    assert np.array_equal(_np(xd), x)


@pytest.mark.gpu
@pytest.mark.parametrize("async_", [False, True])
def test_device_digest_with_tag_vs_oracle(engine, coracle, async_):
    n, in_len, out_len = 3169, 6, 3
    rng = np.random.default_rng([77, int(async_)])
    tag = random_limbs_fast(rng, 1)[0]                               # any scalar is a valid tag
    x = plant_edges(random_limbs_fast(rng, (n, in_len)))
    xbuf, xd = guarded_in(x)
    obuf, od = guarded_out((n, out_len, 4))
    engine.digest_batch_with_tag(tag, xd, out_len, out=od, async_=async_)
    if async_:
        engine.sync()
    assert_items_equal(_np(od), coracle.digest(tag, x, in_len, out_len, threads=TH), "digest_batch_with_tag vs oracle")
    assert_guards(obuf, n, SENTINEL)
    assert_guards(xbuf, n, NONCANONICAL)


@pytest.mark.gpu
@pytest.mark.parametrize("in_len,out_len", [(3, 1), (4, 7), (15, 1)])
@pytest.mark.parametrize("n", [1, 33, 3169])
def test_device_truncated_vs_oracle(engine, oracle, coracle, in_len, out_len, n):
    async_ = (in_len, out_len, n) == (4, 7, 33)
    x = plant_edges(random_limbs_fast(np.random.default_rng([in_len, out_len, n, 1]), (n, in_len)))
    xbuf, xd = guarded_in(x)
    obuf, od = guarded_out((n, out_len, 4))
    engine.hash_batch_truncated(pb.Domain.Other, xd, out_len, out=od, async_=async_)
    if async_:
        engine.sync()
    want = truncated(coracle.digest(_hash_tag(oracle, "Other", in_len, out_len), x, in_len, out_len, threads=TH))
    assert_items_equal(_np(od), want, "truncated device digests vs oracle")
    assert_guards(obuf, n, SENTINEL)
    assert_guards(xbuf, n, NONCANONICAL)


@functools.lru_cache(maxsize=None)
def crypt_case(L, n):
    """Inputs and oracle results of one encryption case (shared by both engine modes): messages, secrets, nonces,
    ciphers, the ciphers with a fixed subset of items tampered (a message scalar of every third item, the
    authentication scalar of every fifth from item 1), and the oracle's decryption of those (messages, ok)."""
    import hades_oracle as o
    rng = np.random.default_rng([L, n, 2])
    msg = plant_edges(random_limbs_fast(rng, (n, L)))
    sec = plant_edges(random_limbs_fast(rng, (n, 2)))
    non = plant_edges(random_limbs_fast(rng, (n, 1))).reshape(n, 4)
    tag = _crypt_tag(o, L)
    cipher = c_oracle.encrypt(tag, msg, L, sec, non)
    bad = cipher.copy()
    bad[0::3, 0, 0] ^= np.uint64(1)
    bad[1::5, L, 3] ^= np.uint64(1 << 40)
    want_msg, want_ok = c_oracle.decrypt(tag, bad, L, sec, non)
    return msg, sec, non, cipher, bad, want_msg, want_ok


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 4, 5, 9])
@pytest.mark.parametrize("n", [1, 33, 129, 3169])
def test_device_crypt_vs_oracle(engine, L, n):
    import torch
    async_ = (L, n) == (5, 129)
    msg, sec, non, cipher, bad, want_msg, want_ok = crypt_case(L, n)
    (mbuf, md), (sbuf, sd), (nbuf, nd) = guarded_in(msg), guarded_in(sec), guarded_in(non)

    # encrypt
    cbuf, cd = guarded_out((n, L + 1, 4))
    engine.encrypt_batch(md, sd, nd, out=cd, async_=async_)
    if async_:
        engine.sync()
    assert_items_equal(_np(cd), cipher, "device ciphers vs oracle")
    assert_guards(cbuf, n, SENTINEL)

    # decrypt the tampered ciphers
    fails = int((want_ok == 0).sum())
    assert not want_ok[0::3].any() and not want_ok[1::5].any() and fails == len(set(range(0, n, 3)) | set(range(1, n, 5)))
    good = want_ok == 1
    bbuf, bd = guarded_in(bad)
    obuf, od = guarded_out((n, L, 4))
    okbuf, okd = guarded_out((n,), torch.uint8)
    nfail = ctypes.c_size_t(12345)
    torch.cuda.synchronize()                      # the inputs were written on torch's stream, the engine has its own
    flags = _native.MEM_DEVICE | (_native.ASYNC if async_ else 0)
    assert engine._lib.p252_decrypt_batch(engine._ctx, bd.data_ptr(), n, L, sd.data_ptr(), nd.data_ptr(), od.data_ptr(),
                                          okd.data_ptr(), ctypes.byref(nfail), flags) == 0
    if async_:
        engine.sync()
    assert np.array_equal(okd.cpu().numpy(), want_ok)
    assert nfail.value == fails
    m = _np(od)
    assert not m[~good].any()                                            # failed items' messages are zero
    assert_items_equal(m[good], want_msg[good], "device messages vs oracle")
    assert np.array_equal(m[good], msg[good])
    for buf, fill in ((obuf, SENTINEL), (okbuf, OK_SENTINEL), (bbuf, NONCANONICAL), (sbuf, NONCANONICAL),
                      (nbuf, NONCANONICAL), (mbuf, NONCANONICAL)):
        assert_guards(buf, n, fill)
    # the public entry point on the same guarded inputs, with its own result buffers and failure count
    m2, ok2 = engine.decrypt_batch(bd, sd, nd, async_=async_)
    if async_:
        engine.sync()
    assert engine.last_decrypt_failures() == fails
    assert np.array_equal(ok2.cpu().numpy(), want_ok) and np.array_equal(_np(m2), m)


@pytest.mark.gpu
@pytest.mark.parametrize("n,async_", [(1, False), (6, False), (7, False), (33, False), (3168, False), (3169, False),
                                      (3169, True)])
def test_device_permute_vs_oracle(engine, coracle, n, async_):
    states = plant_edges(random_limbs_fast(np.random.default_rng([n, 3]), (n, 5)))
    want = coracle.permute(states, threads=TH)
    xbuf, xd = guarded_in(states)
    for dense in (False, True):
        obuf, od = guarded_out((n, 5, 4))
        res = engine.permute_batch(xd, dense=dense, out=od, async_=async_)
        if async_:
            engine.sync()
        assert res is od
        assert_items_equal(_np(od), want, "device permute (dense=%s) vs oracle" % dense)
        assert_guards(obuf, n, SENTINEL)
    assert np.array_equal(_np(xd), states)                               # out-of-place leaves the input alone
    assert_guards(xbuf, n, NONCANONICAL)
    engine.permute_batch_inplace(xd, async_=async_)
    if async_:
        engine.sync()
    assert_items_equal(_np(xd), want, "device in-place permute vs oracle")
    assert_guards(xbuf, n, NONCANONICAL)


# ---- B. the 256 x 2 shape: batches of at least WIDE items on device tensors ------------------------------------------
@pytest.fixture(scope="module")
def wide_engine():
    """One engine for the wide batches: above the small-batch threshold both modes of the shared fixture take the
    same kernels."""
    eng = pb.Engine(0)
    yield eng
    eng.close()


WIDE_SIZES = [WIDE - 1, WIDE, WIDE + 289]     # 128 x 5 (ragged); 256 x 2, whole blocks; last block 1 warp + 1 item


@pytest.mark.gpu
@pytest.mark.parametrize("case", [M4, M2, O11, O52, O95], ids=lambda c: "%s-%d-%d" % c)
@pytest.mark.parametrize("n", WIDE_SIZES, ids=["wide-1", "wide", "wide+289"])
def test_wide_digest_vs_host_path_and_oracle(wide_engine, oracle, coracle, case, n):
    import torch
    dom, in_len, out_len = case
    x = plant_edges(random_limbs_fast(np.random.default_rng([in_len, out_len, n, 4]), (n, in_len)))
    od = torch.full((n, out_len, 4), SENTINEL, dtype=torch.int64, device="cuda")
    wide_engine.hash_batch(getattr(pb.Domain, dom), torch.from_numpy(x.view(np.int64)).cuda(), out_len, out=od)
    got = _np(od)
    # host buffers: the 128 x 5 kernel in chunks of at most 2^17 items, a different shape on every item
    assert_items_equal(got, wide_engine.hash_batch(getattr(pb.Domain, dom), x, out_len), "device vs host-path digests")
    idx = sample_rows(n)
    want = coracle.digest(_hash_tag(oracle, dom, in_len, out_len), x[idx], in_len, out_len, threads=TH)
    assert_items_equal(got[idx], want, "device digests vs oracle (sampled items)")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [WIDE, WIDE + 289], ids=["wide", "wide+289"])
def test_wide_permute_vs_dense_and_oracle(wide_engine, coracle, n):
    states = plant_edges(random_limbs_fast(np.random.default_rng([n, 5]), (n, 5)))
    import torch
    d = torch.from_numpy(states.view(np.int64)).cuda()
    fast = _np(wide_engine.permute_batch(d))
    # the dense kernel is the reference's formulation of Hades (MDS matrix products), a separate implementation
    assert_items_equal(fast, _np(wide_engine.permute_batch(d, dense=True)), "256 x 2 permute vs dense permute")
    idx = sample_rows(n)
    assert_items_equal(fast[idx], coracle.permute(states[idx], threads=TH), "device permute vs oracle (sampled items)")
    wide_engine.permute_batch_inplace(d)
    assert_items_equal(_np(d), fast, "in-place vs out-of-place permute")


@pytest.mark.gpu
@pytest.mark.parametrize("arity,n_leaves", [(2, 1 << 20), (4, 4 ** 11)], ids=["arity2-2^20", "arity4-4^11"])
def test_wide_tree_build_vs_host_build_and_oracle(wide_engine, oracle, coracle, arity, n_leaves):
    import torch
    rng = np.random.default_rng([arity, 6])
    leaves = plant_edges(random_limbs_fast(rng, (n_leaves, 1))).reshape(n_leaves, 4)
    n_nodes = (n_leaves - 1) // (arity - 1)
    out = torch.full((n_nodes, 4), SENTINEL, dtype=torch.int64, device="cuda")
    wide_engine.merkle_build(torch.from_numpy(leaves.view(np.int64)).cuda(), arity=arity, out=out)
    nodes = _np(out)
    assert_items_equal(nodes, wide_engine.merkle_build(leaves, arity=arity), "device vs host-buffer tree nodes")
    # 64 leaf-to-root paths: every node on them recomputed with the oracle from its stored children
    tag = _hash_tag(oracle, "Merkle%d" % arity, arity, 1)
    idx = np.concatenate([[0, n_leaves - 1], rng.integers(0, n_leaves, size=62)])
    below = leaves
    for off, size in pb.merkle.level_offsets(n_leaves, arity):
        idx = idx // arity
        group = below[arity * idx[:, None] + np.arange(arity)]
        want = coracle.digest(tag, group, arity, 1).reshape(-1, 4)
        assert np.array_equal(nodes[off + idx], want), "path nodes of level size %d differ from the oracle" % size
        below = nodes[off:off + size]


# ---- C. (CPU) host chunks stay below the wide shape --------------------------------------------------------------------
def test_host_chunks_stay_below_wide_shape():
    """The B tests compare device batches (256 x 2) with host batches of the same items, which the staged pipeline
    hands to the kernel in chunks.  The largest chunk any item size or P252_CHUNK_ITEMS setting allows is the byte
    target over 64 bytes per item (in_len = out_len = 1), rounded up to 128 items; it must stay below the wide-shape
    threshold, or the host path would run the same kernel and the comparison would test nothing."""
    items = source_constant(CAPI_CU, "kChunkItemsDefault")
    target = source_constant(CAPI_CU, "kChunkBytesTarget")
    largest = (max(1024, target // 64) + 127) // 128 * 128
    for what, chunk in (("the default chunk", items), ("the largest chunk", largest)):
        assert chunk < WIDE, ("%s of %d host items reaches the 256 x 2 shape (P252_WIDE_SHAPE_MIN = %d): the wide-shape "
                              "tests in this file no longer compare two launch shapes" % (what, chunk, WIDE))
