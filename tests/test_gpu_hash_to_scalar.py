"""GPU (-m gpu): batched BlsScalar::hash_to_scalar (p252_hash_to_scalar_batch) and from_bytes_wide
(p252_scalars_from_bytes_wide) against hashlib's BLAKE2b-512 and a big-integer reduction (the oracle's hash_to_scalar):
every length 0..1024 and the block edges 128 k +- 1, every start address mod 16, offsets[0] != 0 and empty items, the
one-block path (max_len <= 128) and the sorted one, HOST and DEVICE buffers, sync and P252_ASYNC; agreement with the
host's p252_hash_to_scalar and with the sponge tags p252_tag derives; from_bytes_wide at the edges of lo and hi; a full
2^20-item batch and a heavy tail; device rejections with guard rows, host refusals, multi-chunk host batches with exact
launch counts and an injected failure, n == 0; device rows used as Schnorr messages; the C and C++ programs."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

import hades_oracle as o
import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.hash import hash_to_scalar, pack_bytes
from poseidon252_b200.scalar import P, jubjub_limbs
from test_hash_to_scalar_cpu import c_smoke, cpp_mirror

pytestmark = pytest.mark.gpu

R = (1 << 256) % P
MAX_LEN = _native.HASH_TO_SCALAR_MAX_LEN
CHUNK_BYTES = 24 << 20
CHUNK_ITEMS = int(os.environ.get("P252_CHUNK_ITEMS", 1 << 17))   # as chunk_items_max() reads it
CHUNK_ITEMS = CHUNK_ITEMS if CHUNK_ITEMS >= 1024 else 1 << 17
# (memory space, async): HOST calls are always synchronous
SPACES = [("host", False), ("device", False), ("device", True)]


@pytest.fixture(scope="module")
def eng():
    e = pb.Engine(0)
    yield e
    e.close()


def mont_rows(values):
    """canonical integers -> (n, 4) uint64 Montgomery limbs, through one bytes buffer"""
    buf = b"".join((v * R % P).to_bytes(32, "little") for v in values)
    return np.frombuffer(buf, dtype=np.uint64).reshape(-1, 4).copy()


def want(data, offsets, rows=None):
    """the oracle's hash_to_scalar of every item (or of `rows`), Montgomery limbs"""
    d = memoryview(np.ascontiguousarray(data, dtype=np.uint8))
    offs = np.asarray(offsets, dtype=np.int64)
    rows = range(offs.shape[0] - 1) if rows is None else rows
    return mont_rows(o.from_bytes_wide(hashlib.blake2b(d[offs[i]:offs[i + 1]], digest_size=64).digest()) for i in rows)


def host(x):
    """a result as a numpy array: 64-bit words as uint64, bytes as uint8"""
    if not hasattr(x, "is_cuda"):
        return np.asarray(x)
    a = x.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    return torch.from_numpy(a).cuda()


def run(e, mem, async_, data, offsets, max_len=None, out=None):
    if mem == "host":
        return e.hash_to_scalar_batch(data, offsets, max_len=max_len, out=out)
    got = e.hash_to_scalar_batch(to_dev(data), to_dev(np.asarray(offsets, dtype=np.uint64)), max_len=max_len, out=out,
                                 async_=async_)
    if async_:
        e.sync()
    return host(got)


def random_batch(rng, lens, lead=0, tail=0):
    """random bytes for items of the given lengths, back to back after `lead` and before `tail` unused bytes"""
    offsets = (np.concatenate([[0], np.cumsum(lens)]) + lead).astype(np.uint64)
    return rng.integers(0, 256, int(offsets[-1]) + tail, dtype=np.uint8), offsets


# ---- lengths ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", SPACES)
def test_every_length_0_to_1024_shuffled(eng, mem, async_):
    rng = np.random.default_rng(1)
    lens = rng.permutation(np.arange(1025))
    data, offsets = random_batch(rng, lens)
    assert np.array_equal(run(eng, mem, async_, data, offsets), want(data, offsets))
    if mem == "device":
        assert eng.last_hash_to_scalar_rejected() == 0


@pytest.mark.parametrize("mem,async_", SPACES)
def test_block_edges_up_to_64_blocks(eng, mem, async_):
    rng = np.random.default_rng(2)
    lens = rng.permutation([128 * k + d for k in range(1, 65) for d in (-1, 0, 1)])
    data, offsets = random_batch(rng, lens)
    assert np.array_equal(run(eng, mem, async_, data, offsets), want(data, offsets))


@pytest.mark.parametrize("mem,async_", SPACES)
@pytest.mark.parametrize("top", [128, 129, 5000])
def test_random_lengths_on_both_paths(eng, mem, async_, top):
    """top = 128: every item one block, no sort; above it the items are sorted by block count"""
    rng = np.random.default_rng(3 + top)
    data, offsets = random_batch(rng, rng.integers(0, top + 1, 3000))
    assert np.array_equal(run(eng, mem, async_, data, offsets, max_len=top), want(data, offsets))


# ---- placement -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_every_start_address_mod_16(eng, mem):
    """the buffer starts at every address mod 16 and items start anywhere, including at its first byte and ending at its
    last one (the aligned loads there are cut to the buffer)"""
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 300, 200)
    lens[::7] = 0                                             # empty items between non-empty ones
    lens[0], lens[-1] = 37, 141
    data, offsets = random_batch(rng, lens)
    for s in range(16):
        big = rng.integers(0, 256, data.shape[0] + 16, dtype=np.uint8)
        big[s:s + data.shape[0]] = data
        if mem == "host":
            got = eng.hash_to_scalar_batch(big[s:s + data.shape[0]], offsets)
        else:
            dev = to_dev(big)
            view = dev[s:s + data.shape[0]]
            assert view.data_ptr() % 16 == s % 16 or dev.data_ptr() % 16 != 0
            got = host(eng.hash_to_scalar_batch(view, to_dev(offsets)))
        assert np.array_equal(got, want(data, offsets)), s


@pytest.mark.parametrize("mem,async_", SPACES)
def test_slice_of_a_larger_csr_array(eng, mem, async_):
    rng = np.random.default_rng(5)
    data, offsets = random_batch(rng, rng.integers(0, 400, 500), lead=1234, tail=77)
    assert int(offsets[0]) == 1234
    got = run(eng, mem, async_, data, offsets[100:301])
    assert np.array_equal(got, want(data, offsets[100:301]))


# ---- the existing calls ----------------------------------------------------------------------------------------------
def test_rows_equal_the_host_hash_to_scalar(eng):
    rng = np.random.default_rng(6)
    msgs = [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in rng.integers(0, 700, 300)]
    got = pb.hash_to_scalar_batch(msgs, engine=eng)
    for i, m in enumerate(msgs):
        assert np.array_equal(got[i], hash_to_scalar(m)), i


def test_tags_equal_the_batch_over_tag_input_bytes(eng):
    """Safe::tag of io-patterns (p252_tag, derived on the host) is the batch over the p252_tag_input bytes"""
    patterns, dseps = [], []
    for dom in pb.Domain:
        dsep = pb.hash.domain_separator(dom)
        for ins in (1, 2, 4, 5, 17, 1000):
            for outs in (1, 3):
                patterns.append([("absorb", ins), ("squeeze", outs)])
                dseps.append(dsep)
    patterns.append([("absorb", 2), ("absorb", 1), ("squeeze", 9), ("absorb", 9), ("squeeze", 1)])   # encryption
    dseps.append(pb.hash.domain_separator(pb.Domain.Encryption))
    inputs = [pb.hash.tag_input(p, d) for p, d in zip(patterns, dseps)]
    tags = np.stack([pb.hash.tag(p, d) for p, d in zip(patterns, dseps)])
    for mem in ("host", "device"):
        data, offsets, longest = pack_bytes(inputs)
        assert np.array_equal(run(eng, mem, False, data, offsets, max_len=longest), tags)


# ---- from_bytes_wide -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_from_bytes_wide_edges(eng, mem):
    edges = (0, 1, P - 1, P, 2 * P - 1, 1 << 255, (1 << 256) - 1)
    pairs = [(lo, hi) for lo in edges for hi in edges]
    rows = np.frombuffer(b"".join(lo.to_bytes(32, "little") + hi.to_bytes(32, "little") for lo, hi in pairs),
                         dtype=np.uint8).reshape(-1, 64)
    expect = mont_rows((lo + (hi << 256)) % P for lo, hi in pairs)
    if mem == "host":
        got = eng.scalars_from_bytes_wide(rows)
    else:
        got = host(eng.scalars_from_bytes_wide(to_dev(rows.view(np.uint64))))
    assert np.array_equal(got, expect)


def test_from_bytes_wide_of_digests_equals_the_batch(eng):
    rng = np.random.default_rng(7)
    data, offsets = random_batch(rng, rng.integers(0, 600, 1000))
    d = data.tobytes()
    digests = np.frombuffer(b"".join(hashlib.blake2b(d[offsets[i]:offsets[i + 1]], digest_size=64).digest()
                                     for i in range(1000)), dtype=np.uint8).reshape(-1, 64)
    assert np.array_equal(eng.scalars_from_bytes_wide(digests), eng.hash_to_scalar_batch(data, offsets))


# ---- full size and the heavy tail -----------------------------------------------------------------------------------
def test_full_size_2e20_mixed_lengths(eng):
    rng = np.random.default_rng(8)
    n = 1 << 20
    data, offsets = random_batch(rng, rng.integers(0, 4097, n))
    got = host(eng.hash_to_scalar_batch(to_dev(data), to_dev(offsets)))
    assert eng.last_hash_to_scalar_rejected() == 0
    assert np.array_equal(got, want(data, offsets))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_heavy_tail(eng, mem):
    rng = np.random.default_rng(9)
    lens = rng.integers(0, 200, 20000)
    lens[12345] = MAX_LEN
    data, offsets = random_batch(rng, lens)
    got = run(eng, mem, False, data, offsets, max_len=MAX_LEN)
    assert np.array_equal(got, want(data, offsets))


# ---- invalid items, refusals, chunks, n == 0 -------------------------------------------------------------------------
@pytest.mark.parametrize("max_len", [100, 128, 1000])
def test_device_rejections_zero_rows_and_guards(eng, max_len):
    rng = np.random.default_rng(10 + max_len)
    n = 600
    data, offsets = random_batch(rng, rng.integers(0, min(max_len, 90) + 1, n))
    offsets = offsets.astype(np.int64)
    nb = int(offsets[-1])
    offsets[11] = offsets[10] + max_len + 1                   # item 10 longer than max_len
    offsets[101] = offsets[102] + 5                           # item 101 decreasing (item 100 longer)
    offsets[300] = -1                                         # items 299 and 300: a huge offset
    offsets[-1] = nb + 3                                      # item n - 1 ends past n_bytes
    full = np.concatenate([data, rng.integers(0, 256, 4096, dtype=np.uint8)])    # a longer tensor than the n_bytes passed
    dev = to_dev(full)
    import torch
    guard = torch.full((n + 2, 4), 0x5a5a, dtype=torch.int64, device="cuda")
    eng.hash_to_scalar_batch(dev[:nb], to_dev(offsets.astype(np.uint64)), max_len=max_len, out=guard[1:n + 1])
    got = host(guard)
    u = offsets.astype(np.uint64)
    lens = u[1:] - u[:-1]
    bad = np.nonzero((u[:-1] > u[1:]) | (u[1:] > nb) | (lens > max_len))[0]
    assert {10, 101, 299, 300, n - 1} <= set(bad.tolist())
    assert eng.last_hash_to_scalar_rejected() == len(bad)
    assert (got[0] == 0x5a5a).all() and (got[n + 1] == 0x5a5a).all()
    rows = got[1:n + 1]
    assert not rows[bad].any()
    good = np.setdiff1d(np.arange(n), bad)
    assert np.array_equal(rows[good], want(full, offsets, rows=good))


def test_host_refusals_nothing_written(eng):
    rng = np.random.default_rng(11)
    data, offsets = random_batch(rng, rng.integers(0, 50, 60))
    offsets = offsets.astype(np.int64)

    def refused(offs, n_bytes=None, max_len=64):
        out = np.full((offs.shape[0] - 1, 4), 0xcd, dtype=np.uint64)
        with pytest.raises(pb.EngineError) as ei:
            eng.hash_to_scalar_batch(data[:n_bytes], offs.astype(np.uint64), max_len=max_len, out=out)
        assert ei.value.code == -1
        assert (out == 0xcd).all()

    o2 = offsets.copy()
    o2[6] = o2[5] + 65
    refused(o2)                                               # item 5 longer than max_len
    o2 = offsets.copy()
    o2[6] = o2[7] + 1
    refused(o2)                                               # decreasing offsets
    refused(offsets, n_bytes=int(offsets[-1]) - 1)            # past n_bytes
    o2 = offsets.copy()
    o2[3] = o2[4] + 2                                         # the lowest invalid item (2 or 3) decides ...
    o2[40] = o2[39] + 100                                     # ... ahead of a later one
    refused(o2)
    refused(offsets, max_len=MAX_LEN + 1)                     # batch checks
    with pytest.raises(pb.EngineError):
        eng.hash_to_scalar_batch(to_dev(data), to_dev(offsets.astype(np.uint64)), max_len=MAX_LEN + 1)
    lib, ctx = _native.lib(), eng._ctx
    buf = (ctypes.c_uint8 * 8)()
    off = (ctypes.c_uint64 * 2)(0, 8)
    out = (ctypes.c_uint64 * 4)(*([7] * 4))
    assert lib.p252_hash_to_scalar_batch(ctx, buf, 8, off, 1 << 31, 8, out, None, 0) == -1        # n >= 2^31
    assert lib.p252_hash_to_scalar_batch(ctx, None, 8, off, 1, 8, out, None, 0) == -1             # NULL bytes
    assert lib.p252_hash_to_scalar_batch(ctx, buf, 8, None, 1, 8, out, None, 0) == -1             # NULL offsets
    assert list(out) == [7] * 4
    # max_len == 0 is a valid bound: empty items hash, the others are refused
    e = eng.hash_to_scalar_batch(np.zeros(0, np.uint8), np.zeros(3, np.uint64), max_len=0)
    assert np.array_equal(e, want(np.zeros(0, np.uint8), [0, 0, 0]))


def chunk_bounds(offsets):
    """the chunks of a HOST batch, as capi.cu's chunk_bounds with element size 1"""
    n, bounds, lo = offsets.shape[0] - 1, [0], 0
    while lo < n:
        hi = lo + 1
        while hi < n and hi - lo < CHUNK_ITEMS and int(offsets[hi + 1]) - int(offsets[lo]) <= CHUNK_BYTES:
            hi += 1
        bounds.append(hi)
        lo = hi
    return bounds


@pytest.mark.parametrize("top,per_chunk", [(128, 1), (3000, 2)])
def test_host_multi_chunk_launch_counts_and_injected_fault(eng, top, per_chunk):
    rng = np.random.default_rng(12 + top)
    n = 300000 if top == 128 else 40000
    data, offsets = random_batch(rng, rng.integers(0, top + 1, n))
    chunks = len(chunk_bounds(offsets)) - 1
    assert chunks >= 3
    before = eng.launch_count
    got = eng.hash_to_scalar_batch(data, offsets, max_len=top)
    assert eng.launch_count - before == chunks * per_chunk
    rows = rng.choice(n, 2000, replace=False)
    assert np.array_equal(got[rows], want(data, offsets, rows=rows))
    assert _native.lib().p252_debug_fail_chunk(eng._ctx, 1) == 0
    out = np.zeros((n, 4), dtype=np.uint64)
    with pytest.raises(pb.EngineError) as ei:
        eng.hash_to_scalar_batch(data, offsets, max_len=top, out=out)
    assert "injected" in str(ei.value)
    assert np.array_equal(eng.hash_to_scalar_batch(data, offsets, max_len=top), got)          # context still usable
    dev = host(eng.hash_to_scalar_batch(to_dev(data), to_dev(offsets), max_len=top))
    assert np.array_equal(dev, got)


def test_n_zero(eng):
    data = np.arange(10, dtype=np.uint8)
    for mem in ("host", "device"):
        before = eng.launch_count
        for offs in (np.zeros(1, np.uint64), np.array([4], np.uint64)):
            got = run(eng, mem, False, data, offs)
            assert got.shape == (0, 4)
        assert eng.launch_count == before


# ---- end to end: payload hashes as Schnorr messages -----------------------------------------------------------------
def test_device_rows_as_schnorr_messages(eng):
    rng = np.random.default_rng(13)
    n = 4096
    data, offsets = random_batch(rng, rng.integers(0, 900, n))
    G = jo.points_mont([jo.GENERATOR])[0]
    sk = jubjub_limbs([jo.random_secret(rng)])
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(n)])
    pk, _ = eng.fixed_base_batch(sk, G)
    m_host = np.stack([hash_to_scalar(data[int(offsets[i]):int(offsets[i + 1])].tobytes()) for i in range(n)])
    m_dev = eng.hash_to_scalar_batch(to_dev(data), to_dev(offsets))
    assert np.array_equal(host(m_dev), m_host)
    u_h, R_h, ok_h = eng.schnorr_sign_batch(sk, r, m_host, G)
    u_d, R_d, ok_d = eng.schnorr_sign_batch(to_dev(sk), to_dev(r), m_dev, G)
    assert ok_h.all() and np.array_equal(host(ok_d), ok_h)
    assert np.array_equal(host(u_d), u_h) and np.array_equal(host(R_d), R_h)
    v_d = eng.schnorr_verify_batch(to_dev(pk), u_d, R_d, m_dev, G)
    v_h = eng.schnorr_verify_batch(pk, u_h, R_h, m_host, G)
    assert v_h.all() and np.array_equal(host(v_d), v_h)


# ---- front end and the C / C++ programs ------------------------------------------------------------------------------
def test_module_front_end(eng):
    rng = np.random.default_rng(14)
    msgs = [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in rng.integers(0, 300, 100)]
    data, offsets, _ = pack_bytes(msgs)
    w = want(data, offsets)
    assert np.array_equal(pb.hash_to_scalar_batch(msgs, engine=eng), w)
    assert np.array_equal(host(pb.hash_to_scalar_batch((to_dev(data), to_dev(offsets)), engine=eng)), w)
    assert np.array_equal(pb.hash_to_scalar_batch((data, offsets), engine=eng), w)
    assert np.array_equal(pb.hash_to_scalar_batch([], engine=eng), np.zeros((0, 4), np.uint64))


def test_c_smoke_on_the_device():
    res = c_smoke()
    assert res.returncode == 0 and "HASH_TO_SCALAR_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_mirror_on_the_device():
    res = cpp_mirror()
    assert res.returncode == 0 and res.stdout.strip() == "hash_to_scalar mirror ok", (res.returncode, res.stdout, res.stderr)
