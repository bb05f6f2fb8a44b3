"""GPU (-m gpu): variable-length digest batches (p252_hash_batch_varlen) against the C oracle's digest per length group,
with tags from hades_oracle (not from the library); equality with the fixed-length p252_hash_batch and with grouped
per-length calls; Merkle domains; device-side rejections and host-side refusals; host and device buffers, async calls,
tag-table growth, multi-chunk host batches with fault injection, and a full-size batch.  Both digest kernels (the
two-parameter `engine` fixture)."""
import functools

import numpy as np
import pytest

import c_oracle
import hades_oracle as o
import poseidon252_b200 as pb
from poseidon252_b200.scalar import random_limbs_fast, to_mont

pytestmark = pytest.mark.gpu

MEMS = ["host", "device"]


def host(x):
    return x.cpu().numpy().view(np.uint64) if hasattr(x, "is_cuda") else np.asarray(x)


def to_mem(a, mem):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if mem == "host":
        return a
    import torch
    return torch.from_numpy(a.view(np.int64)).cuda()


@functools.lru_cache(maxsize=None)
def otag(domain, length, out_len):
    """tag of Hash::digest over `length` inputs with `out_len` outputs, from the oracle's restatement"""
    dsep = getattr(o.Domain, pb.Domain(domain).name)
    return to_mont(o.hash_to_scalar(o.tag_input([o.Absorb(length), o.Squeeze(out_len)], dsep)))


def oracle_varlen(domain, data, offsets, out_len, rows=None):
    """expected (len(rows), out_len, 4): the C oracle's digest per length group"""
    offsets = np.asarray(offsets, dtype=np.int64)
    rows = np.arange(offsets.shape[0] - 1) if rows is None else np.asarray(rows)
    lens = offsets[rows + 1] - offsets[rows]
    want = np.zeros((rows.shape[0], out_len, 4), dtype=np.uint64)
    for L in np.unique(lens):
        sel = np.nonzero(lens == L)[0]
        idx = offsets[rows[sel]][:, None] + np.arange(L)[None, :]
        want[sel] = c_oracle.digest(otag(domain, int(L), out_len), data[idx], int(L), out_len)
    return want


def grouped(engine, domain, data, offsets, out_len):
    """the status quo: one p252_hash_batch per distinct length, gathered and scattered on the host"""
    offsets = np.asarray(offsets, dtype=np.int64)
    lens = offsets[1:] - offsets[:-1]
    out = np.zeros((lens.shape[0], out_len, 4), dtype=np.uint64)
    for L in np.unique(lens):
        sel = np.nonzero(lens == L)[0]
        idx = offsets[sel][:, None] + np.arange(L)[None, :]
        out[sel] = engine.hash_batch(domain, np.ascontiguousarray(data[idx]), out_len)
    return out


def batch(rng, lens, lead=0):
    """random scalars for items of the given lengths, packed back to back after `lead` unused scalars"""
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(lead)
    return random_limbs_fast(rng, int(offsets[-1])), offsets


def coop_max():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 24


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("domain", [pb.Domain.Other, pb.Domain.Encryption])
@pytest.mark.parametrize("out_len", [1, 3, 5])
def test_every_length_shuffled_matches_oracle(engine, mem, domain, out_len):
    rng = np.random.default_rng(100 + out_len)
    lens = rng.permutation(np.arange(1, 257))
    data, offsets = batch(rng, lens, lead=7)                 # offsets[0] = 7: a slice of a larger CSR array
    got = engine.hash_batch_varlen(domain, to_mem(data, mem), to_mem(offsets, mem), out_len)
    assert np.array_equal(host(got), oracle_varlen(domain, data, offsets, out_len))
    assert engine.last_varlen_rejected() == 0


@pytest.mark.parametrize("mem", MEMS)
def test_equal_lengths_bit_identical_to_hash_batch(engine, mem):
    rng = np.random.default_rng(2)
    cm = coop_max()
    for L in (1, 4, 5, 8, 42):
        for n in (1, 31, 33, cm, cm + 1, 1 << 16):
            data = random_limbs_fast(rng, n * L)
            offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(L)
            want = engine.hash_batch(pb.Domain.Other, data.reshape(n, L, 4))
            got = engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, mem), to_mem(offsets, mem))
            assert np.array_equal(host(got), want), (L, n)


@pytest.mark.parametrize("mem", MEMS)
def test_random_mixes_equal_grouped_calls(engine, mem):
    rng = np.random.default_rng(3)
    mixes = {"uniform": rng.integers(1, 65, 5000),
             "geometric": np.minimum(rng.geometric(0.08, 5000), 700),
             "one_huge": np.concatenate([rng.integers(1, 9, 150), [pb._native.VARLEN_MAX_LEN], rng.integers(1, 9, 150)])}
    for name, lens in mixes.items():
        for out_len in (1, 6):
            data, offsets = batch(rng, lens)
            got = engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, mem), to_mem(offsets, mem), out_len)
            assert np.array_equal(host(got), grouped(engine, pb.Domain.Other, data, offsets, out_len)), (name, out_len)
    # the huge item checked against the oracle as well
    assert np.array_equal(host(got)[150], oracle_varlen(pb.Domain.Other, data, offsets, 6, rows=[150])[0])


@pytest.mark.parametrize("mem", MEMS)
def test_merkle_batches_at_arity(engine, mem):
    rng = np.random.default_rng(4)
    for domain, arity in ((pb.Domain.Merkle4, 4), (pb.Domain.Merkle2, 2)):
        n = 3000
        data = random_limbs_fast(rng, n * arity)
        offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(arity)
        got = engine.hash_batch_varlen(domain, to_mem(data, mem), to_mem(offsets, mem))
        assert np.array_equal(host(got), engine.hash_batch(domain, data.reshape(n, arity, 4)))
        assert np.array_equal(host(got)[:50], oracle_varlen(domain, data, offsets, 1, rows=np.arange(50)))


def mixed_merkle(rng):
    lens = np.full(500, 4)
    lens[[3, 77, 499]] = (3, 5, 1)
    data, offsets = batch(rng, lens)
    return data, offsets, [3, 77, 499]


def test_mixed_merkle_host_refused_nothing_written(engine):
    data, offsets, _ = mixed_merkle(np.random.default_rng(5))
    out = np.full((500, 1, 4), 0xabab, dtype=np.uint64)
    with pytest.raises(pb.IOPatternViolation):
        engine.hash_batch_varlen(pb.Domain.Merkle4, data, offsets, max_len=8, out=out)
    assert (out == 0xabab).all()


def test_mixed_merkle_device_zero_rows(engine):
    data, offsets, bad = mixed_merkle(np.random.default_rng(5))
    got = host(engine.hash_batch_varlen(pb.Domain.Merkle4, to_mem(data, "device"), to_mem(offsets, "device"), max_len=8))
    assert engine.last_varlen_rejected() == len(bad)
    good = np.setdiff1d(np.arange(500), bad)
    assert not got[bad].any()
    assert np.array_equal(got[good], oracle_varlen(pb.Domain.Merkle4, data, offsets, 1, rows=good))


def test_device_rejections(engine):
    rng = np.random.default_rng(6)
    lens = rng.integers(1, 20, 400)
    data, offsets = batch(rng, lens)
    offsets = offsets.astype(np.int64)
    n_scalars = int(offsets[-1])
    offsets[10] = offsets[9]                                  # item 9: length 0
    offsets[41] = offsets[40] + 25                            # item 40: length 25 > max_len 24
    offsets[100] = offsets[101] + 5                           # item 100: offsets decrease (item 99 gets longer)
    offsets[-1] = n_scalars + 3                               # item 399: ends past n_scalars
    full = random_limbs_fast(rng, n_scalars + 64)                # the tensor is longer than the n_scalars passed
    full[:n_scalars] = data
    dev = to_mem(full, "device")
    offs = to_mem(offsets.astype(np.uint64), "device")
    got = host(engine.hash_batch_varlen(pb.Domain.Other, dev[:n_scalars], offs, 2, max_len=24))
    all_lens = offsets[1:] - offsets[:-1]                     # neighbours of the edited offsets may turn invalid too
    bad = np.nonzero((all_lens < 1) | (all_lens > 24) | (offsets[1:] > n_scalars))[0]
    assert {9, 40, 100, 399} <= set(bad.tolist())
    assert engine.last_varlen_rejected() == len(bad)
    assert not got[bad].any()
    good = np.setdiff1d(np.arange(400), bad)
    assert np.array_equal(got[good], oracle_varlen(pb.Domain.Other, full, offsets, 2, rows=good))


def test_host_rejections_nothing_written(engine):
    rng = np.random.default_rng(7)
    data, offsets = batch(rng, rng.integers(1, 10, 50))
    offsets = offsets.astype(np.int64)

    def refused(exc, offs, n_scalars=None, code=None):
        out = np.full((offs.shape[0] - 1, 1, 4), 0xcd, dtype=np.uint64)
        with pytest.raises(exc) as ei:
            engine.hash_batch_varlen(pb.Domain.Other, data[:n_scalars], offs.astype(np.uint64), max_len=16, out=out)
        if code is not None:
            assert ei.value.code == code
        assert (out == 0xcd).all()

    o2 = offsets.copy()
    o2[6] = o2[5]
    refused(pb.InvalidIOPattern, o2)                                    # length 0
    o2 = offsets.copy()
    o2[6] = o2[5] + 17
    refused(pb.EngineError, o2, code=-1)                                # length > max_len
    o2 = offsets.copy()
    o2[6] = o2[7] + 1
    refused(pb.EngineError, o2, code=-1)                                # decreasing offsets
    refused(pb.EngineError, offsets, n_scalars=int(offsets[-1]) - 1, code=-1)   # past n_scalars
    o2 = offsets.copy()
    o2[3] = o2[4] + 2                                                   # item 3 decreasing: INVALID_ARGUMENT ...
    o2[31] = o2[30]                                                     # ... wins over item 30's length 0
    refused(pb.EngineError, o2, code=-1)
    # batch-level checks
    out_ok = np.zeros((50, 1, 4), dtype=np.uint64)
    with pytest.raises(pb.InvalidIOPattern):
        engine.hash_batch_varlen(pb.Domain.Other, data, offsets.astype(np.uint64), 0)
    with pytest.raises(pb.IOPatternViolation):
        engine.hash_batch_varlen(pb.Domain.Merkle4, data, offsets.astype(np.uint64), 2)
    for m in (0, pb._native.VARLEN_MAX_LEN + 1):
        with pytest.raises(pb.EngineError):
            engine.hash_batch_varlen(pb.Domain.Other, data, offsets.astype(np.uint64), max_len=m, out=out_ok)
        with pytest.raises(pb.EngineError):
            engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device"), max_len=m)
    assert not out_ok.any()


def test_host_equals_device_empty_and_async(engine):
    rng = np.random.default_rng(8)
    data, offsets = batch(rng, rng.integers(1, 100, 3000))
    h = engine.hash_batch_varlen(pb.Domain.Other, data, offsets, 4)
    d = engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device"), 4)
    assert np.array_equal(h, host(d))
    a = engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device"), 4, async_=True)
    engine.sync()
    assert np.array_equal(h, host(a))
    for mem in MEMS:                                          # n = 0
        got = engine.hash_batch_varlen(pb.Domain.Other, to_mem(np.zeros((0, 4)), mem), to_mem(np.zeros(1), mem), 3)
        assert tuple(got.shape) == (0, 3, 4)
        got = engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, mem), to_mem(offsets[5:6], mem), 3)
        assert tuple(got.shape) == (0, 3, 4)


def test_tag_table_growth_between_async_calls(engine):
    """A fresh context: each call below rebuilds the tag table while the previous call may still be running."""
    rng = np.random.default_rng(9)
    eng = pb.Engine(0)
    try:
        calls = []
        for lens, out_len in ((rng.integers(1, 9, 2000), 1), (rng.integers(1, 301, 2000), 1), (rng.integers(1, 301, 50), 3)):
            data, offsets = batch(rng, lens)
            got = eng.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device"), out_len,
                                        async_=True)
            calls.append((data, offsets, out_len, got))
        eng.sync()
        for data, offsets, out_len, got in calls:
            assert np.array_equal(host(got), oracle_varlen(pb.Domain.Other, data, offsets, out_len))
    finally:
        eng.close()


def test_host_multi_chunk_and_injected_fault(engine):
    rng = np.random.default_rng(10)
    lens = rng.integers(32, 97, 40000)                        # ~2.6 M scalars: four chunks of <= 24 MiB input
    lens[123] = pb._native.VARLEN_MAX_LEN
    data, offsets = batch(rng, lens)
    assert data.nbytes > 3 * (24 << 20)
    want = host(engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device"), 2))
    assert np.array_equal(engine.hash_batch_varlen(pb.Domain.Other, data, offsets, 2), want)
    lib, ctx = pb._native.lib(), engine._ctx
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    out = np.zeros((lens.shape[0], 2, 4), dtype=np.uint64)
    with pytest.raises(pb.EngineError) as ei:
        engine.hash_batch_varlen(pb.Domain.Other, data, offsets, 2, out=out)
    assert "injected" in str(ei.value)
    assert np.array_equal(engine.hash_batch_varlen(pb.Domain.Other, data, offsets, 2), want)   # context still usable
    rows = rng.choice(lens.shape[0], 64, replace=False)
    assert np.array_equal(want[rows], oracle_varlen(pb.Domain.Other, data, offsets, 2, rows=rows))


def test_hash_digest_batch_varlen_front_end(engine):
    rng = np.random.default_rng(11)
    items = [random_limbs_fast(rng, int(k)) for k in rng.integers(1, 30, 200)]
    got = pb.Hash.digest_batch_varlen(pb.Domain.Other, items, output_len=2, engine=engine)
    data, offsets, _ = pb.pack_varlen(items)
    assert np.array_equal(got, oracle_varlen(pb.Domain.Other, data, offsets, 2))
    for i in (0, 57, 199):                                     # = Hash::digest with output_len, item by item
        h = pb.Hash(pb.Domain.Other, engine)
        h.output_len(2)
        h.update(items[i])
        assert np.array_equal(got[i], h.finalize())
    # the reference ignores output_len for the other domains; a (data, offsets) pair of device tensors works as well
    got = pb.Hash.digest_batch_varlen(pb.Domain.Encryption, (to_mem(data, "device"), to_mem(offsets, "device")),
                                      output_len=2, engine=engine)
    assert np.array_equal(host(got), oracle_varlen(pb.Domain.Encryption, data, offsets, 1))


def test_full_size_2e20_items(engine):
    rng = np.random.default_rng(12)
    lens = rng.integers(1, 65, 1 << 20)
    data, offsets = batch(rng, lens)
    got = host(engine.hash_batch_varlen(pb.Domain.Other, to_mem(data, "device"), to_mem(offsets, "device")))
    assert engine.last_varlen_rejected() == 0
    rows = rng.choice(1 << 20, 4096, replace=False)
    assert np.array_equal(got[rows], oracle_varlen(pb.Domain.Other, data, offsets, 1, rows=rows))
