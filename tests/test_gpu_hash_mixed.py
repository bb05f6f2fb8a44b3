"""GPU (-m gpu): mixed digest batches (p252_hash_batch_mixed) -- every domain x {finalize, truncated} x input and output
length combination in one shuffled call against the C oracle's digest under tags from hades_oracle (not from the
library), which checks the tags derived on the device; equality with p252_hash_batch_varlen and
p252_hash_batch_truncated per group; Hash.finalize_batch against Hash.finalize / finalize_truncated; slices of larger
CSR arrays; device rejections for every item rule with guard rows; host refusals by the lowest-index invalid item;
multi-chunk host batches with fault injection; n == 0; the full-size node mix of tools/bench_hash_mixed.py; the C and C++
programs.  Both digest kernels (the two-parameter `engine` fixture), host and device buffers, async device calls."""
import functools

import numpy as np
import pytest

import bench_hash_mixed as bm
import c_oracle
import hades_oracle as o
import poseidon252_b200 as pb
from poseidon252_b200.scalar import from_mont, random_limbs_fast, to_mont

pytestmark = pytest.mark.gpu

T = pb._native.MIXED_TRUNCATED
MEMS = ["host", "device", "device-async"]
ARITY = {int(pb.Domain.Merkle4): 4, int(pb.Domain.Merkle2): 2}


def host(x):
    return x.cpu().numpy().view(np.uint64) if hasattr(x, "is_cuda") else np.asarray(x)


def to_mem(a, mem, dtype=np.uint64):
    a = np.ascontiguousarray(a, dtype=dtype)
    if mem == "host":
        return a
    import torch
    return torch.from_numpy(a.view(np.int64) if dtype == np.uint64 else a).cuda()


@functools.lru_cache(maxsize=None)
def otag(domain, length, out_len):
    """tag of Hash::digest over `length` inputs with `out_len` outputs, from the oracle's restatement"""
    dsep = getattr(o.Domain, pb.Domain(domain).name)
    return to_mont(o.hash_to_scalar(o.tag_input([o.Absorb(length), o.Squeeze(out_len)], dsep)))


def truncate(rows):
    """finalize_truncated's rows from finalize()'s: canonical value & (2^250 - 1) as raw limbs"""
    vals = [int(v) & ((1 << 250) - 1) for v in from_mont(rows.reshape(-1, 4))]
    return np.array([[(v >> (64 * k)) & ((1 << 64) - 1) for k in range(4)] for v in vals], dtype=np.uint64).reshape(rows.shape)


def oracle_mixed(mode, data, offsets, out_offsets, items=None):
    """{item: expected (out_len, 4) rows}, the C oracle's digest per (domain, len, out_len) group"""
    offsets, out_offsets = np.asarray(offsets, dtype=np.int64), np.asarray(out_offsets, dtype=np.int64)
    items = np.arange(len(mode)) if items is None else np.asarray(items)
    lens = offsets[items + 1] - offsets[items]
    ols = out_offsets[items + 1] - out_offsets[items]
    doms = np.asarray(mode)[items] & 3
    want = {}
    for key in set(zip(doms.tolist(), lens.tolist(), ols.tolist())):
        d, L, ol = key
        sel = items[(doms == d) & (lens == L) & (ols == ol)]
        rows = c_oracle.digest(otag(d, L, ol), data[offsets[sel][:, None] + np.arange(L)[None, :]], L, ol)
        for i, r in zip(sel, rows):
            want[int(i)] = truncate(r) if mode[i] & T else r
    return want


def check_rows(got, want, out_offsets):
    for i, w in want.items():
        assert np.array_equal(got[out_offsets[i]:out_offsets[i + 1]], w), i


def call(engine, mem, mode, data, offsets, out_offsets, **kw):
    got = engine.hash_batch_mixed(to_mem(mode, mem, np.uint8), to_mem(data, mem), to_mem(offsets, mem),
                                  to_mem(out_offsets, mem), async_=mem == "device-async", **kw)
    if mem == "device-async":
        engine.sync()
    return host(got)


def every_combination(rng, lead=0, out_lead=0):
    """every valid domain x {finalize, truncated} x len x out_len, shuffled, after `lead` / `out_lead` unused rows"""
    lens_set, outs_set = list(range(1, 10)) + [63, 64, 65], list(range(1, 10)) + [16, 17]
    items = [(d | t, L, ol) for d in range(4) for t in (0, T) for L in lens_set for ol in outs_set
             if d not in ARITY or (L == ARITY[d] and ol == 1)]
    items = [items[k] for k in rng.permutation(len(items))]
    mode = np.array([m for m, _, _ in items], dtype=np.uint8)
    offsets = bm.csr([L for _, L, _ in items]) + np.uint64(lead)
    out_offsets = bm.csr([ol for _, _, ol in items]) + np.uint64(out_lead)
    return mode, random_limbs_fast(rng, int(offsets[-1])), offsets, out_offsets


@pytest.mark.parametrize("mem", MEMS)
def test_every_combination_matches_oracle(engine, mem):
    mode, data, offsets, out_offsets = every_combination(np.random.default_rng(1))
    got = call(engine, mem, mode, data, offsets, out_offsets)
    assert got.shape == (int(out_offsets[-1]), 4)
    check_rows(got, oracle_mixed(mode, data, offsets, out_offsets), out_offsets)
    assert engine.last_mixed_rejected() == 0


@pytest.mark.parametrize("mem", MEMS)
def test_slice_of_larger_csr_arrays(engine, mem):
    """offsets[0] = 7 and out_offsets[0] = 5: rows before them are neither read as input nor written"""
    mode, data, offsets, out_offsets = every_combination(np.random.default_rng(2), lead=7, out_lead=5)
    n_out = int(out_offsets[-1]) + 3
    out = to_mem(np.full((n_out, 4), 0xabab, dtype=np.uint64), "host" if mem == "host" else "device")
    engine.hash_batch_mixed(to_mem(mode, mem, np.uint8), to_mem(data, mem), to_mem(offsets, mem), to_mem(out_offsets, mem),
                            out=out, async_=mem == "device-async")
    engine.sync()
    got = host(out)
    assert (got[:5] == 0xabab).all() and (got[-3:] == 0xabab).all()
    check_rows(got, oracle_mixed(mode, data, offsets, out_offsets), out_offsets)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_equal_to_the_existing_calls(engine, mem):
    """finalized items = p252_hash_batch_varlen per (domain, out_len); truncated = p252_hash_batch_truncated per
    (domain, len, out_len) -- the status quo arm of the benchmark"""
    rng = np.random.default_rng(3)
    n = 6000
    mode = rng.choice([0, 1, 2, 3, T, T | 1, T | 2, T | 3], n).astype(np.uint8)
    lens = np.where((mode & 3) == 0, 4, np.where((mode & 3) == 1, 2, rng.integers(1, 40, n)))
    out_lens = np.where((mode & 3) < 2, 1, rng.integers(1, 12, n))
    offsets, out_offsets = bm.csr(lens), bm.csr(out_lens)
    data = random_limbs_fast(rng, int(offsets[-1]))
    got = call(engine, mem, mode, data, offsets, out_offsets)
    assert np.array_equal(got, bm.status_quo_host(engine, bm.groups(mode, lens, out_lens), data, offsets, out_offsets))
    items = rng.choice(n, 200, replace=False)
    check_rows(got, oracle_mixed(mode, data, offsets, out_offsets, items), out_offsets)


def test_finalize_batch_front_end(engine):
    rng = np.random.default_rng(4)
    hashes, trunc = [], []
    for k in range(300):
        d = pb.Domain(int(rng.integers(0, 4)))
        total = ARITY.get(int(d), int(rng.integers(1, 30)))
        cuts = np.sort(rng.integers(1, total + 1, int(rng.integers(0, 3))))   # several update() chunks, none empty
        h = pb.Hash(d, engine)
        h.output_len(int(rng.integers(1, 7)))                                  # honoured for Domain::Other only
        for a, b in zip(np.concatenate([[0], cuts]), np.concatenate([cuts, [total]])):
            if b > a:
                h.update(random_limbs_fast(rng, int(b - a)))
        hashes.append(h)
        trunc.append(bool(rng.integers(0, 2)))
    got = pb.Hash.finalize_batch(hashes, truncated=trunc, engine=engine)
    for h, t, g in zip(hashes, trunc, got):
        assert np.array_equal(g, h.finalize_truncated() if t else h.finalize())
    assert all(np.array_equal(a, h.finalize()) for a, h in zip(pb.finalize_batch(hashes[:20], engine=engine), hashes))


def rejected_batch(rng):
    """a valid batch of 300 items, then one item edited to break each rule; -> descriptors and the bounds"""
    n = 300
    mode = rng.choice([2, 3, T | 2, T | 3], n).astype(np.uint8)
    lens, out_lens = rng.integers(1, 10, n), rng.integers(1, 6, n)
    mode[40], lens[40] = 0, 3                                  # rule 4: Merkle4 of 3 scalars
    mode[41], lens[41], out_lens[41] = 1, 2, 2                 # rule 4: Merkle2 with 2 outputs
    mode[90], lens[90] = 3, 12                                 # rule 6: len > max_len 10
    out_lens[95] = 8                                           # rule 6: out_len > max_out_len 6
    offsets, out_offsets = bm.csr(lens).astype(np.int64), bm.csr(out_lens).astype(np.int64)
    n_scalars, n_out = int(offsets[-1]), int(out_offsets[-1])
    mode[10] |= 0x04                                           # rule 1: an unknown mode bit
    offsets[21] = offsets[20] - 1                              # rule 2: item 20 decreasing (item 21 grows)
    offsets[-1] = n_scalars + 3                                # rule 2: the last item ends past n_scalars
    out_offsets[31] = out_offsets[30] - 1                      # rule 3: item 30 decreasing (overlaps item 29)
    out_offsets[-2] = n_out + 1                                # rule 3: item 298 ends past n_out
    offsets[51] = offsets[50]                                  # rule 5: len 0
    out_offsets[61] = out_offsets[60]                          # rule 5: out_len 0
    return mode, offsets.astype(np.uint64), out_offsets.astype(np.uint64), n_scalars, n_out


def item_status(mode, offsets, out_offsets, i, n_scalars, n_out, max_len, max_out_len):
    """the header's item checks, in order: 0 = valid, else the p252_status"""
    a, b, oa, ob = (int(v) for v in (offsets[i], offsets[i + 1], out_offsets[i], out_offsets[i + 1]))
    m = int(mode[i])
    if m & ~0x83:
        return -1
    if a > b or b > n_scalars or oa > ob or ob > n_out:
        return -1
    if (m & 3) in ARITY and (b - a != ARITY[m & 3] or ob - oa != 1):
        return 1
    if a == b or oa == ob:
        return 2
    return -1 if b - a > max_len or ob - oa > max_out_len else 0


@pytest.mark.parametrize("mem", ["device", "device-async"])
def test_device_rejections(engine, mem):
    rng = np.random.default_rng(5)
    mode, offsets, out_offsets, n_scalars, n_out = rejected_batch(rng)
    n = len(mode)
    status = [item_status(mode, offsets, out_offsets, i, n_scalars, n_out, 10, 6) for i in range(n)]
    bad = [i for i in range(n) if status[i]]
    assert {10, 20, 30, 40, 41, 50, 60, 90, 95, 298, 299} <= set(bad)
    full = random_limbs_fast(rng, n_scalars + 64)              # the tensor is longer than the n_scalars passed
    G = 8                                                      # guard rows before and after out
    out_full = to_mem(np.full((n_out + 2 * G, 4), 0xcdcd, dtype=np.uint64), "device")
    engine.hash_batch_mixed(to_mem(mode, mem, np.uint8), to_mem(full, mem)[:n_scalars], to_mem(offsets, mem),
                            to_mem(out_offsets, mem), max_len=10, max_out_len=6, out=out_full[G:G + n_out],
                            async_=mem == "device-async")
    engine.sync()
    assert engine.last_mixed_rejected() == len(bad)
    got = host(out_full)
    assert (got[:G] == 0xcdcd).all() and (got[G + n_out:] == 0xcdcd).all()
    got = got[G:G + n_out]
    ranges = {i: (int(out_offsets[i]), int(out_offsets[i + 1])) for i in range(n)
              if out_offsets[i] <= out_offsets[i + 1] <= n_out}  # valid output ranges: rows, zero rows
    cover = np.zeros(n_out, dtype=np.int64)
    for a, b in ranges.values():
        cover[a:b] += 1
    assert (got[cover == 0] == 0xcdcd).all()                   # nothing outside the valid ranges
    good = [i for i in range(n) if not status[i]]
    want = oracle_mixed(mode, full, offsets, out_offsets, good)
    for i, (a, b) in ranges.items():
        keep = cover[a:b] == 1                                 # rows where valid ranges overlap are unspecified
        if status[i]:
            assert not got[a:b][keep].any(), i
        else:
            assert np.array_equal(got[a:b][keep], want[i][keep]), i


def test_host_refusals_lowest_index_decides(engine):
    rng = np.random.default_rng(6)
    mode, offsets, out_offsets, n_scalars, n_out = rejected_batch(rng)
    data = random_limbs_fast(rng, n_scalars)
    n = len(mode)
    exc = {-1: pb.EngineError, 1: pb.IOPatternViolation, 2: pb.InvalidIOPattern}
    for lo in (0, 11, 21, 31, 42, 51, 61, 91, 96, 299):        # the batch from item lo: its first bad item decides
        st = [item_status(mode[lo:], offsets[lo:], out_offsets[lo:], i, n_scalars, n_out, 10, 6) for i in range(n - lo)]
        first = next(s for s in st if s)
        out = np.full((n_out, 4), 0xabab, dtype=np.uint64)
        with pytest.raises(exc[first]) as ei:
            engine.hash_batch_mixed(mode[lo:], data, offsets[lo:], out_offsets[lo:], max_len=10, max_out_len=6, out=out)
        if first == -1:
            assert ei.value.code == -1
        assert (out == 0xabab).all(), lo
    # batch checks
    m, d, off, oo = every_combination(rng)
    for kw in ({"max_len": 0}, {"max_len": pb._native.VARLEN_MAX_LEN + 1}, {"max_out_len": 0},
               {"max_out_len": pb._native.VARLEN_MAX_LEN + 1}):
        for mem in ("host", "device"):
            with pytest.raises(pb.EngineError):
                engine.hash_batch_mixed(to_mem(m, mem, np.uint8), to_mem(d, mem), to_mem(off, mem), to_mem(oo, mem), **kw)


def test_host_multi_chunk_and_injected_fault(engine):
    """items with 65536 output rows (2 MiB each) bound the chunks by output bytes: the input is tiny"""
    rng = np.random.default_rng(7)
    n = 3000
    mode = rng.choice([3, T | 3], n).astype(np.uint8)
    lens, out_lens = rng.integers(1, 20, n), rng.integers(1, 5, n)
    huge = rng.choice(n, 40, replace=False)
    out_lens[huge] = pb._native.VARLEN_MAX_LEN
    offsets, out_offsets = bm.csr(lens), bm.csr(out_lens)
    assert int(out_offsets[-1]) * 32 > 3 * (24 << 20)
    data = random_limbs_fast(rng, int(offsets[-1]))
    want = call(engine, "device", mode, data, offsets, out_offsets)
    assert np.array_equal(call(engine, "host", mode, data, offsets, out_offsets), want)
    lib, ctx = pb._native.lib(), engine._ctx
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError) as ei:
        engine.hash_batch_mixed(mode, data, offsets, out_offsets)
    assert "injected" in str(ei.value)
    assert np.array_equal(call(engine, "host", mode, data, offsets, out_offsets), want)   # context still usable
    items = np.concatenate([huge[:2], rng.choice(n, 62, replace=False)])
    check_rows(want, oracle_mixed(mode, data, offsets, out_offsets, items), out_offsets)


@pytest.mark.parametrize("mem", MEMS)
def test_empty_batch_runs_nothing(engine, mem):
    before = engine.launch_count
    got = call(engine, mem, np.zeros(0), np.zeros((0, 4)), np.zeros(1), np.zeros(1))
    assert got.shape == (0, 4)
    got = call(engine, mem, np.zeros(0), random_limbs_fast(np.random.default_rng(8), 9), np.array([5]), np.array([3]))
    assert got.shape == (3, 4)
    assert engine.launch_count == before and engine.last_mixed_rejected() == 0


def test_full_size_node_mix(engine):
    mode, lens, out_lens = bm.workload(1 << 20)
    offsets, out_offsets = bm.csr(lens), bm.csr(out_lens)
    rng = np.random.default_rng(9)
    data = random_limbs_fast(rng, int(offsets[-1]))
    got = call(engine, "device", mode, data, offsets, out_offsets)
    assert engine.last_mixed_rejected() == 0
    assert np.array_equal(got, bm.status_quo_host(engine, bm.groups(mode, lens, out_lens), data, offsets, out_offsets))
    check_rows(got, oracle_mixed(mode, data, offsets, out_offsets, rng.choice(1 << 20, 4096, replace=False)), out_offsets)


def test_c_smoke_and_cpp_mirror_on_the_device():
    from test_hash_mixed_cpu import c_smoke, cpp_mirror
    res = c_smoke()
    assert res.returncode == 0 and "HASH_MIXED_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)
    res = cpp_mirror()
    assert res.returncode == 0 and res.stdout.strip() == "hash_mixed mirror ok", (res.returncode, res.stdout, res.stderr)
