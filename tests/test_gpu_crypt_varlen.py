"""GPU (-m gpu): variable-length encrypt / decrypt batches (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen)
against the C oracle's encrypt per length group, with tags from hades_oracle (not from the library); equality with the
fixed-length p252_encrypt_batch / p252_decrypt_batch; tampering; slices of a larger CSR; device-side rejections with
canaries around the output; host-side refusals; host and device buffers, async calls, tag-table growth, alternation with
varlen digests; multi-chunk host batches with fault injection and staging wipe; a full-size batch; the module front ends.
Both kernels (the two-parameter `engine` fixture: lane-split for small batches, and the throughput kernel only)."""
import ctypes
import functools

import numpy as np
import pytest

import c_oracle
import hades_oracle as o
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import random_limbs_fast, to_mont

pytestmark = pytest.mark.gpu

MEMS = ["host", "device"]
SENT = 0x5a5a5a5a5a5a5a5a


def host(x):
    if hasattr(x, "is_cuda"):
        a = x.cpu().numpy()
        return a.view(np.uint64) if a.dtype == np.int64 else a
    return np.asarray(x)


def to_mem(a, mem):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if mem == "host":
        return a
    import torch
    return torch.from_numpy(a.view(np.int64)).cuda()


@functools.lru_cache(maxsize=None)
def otag(L):
    """tag of encrypt / decrypt for message length L, from the oracle's restatement"""
    pat = [o.Absorb(2), o.Absorb(1), o.Squeeze(L), o.Absorb(L), o.Squeeze(1)]
    return to_mont(o.hash_to_scalar(o.tag_input(pat, o.Domain.Encryption)))


def batch(rng, lens, lead=0):
    """messages of the given lengths back to back after `lead` unused scalars, with secrets and nonces"""
    n = len(lens)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(lead)
    return (random_limbs_fast(rng, int(offsets[-1])), offsets, random_limbs_fast(rng, (n, 2)),
            random_limbs_fast(rng, n))


def oracle_check(cipher, data, offsets, uv, nonce, rows=None):
    """every row in `rows` of the cipher CSR (packed from 0) equals the C oracle's encrypt of its message"""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = offsets.shape[0] - 1
    rows = np.arange(n) if rows is None else np.asarray(rows)
    lens = offsets[rows + 1] - offsets[rows]
    coff = offsets - offsets[0] + np.arange(n + 1)
    for L in np.unique(lens):
        sel = rows[lens == L]
        want = c_oracle.encrypt(otag(int(L)), data[offsets[sel][:, None] + np.arange(L)], int(L), uv[sel], nonce[sel])
        got = cipher[coff[sel][:, None] + np.arange(L + 1)]
        assert np.array_equal(got, want), int(L)


def coop_max():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 24


def raw_decrypt(engine, ciph, n_scalars, offs, n, max_len, uv, nonce, msg, ok, flags):
    """p252_decrypt_batch_varlen on caller-owned pointers (numpy arrays or tensors) -> (rc, n_failed, n_rejected)"""
    ptr = lambda x: x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data
    failed, rejected = ctypes.c_size_t(99), ctypes.c_size_t(99)
    rc = _native.lib().p252_decrypt_batch_varlen(engine._ctx, ptr(ciph), n_scalars, ptr(offs), n, max_len, ptr(uv),
                                                 ptr(nonce), ptr(msg), ptr(ok), ctypes.byref(failed),
                                                 ctypes.byref(rejected), flags)
    return rc, failed.value, rejected.value


# 1 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_every_length_shuffled_matches_oracle_and_round_trips(engine, mem):
    rng = np.random.default_rng(1)
    lens = rng.permutation(np.repeat(np.arange(1, 129), 3))
    data, offsets, uv, nonce = batch(rng, lens, lead=5)
    cipher, coff = engine.encrypt_batch_varlen(to_mem(data, mem), to_mem(offsets, mem), to_mem(uv, mem), to_mem(nonce, mem))
    assert engine.last_crypt_rejected() == 0
    cipher, coff = host(cipher), host(coff)
    assert np.array_equal(coff, pb.cipher_offsets(offsets))
    oracle_check(cipher, data, offsets, uv, nonce)
    msg, moff, ok = engine.decrypt_batch_varlen(to_mem(cipher, mem), to_mem(coff, mem), to_mem(uv, mem), to_mem(nonce, mem))
    assert host(ok).all() and engine.last_decrypt_failures() == 0 and engine.last_crypt_rejected() == 0
    assert np.array_equal(host(moff), offsets - offsets[0])
    assert np.array_equal(host(msg)[:int(offsets[-1] - offsets[0])], data[int(offsets[0]):])


# 2 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_equal_lengths_bit_identical_to_fixed_length_calls(engine, mem):
    rng = np.random.default_rng(2)
    cm = coop_max()
    for L in (1, 2, 4, 5, 42):
        for n in (cm - 1, cm, cm + 1, 4096):
            data, offsets, uv, nonce = batch(rng, np.full(n, L))
            want = engine.encrypt_batch(data.reshape(n, L, 4), uv, nonce)
            cipher, _ = engine.encrypt_batch_varlen(to_mem(data, mem), to_mem(offsets, mem), to_mem(uv, mem), to_mem(nonce, mem))
            assert np.array_equal(host(cipher).reshape(n, L + 1, 4), want), (L, n)
            bad = want.copy()
            bad[::7, L, 0] ^= np.uint64(1)                         # every 7th authentication scalar
            wm, wok = engine.decrypt_batch(bad, uv, nonce)
            coff = np.arange(n + 1, dtype=np.uint64) * np.uint64(L + 1)
            msg, _, ok = engine.decrypt_batch_varlen(to_mem(bad.reshape(-1, 4), mem), to_mem(coff, mem), to_mem(uv, mem),
                                                     to_mem(nonce, mem))
            assert np.array_equal(host(ok), wok) and np.array_equal(host(msg).reshape(n, L, 4), wm), (L, n)
            assert engine.last_decrypt_failures() == (n + 6) // 7


# 3 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_tampering_in_a_mixed_batch(engine, mem):
    rng = np.random.default_rng(3)
    n = 300
    data, offsets, uv, nonce = batch(rng, rng.integers(1, 21, n))
    cipher, coff = engine.encrypt_batch_varlen(data, offsets, uv, nonce)
    coff = coff.astype(np.int64)
    bad, buv, bnon = cipher.copy(), uv.copy(), nonce.copy()
    kinds = rng.permutation(n)[:100].reshape(5, 20)               # 20 items per kind
    for i in kinds[0]:
        bad[coff[i] + rng.integers(0, coff[i + 1] - coff[i] - 1), 1] ^= np.uint64(1 << 7)   # a message scalar
    for i in kinds[1]:
        bad[coff[i + 1] - 1, 0] ^= np.uint64(1)                   # the authentication scalar
    bnon[kinds[2], 2] ^= np.uint64(1 << 33)                        # the nonce
    buv[kinds[3], 0, 0] ^= np.uint64(2)                            # u
    buv[kinds[4], 1, 3] ^= np.uint64(1 << 20)                      # v
    msg, moff, ok = engine.decrypt_batch_varlen(to_mem(bad, mem), to_mem(coff.astype(np.uint64), mem), to_mem(buv, mem),
                                                to_mem(bnon, mem))
    msg, moff, ok = host(msg), host(moff).astype(np.int64), host(ok)
    tampered = np.zeros(n, dtype=bool)
    tampered[kinds.reshape(-1)] = True
    assert np.array_equal(ok, (~tampered).astype(np.uint8))
    assert engine.last_decrypt_failures() == 100
    for i in range(n):
        m = msg[moff[i]:moff[i + 1]]
        assert (not m.any()) if tampered[i] else np.array_equal(m, data[offsets[i]:offsets[i + 1]]), i


# 4 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_slice_of_a_larger_csr(engine, mem):
    rng = np.random.default_rng(4)
    data, offsets, uv, nonce = batch(rng, rng.integers(1, 40, 200))
    full, fcoff = engine.encrypt_batch_varlen(data, offsets, uv, nonce)
    lo, hi = 50, 150
    part, pcoff = engine.encrypt_batch_varlen(to_mem(data, mem), to_mem(offsets[lo:hi + 1], mem), to_mem(uv[lo:hi], mem),
                                              to_mem(nonce[lo:hi], mem))
    part, pcoff = host(part), host(pcoff)
    assert pcoff[0] == 0 and np.array_equal(pcoff, fcoff[lo:hi + 1] - fcoff[lo])
    assert np.array_equal(part[:int(pcoff[-1])], full[int(fcoff[lo]):int(fcoff[hi])])
    # and decrypting a slice of the cipher CSR gives the slice of the messages, packed from 0
    msg, moff, ok = engine.decrypt_batch_varlen(to_mem(full, mem), to_mem(fcoff[lo:hi + 1], mem), to_mem(uv[lo:hi], mem),
                                                to_mem(nonce[lo:hi], mem))
    assert host(ok).all()
    assert np.array_equal(host(msg)[:int(host(moff)[-1])], data[int(offsets[lo]):int(offsets[hi])])


# 5 ------------------------------------------------------------------------------------------------------------------
def valid_items(offsets, n_scalars, max_len, decrypt):
    """the item rules of the header, restated"""
    off = [int(v) for v in offsets]
    n = len(off) - 1
    a0, an = off[0], off[-1]
    lo, hi = (2, max_len + 1) if decrypt else (1, max_len)
    res = np.zeros(n, dtype=bool)
    for i in range(n):
        a, b = off[i], off[i + 1]
        v = a0 <= a <= b <= an <= n_scalars and lo <= b - a <= hi
        if decrypt:
            v = v and a - a0 >= i and an - b >= n - 1 - i
        res[i] = v
    return res


def test_device_rejections_encrypt(engine):
    import torch
    rng = np.random.default_rng(5)
    n = 400
    data, offsets, uv, nonce = batch(rng, rng.integers(1, 20, n))
    offsets = offsets.astype(np.int64)
    offsets[10] = offsets[9]                                  # item 9: length 0
    offsets[41] = offsets[40] + 25                            # item 40: length 25 > max_len 24
    offsets[100] = offsets[101] + 5                           # item 100: offsets decrease
    offsets = offsets.astype(np.uint64)
    ns = int(offsets[-1])
    valid = valid_items(offsets, ns, 24, False)
    assert not valid[[9, 40, 100]].any()
    rows, pad = ns + n, 64
    buf = torch.full((rows + 2 * pad, 4), SENT, dtype=torch.int64, device="cuda")
    dev = to_mem(np.concatenate([data, random_limbs_fast(rng, 32)]), "device")     # the tensor is longer than n_scalars
    cipher, coff = engine.encrypt_batch_varlen(dev[:ns], to_mem(offsets, "device"), to_mem(uv, "device"),
                                               to_mem(nonce, "device"), max_len=24, out=buf[pad:pad + rows])
    assert engine.last_crypt_rejected() == int((~valid).sum())
    b = host(buf)
    assert (b[:pad] == SENT).all() and (b[pad + rows:] == SENT).all()
    oracle_check(host(cipher), data, offsets, uv, nonce, rows=np.nonzero(valid)[0])
    # n_scalars shorter than the data the offsets describe: offsets[n] > n_scalars rejects every item, nothing written
    buf.fill_(SENT)
    engine.encrypt_batch_varlen(dev[:ns - 1], to_mem(offsets, "device"), to_mem(uv, "device"), to_mem(nonce, "device"),
                                max_len=24, out=buf[pad:pad + rows - 1])
    assert engine.last_crypt_rejected() == n and (host(buf) == SENT).all()


def test_device_rejections_decrypt(engine):
    import torch
    rng = np.random.default_rng(6)
    n = 400
    data, offsets, uv, nonce = batch(rng, rng.integers(1, 20, n))
    cipher, coff = engine.encrypt_batch_varlen(data, offsets, uv, nonce)
    orig = coff.astype(np.int64)
    c = orig.copy()
    c[1] = c[2] = c[0]                                        # items 0, 1 empty, so item 2 (length 2) would start its
    c[3] = c[0] + 2                                           #   message before the output (a - a0 < i)
    c[11] = c[10] + 1                                         # item 10: cipher length 1
    c[21] = c[20]                                             # item 20: cipher length 0
    c[51] = c[50] + 26                                        # item 50: length 26 > max_len + 1 = 25
    c[100] = c[101] + 3                                       # item 100: offsets decrease
    c[n - 1] = c[n] - 1                                       # item n-1: cipher length 1, item n-2 empty, so item
    c[n - 2] = c[n - 1]                                       #   n-3 (length 3) would end its message past the output
    c[n - 3] = c[n - 1] - 3                                   #   (an - b < n - 1 - i)
    c = c.astype(np.uint64)
    ns = cipher.shape[0]
    valid = valid_items(c, ns, 24, True)
    assert not valid[[0, 1, 2, 10, 20, 50, 100, n - 1, n - 2, n - 3]].any()
    # a valid item whose range the edits moved decrypts garbage: an authentication failure, not a rejection
    same = (c[:-1] == orig[:-1].astype(np.uint64)) & (c[1:] == orig[1:].astype(np.uint64))
    want_ok = valid & same
    rows, pad = ns - n, 64
    msg = torch.full((rows + 2 * pad, 4), SENT, dtype=torch.int64, device="cuda")
    ok = torch.full((n,), 0x77, dtype=torch.uint8, device="cuda")
    dc, doff = to_mem(cipher, "device"), to_mem(c, "device")
    duv, dnon = to_mem(uv, "device"), to_mem(nonce, "device")
    rc, failed, rejected = raw_decrypt(engine, dc, ns, doff, n, 24, duv, dnon, msg[pad:], ok, _native.MEM_DEVICE)
    assert rc == 0
    assert rejected == int((~valid).sum()) and failed == int((valid & ~same).sum())
    m = host(msg)
    assert (m[:pad] == SENT).all() and (m[pad + rows:] == SENT).all()
    assert np.array_equal(ok.cpu().numpy(), want_ok.astype(np.uint8))
    # with invalid items in the batch, the output ranges of valid neighbours may overlap (the rules only keep every
    # write inside the output): check the verified items whose range no other valid item touches
    moff = pb.message_offsets(c).astype(np.int64)
    cover = np.zeros(rows, dtype=np.int64)
    for i in np.nonzero(valid)[0]:
        cover[moff[i]:moff[i + 1]] += 1
    checked = 0
    for i in np.nonzero(want_ok)[0]:
        if (cover[moff[i]:moff[i + 1]] == 1).all():
            assert np.array_equal(m[pad + moff[i]:pad + moff[i + 1]], data[offsets[i]:offsets[i + 1]]), i
            checked += 1
    assert checked > n - 30


# 6 ------------------------------------------------------------------------------------------------------------------
def test_host_refusals_nothing_written(engine):
    rng = np.random.default_rng(7)
    n = 50
    data, offsets, uv, nonce = batch(rng, rng.integers(2, 10, n))
    offsets = offsets.astype(np.int64)
    lib = _native.lib()

    def refused(code, offs, n_scalars=None, decrypt=False, max_len=16):
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        ns = data.shape[0] if n_scalars is None else n_scalars
        out = np.full((data.shape[0] + n, 4), SENT, dtype=np.uint64)
        if decrypt:
            ok = np.full(n, 0x77, dtype=np.uint8)
            rc, _, _ = raw_decrypt(engine, data, ns, offs, n, max_len, uv, nonce, out, ok, _native.MEM_HOST)
            assert (ok == 0x77).all()
        else:
            rc = lib.p252_encrypt_batch_varlen(engine._ctx, data.ctypes.data, ns, offs.ctypes.data, n, max_len, uv.ctypes.data,
                                               nonce.ctypes.data, out.ctypes.data, None, _native.MEM_HOST)
        assert rc == code
        assert (out == SENT).all()

    INVALID_ARGUMENT, INVALID_IO_PATTERN = -1, 2
    for dec in (False, True):
        o2 = offsets.copy()
        o2[6] = o2[7] + 1
        refused(INVALID_ARGUMENT, o2, decrypt=dec)                              # decreasing offsets
        refused(INVALID_ARGUMENT, offsets, n_scalars=int(offsets[-1]) - 1, decrypt=dec)   # past n_scalars
        o2 = offsets.copy()
        o2[6] = o2[5]
        refused(INVALID_IO_PATTERN, o2, decrypt=dec)                            # length 0
        o2 = offsets.copy()
        o2[6] = o2[5] + 18
        refused(INVALID_ARGUMENT, o2, decrypt=dec)                              # length > max_len (+1)
        o2 = offsets.copy()
        o2[3] = o2[4] + 2                                                       # item 3 decreasing wins over ...
        o2[31] = o2[30]                                                         # ... item 30's length 0
        refused(INVALID_ARGUMENT, o2, decrypt=dec)
        refused(INVALID_ARGUMENT, offsets, decrypt=dec, max_len=0)              # batch checks
        refused(INVALID_ARGUMENT, offsets, decrypt=dec, max_len=_native.VARLEN_MAX_LEN + 1)
    o2 = offsets.copy()
    o2[6] = o2[5] + 1
    refused(INVALID_IO_PATTERN, o2, decrypt=True)                               # a cipher of length 1
    with pytest.raises(pb.InvalidIOPattern):
        pb.encrypt_batch_varlen([data[:3], data[:0]], uv[:2], nonce[:2], engine=engine)
    # device batch checks: misaligned data, and n >= 2^31
    dev = to_mem(data, "device")
    with pytest.raises(pb.EngineError):
        engine.encrypt_batch_varlen(dev.view(-1)[1:1 + 4 * 40].view(40, 4), to_mem(np.arange(3, dtype=np.uint64), "device"),
                                    to_mem(uv[:2], "device"), to_mem(nonce[:2], "device"), max_len=4)
    assert lib.p252_encrypt_batch_varlen(engine._ctx, data.ctypes.data, data.shape[0], offsets.ctypes.data, 1 << 31, 16,
                                         uv.ctypes.data, nonce.ctypes.data, data.ctypes.data, None, _native.MEM_HOST) == -1


# 7 ------------------------------------------------------------------------------------------------------------------
def test_host_equals_device_empty_and_async(engine):
    rng = np.random.default_rng(8)
    data, offsets, uv, nonce = batch(rng, rng.integers(1, 100, 3000))
    h, hoff = engine.encrypt_batch_varlen(data, offsets, uv, nonce)
    d, doff = engine.encrypt_batch_varlen(to_mem(data, "device"), to_mem(offsets, "device"), to_mem(uv, "device"),
                                          to_mem(nonce, "device"))
    assert np.array_equal(h, host(d)) and np.array_equal(hoff, host(doff))
    dev = [to_mem(x, "device") for x in (data, offsets, uv, nonce)]      # alive until the stream has read them
    a, aoff = engine.encrypt_batch_varlen(*dev, max_len=99, async_=True)
    m, moff, ok = engine.decrypt_batch_varlen(a, aoff, dev[2], dev[3], max_len=99, async_=True)
    engine.sync()
    assert np.array_equal(h, host(a)) and host(ok).all() and engine.last_decrypt_failures() == 0
    assert np.array_equal(host(m), data)
    hm, hmoff, hok = engine.decrypt_batch_varlen(h, hoff, uv, nonce)
    assert np.array_equal(hm, data) and hok.all()
    for mem in MEMS:                                          # n = 0
        z = to_mem(np.zeros((0, 4)), mem)
        c, coff = engine.encrypt_batch_varlen(to_mem(data, mem), to_mem(offsets[5:6], mem), to_mem(np.zeros((0, 2, 4)), mem), z)
        assert host(coff).tolist() == [0]
        m, moff, ok = engine.decrypt_batch_varlen(to_mem(data, mem), to_mem(offsets[5:6], mem),
                                                  to_mem(np.zeros((0, 2, 4)), mem), z)
        assert host(moff).tolist() == [0] and tuple(ok.shape) == (0,)


def test_tag_table_growth_and_alternation_with_varlen_digests(engine):
    """A fresh context: the encryption table grows between async calls while varlen digests of other max_len values
    rebuild their own table in between; every result is checked against the oracle."""
    def digest_oracle(data, offsets):
        lens = np.diff(offsets.astype(np.int64))
        want = np.zeros((lens.shape[0], 2, 4), dtype=np.uint64)
        for L in np.unique(lens):
            sel = np.nonzero(lens == L)[0]
            tag = to_mont(o.hash_to_scalar(o.tag_input([o.Absorb(int(L)), o.Squeeze(2)], o.Domain.Other)))
            want[sel] = c_oracle.digest(tag, data[offsets[sel].astype(np.int64)[:, None] + np.arange(L)], int(L), 2)
        return want

    rng = np.random.default_rng(9)
    eng = pb.Engine(0)
    try:
        calls = []
        for lens in (rng.integers(1, 9, 2000), rng.integers(1, 301, 2000), rng.integers(1, 301, 50), rng.integers(1, 40, 500)):
            data, offsets, uv, nonce = batch(rng, lens)
            dev = [to_mem(x, "device") for x in (data, offsets, uv, nonce)]   # alive until the stream has read them
            dig = eng.hash_batch_varlen(pb.Domain.Other, dev[0], dev[1], 2, max_len=int(lens.max()) + 3, async_=True)
            c, coff = eng.encrypt_batch_varlen(*dev, max_len=int(lens.max()), async_=True)
            calls.append((data, offsets, uv, nonce, c, dig, dev))
        eng.sync()
        for data, offsets, uv, nonce, c, dig, _ in calls:
            oracle_check(host(c), data, offsets, uv, nonce)
            assert np.array_equal(host(dig), digest_oracle(data, offsets))
    finally:
        eng.close()


# 8 ------------------------------------------------------------------------------------------------------------------
def test_host_multi_chunk_fault_and_staging_wipe(engine):
    rng = np.random.default_rng(10)
    lens = rng.integers(32, 97, 40000)                        # ~2.6 M scalars: four chunks of <= 24 MiB input
    data, offsets, uv, nonce = batch(rng, lens)
    assert data.nbytes > 3 * (24 << 20)
    lib, ctx = _native.lib(), engine._ctx
    nz = ctypes.c_size_t(1)
    want, wcoff = engine.encrypt_batch_varlen(to_mem(data, "device"), to_mem(offsets, "device"), to_mem(uv, "device"),
                                              to_mem(nonce, "device"))
    want, wcoff = host(want), host(wcoff)
    got, _ = engine.encrypt_batch_varlen(data, offsets, uv, nonce)
    assert np.array_equal(got, want)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    out = np.zeros_like(want)
    with pytest.raises(pb.EngineError) as ei:
        engine.encrypt_batch_varlen(data, offsets, uv, nonce, out=out)
    assert "injected" in str(ei.value)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    got, _ = engine.encrypt_batch_varlen(data, offsets, uv, nonce)          # context still usable
    assert np.array_equal(got, want)
    msg, _, ok = engine.decrypt_batch_varlen(want, wcoff, uv, nonce)
    assert ok.all() and np.array_equal(msg, data)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.decrypt_batch_varlen(want, wcoff, uv, nonce)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    oracle_check(want, data, offsets, uv, nonce, rows=rng.choice(lens.shape[0], 64, replace=False))


# 9 ------------------------------------------------------------------------------------------------------------------
def test_full_size_2e20_items(engine):
    rng = np.random.default_rng(12)
    lens = rng.integers(1, 17, 1 << 20)
    data, offsets, uv, nonce = batch(rng, lens)
    d_uv, d_non = to_mem(uv, "device"), to_mem(nonce, "device")
    c, coff = engine.encrypt_batch_varlen(to_mem(data, "device"), to_mem(offsets, "device"), d_uv, d_non, max_len=16)
    assert engine.last_crypt_rejected() == 0
    oracle_check(host(c), data, offsets, uv, nonce, rows=rng.choice(1 << 20, 4096, replace=False))
    m, moff, ok = engine.decrypt_batch_varlen(c, coff, d_uv, d_non, max_len=16)
    assert bool(ok.all()) and engine.last_decrypt_failures() == 0
    assert np.array_equal(host(m), data)


# 10 -----------------------------------------------------------------------------------------------------------------
def test_module_front_ends(engine):
    rng = np.random.default_rng(11)
    n = 200
    items = [random_limbs_fast(rng, int(k)) for k in rng.integers(1, 30, n)]
    uv, nonce = random_limbs_fast(rng, (n, 2)), random_limbs_fast(rng, n)
    ciphers = pb.encrypt_batch_varlen(items, uv, nonce, engine=engine)
    assert isinstance(ciphers, list) and len(ciphers) == n
    for i in (0, 57, 199):                                    # = encrypt() item by item
        assert np.array_equal(ciphers[i], pb.encrypt(items[i], uv[i], nonce[i], engine))
    data, offsets, _ = pb.pack_varlen(items)
    oracle_check(np.concatenate(ciphers), data, offsets, uv, nonce)
    ciphers[3] = ciphers[3].copy()
    ciphers[3][0, 0] ^= np.uint64(1)
    msgs, ok = pb.decrypt_batch_varlen(ciphers, uv, nonce, engine=engine)
    assert ok.tolist() == [0 if i == 3 else 1 for i in range(n)]
    assert all(np.array_equal(msgs[i], items[i]) for i in range(n) if i != 3) and not msgs[3].any()
    # a (data, offsets) pair of device tensors works as well
    c, coff = pb.encrypt_batch_varlen((to_mem(data, "device"), to_mem(offsets, "device")), to_mem(uv, "device"),
                                      to_mem(nonce, "device"), engine=engine)
    assert np.array_equal(host(c), np.concatenate(pb.encrypt_batch_varlen(items, uv, nonce, engine=engine)))
