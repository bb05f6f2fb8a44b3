"""Stealth addresses on the device (p252_stealth_address_batch / p252_stealth_owns_batch) against the model of
stealth_oracle.py (affine complete addition, double-and-add, the Python Hades), against the existing calls they are
built from (fixed_base_batch, encrypt_batch_ephemeral, dhke_batch -> hash_batch_truncated -> fixed_base_batch), and the
receiver's scan against the construction of the notes."""
import ctypes
import functools

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs

pytestmark = pytest.mark.gpu

R_EDGES = [0, 1, 7, 8, 9, 15, 16, int("7" * 62, 16), int("8" * 62, 16), int("8" * 63, 16), (1 << 248) - 8,
           jo.R_J - 1, (1 << 251) + 1, (1 << 251) + 0x8888]
CANARY = 0xA5A5A5A5A5A5A5A5
G = jo.GENERATOR


def to_mem(a, mem):
    if mem == "host":
        return a
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a if a.dtype == np.uint8 else a.view(np.int64)).cuda()


def host(x):
    if isinstance(x, np.ndarray):
        return x
    a = x.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def mont(pt):
    return jo.points_mont([pt])[0]


def s_int(row):
    return sum(int(row[k]) << (64 * k) for k in range(4))


@functools.lru_cache(maxsize=None)
def mul(k, pt):
    return jo.mul(k, pt)


@functools.lru_cache(maxsize=None)
def model(r, A, B):
    """(R, note_pk) rows as the device writes them: zeroed for an invalid item; and ok"""
    if not (0 <= r < jo.R_J) or not jo.on_curve(A) or not jo.on_curve(B):
        return (0, 0), (0, 0), 0
    return mul(r, G), jo.add(mul(so.hash_point(mul(r, A)), G), B), 1


def expect(rs, As, Bs):
    rows = [model(r, A, B) for r, A, B in zip(rs, As, Bs)]
    R = jo.points_mont([x[0] for x in rows])
    pk = jo.points_mont([x[1] for x in rows])
    ok = np.array([x[2] for x in rows], dtype=np.uint8)
    R[ok == 0] = 0
    pk[ok == 0] = 0
    return R, pk, ok


@functools.lru_cache(maxsize=None)
def classes():
    """a point of every order class: identity, order 2, 4 and 8, G, a subgroup and a full-group point"""
    rng = np.random.default_rng(100)
    ident, o2, o4, _, o8 = jo.small_order_points(rng)
    return (ident, o2, o4, o8, G, jo.random_subgroup_point(rng), jo.random_point(rng))


@functools.lru_cache(maxsize=None)
def receiver(seed):
    rng = np.random.default_rng(seed)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    return a, b, mul(a, G), mul(b, G)


def notes(rng, n, A, B):
    """n notes to (A, B): (r rows, R rows, note_pk rows) from the model"""
    r = [jo.random_secret(rng) for _ in range(n)]
    R, pk, ok = expect(r, [A] * n, [B] * n)
    assert ok.all()
    return r, R, pk


# 1 ---- the sender against the model: edge r x every order class of A and B ------------------------------------------
@pytest.mark.parametrize("mem,async_", [("host", False), ("device", False), ("device", True)])
@pytest.mark.parametrize("n_public", ["one", "n"])
def test_sender_against_model(engine, mem, async_, n_public):
    cls = classes()
    gm = mont(G)
    if n_public == "n":
        rs, As, Bs = [], [], []
        for i, r in enumerate(R_EDGES):
            for k in range(len(cls)):
                rs.append(r)
                As.append(cls[k])
                Bs.append(cls[(k + i) % len(cls)])
        calls = [(rs, As, Bs)]
    else:
        calls = [(R_EDGES, [cls[k]] * len(R_EDGES), [cls[(k + 3) % len(cls)]] * len(R_EDGES)) for k in range(len(cls))]
    for rs, As, Bs in calls:
        wR, wpk, wok = expect(rs, As, Bs)
        k = 1 if n_public == "one" else len(rs)
        R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs(rs), mem), gm, to_mem(jo.points_mont(As[:k]), mem),
                                                 to_mem(jo.points_mont(Bs[:k]), mem), async_=async_)
        if async_:
            engine.sync()
        assert np.array_equal(host(ok), wok) and np.array_equal(host(R), wR) and np.array_equal(host(pk), wpk)
        assert engine.last_stealth_invalid() == 0
    R1, pk1 = pb.stealth_address(5, gm, mont(cls[5]), mont(cls[6]), engine=engine)
    assert jo.points_from_mont(np.stack([R1, pk1])) == list(model(5, cls[5], cls[6])[:2])


# 2 ---- the sender against the calls it is built from ------------------------------------------------------------------
def test_sender_equals_existing_calls_large(engine):
    import torch
    rng = np.random.default_rng(2)
    n = 1 << 18
    r = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    r[:, 3] %= np.uint64(jo.R_J >> 192)
    keys = [receiver(s) for s in (11, 12, 13)]
    pick = rng.integers(0, 3, n)
    A = jo.points_mont([k[2] for k in keys])[pick]
    B = jo.points_mont([k[3] for k in keys])[pick]
    gm = mont(G)
    dr, dA, dB = to_mem(r, "device"), to_mem(A, "device"), to_mem(B, "device")
    R, pk, ok = engine.stealth_address_batch(dr, gm, dA, dB)
    R1, ok1 = engine.fixed_base_batch(dr, gm)
    _, R2, ok2 = engine.encrypt_batch_ephemeral(to_mem(np.zeros((n, 1, 4), np.uint64), "device"), dr, gm, dA,
                                                to_mem(np.zeros((n, 4), np.uint64), "device"))
    shared, oks = engine.dhke_batch(dr, dA)
    h = engine.hash_batch_truncated(pb.Domain.Other, shared)
    hG, okh = engine.fixed_base_batch(h.reshape(n, 4).contiguous(), gm)
    torch.cuda.synchronize()
    assert host(ok).all() and host(ok1).all() and host(ok2).all() and host(oks).all() and host(okh).all()
    assert torch.equal(R, R1) and torch.equal(R, R2)
    assert engine.last_stealth_invalid() == 0
    rows = rng.choice(n, 16, replace=False)
    hg, pkh, Bh = jo.points_from_mont(host(hG)[rows]), jo.points_from_mont(host(pk)[rows]), jo.points_from_mont(B[rows])
    for i in range(len(rows)):
        assert jo.add(hg[i], Bh[i]) == pkh[i]                     # + B, applied in the model
    wR, wpk, _ = expect([s_int(r[i]) for i in rows[:4]], [keys[pick[i]][2] for i in rows[:4]],
                        [keys[pick[i]][3] for i in rows[:4]])
    assert np.array_equal(host(R)[rows[:4]], wR) and np.array_equal(host(pk)[rows[:4]], wpk)


# 3 ---- round trips: three receivers' notes mixed in one batch --------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_each_receiver_owns_exactly_its_notes(engine, mem):
    rng = np.random.default_rng(3)
    n = 90
    keys = [receiver(s) for s in (21, 22, 23)]
    who = rng.integers(0, 3, n)
    r = [jo.random_secret(rng) for _ in range(n)]
    gm = mont(G)
    A = jo.points_mont([keys[w][2] for w in who])
    B = jo.points_mont([keys[w][3] for w in who])
    R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs(r), mem), gm, to_mem(A, mem), to_mem(B, mem))
    assert host(ok).all()
    for k, (a, b, Ak, Bk) in enumerate(keys):
        owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(Bk), gm, R, pk)
        assert np.array_equal(host(owned), (who == k).astype(np.uint8))
        assert engine.last_stealth_owned() == int((who == k).sum()) and engine.last_stealth_invalid() == 0
    a, b, Ak, Bk = keys[0]
    i = int(np.flatnonzero(who == 0)[0])
    assert pb.owns(a, mont(Bk), gm, host(R)[i], host(pk)[i], engine=engine) is True
    assert pb.owns(keys[1][0], mont(keys[1][3]), gm, host(R)[i], host(pk)[i], engine=engine) is False


@pytest.mark.parametrize("async_", [False, True])
def test_scan_counts_on_device(engine, async_):
    rng = np.random.default_rng(4)
    a, b, A, B = receiver(31)
    r, R, pk = notes(rng, 40, A, B)
    pk[::3] = jo.points_mont([jo.IDENTITY])[0]               # every third note is not ours
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), "device"), mont(B), mont(G), to_mem(R, "device"),
                                      to_mem(pk, "device"), async_=async_)
    if async_:
        engine.sync()
    want = np.ones(40, dtype=np.uint8)
    want[::3] = 0
    assert np.array_equal(host(owned), want) and engine.last_stealth_owned() == int(want.sum())
    assert engine.last_stealth_invalid() == 0


# 4 ---- tampered notes are not owned -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_tampered_notes_not_owned(engine, mem):
    rng = np.random.default_rng(5)
    a, b, A, B = receiver(41)
    r, R, pk = notes(rng, 4, A, B)
    Rp, pkp = jo.points_from_mont(R), jo.points_from_mont(pk)
    P = jo.P
    cases = [(Rp[0], pkp[0], 1),
             (Rp[0], ((-pkp[0][0]) % P, pkp[0][1]), 0),             # u negated
             (Rp[0], (pkp[0][0], (pkp[0][1] + 1) % P), 0),          # v + 1
             (Rp[0], (pkp[0][1], pkp[0][0]), 0),                    # coordinates swapped
             (Rp[0], jo.IDENTITY, 0),                               # the identity
             (jo.neg(Rp[1]), pkp[1], 0),                            # -R
             (Rp[2], pkp[3], 0)]                                    # another note's R
    Rs = jo.points_mont([c[0] for c in cases])
    pks = jo.points_mont([c[1] for c in cases])
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(B), mont(G), to_mem(Rs, mem), to_mem(pks, mem))
    assert list(host(owned)) == [c[2] for c in cases] and engine.last_stealth_invalid() == 0
    # a small-order spend key B' = B + T, order 2: the sender's notes to (A, B') are not (a, B)'s, and conversely
    o2 = (0, P - 1)
    Bt = jo.add(B, o2)
    R2, pk2, ok2 = engine.stealth_address_batch(to_mem(jubjub_limbs(r), mem), mont(G), to_mem(jo.points_mont([A]), mem),
                                                to_mem(jo.points_mont([Bt]), mem))
    assert host(ok2).all()
    assert not host(engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(B), mont(G), R2, pk2)).any()
    assert host(engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(Bt), mont(G), R2, pk2)).all()
    # B = -[h] G makes note_pk the identity (0, 1), which its receiver owns
    h = so.hash_point(mul(r[0], A))
    Bneg = jo.neg(mul(h, G))
    R3, pk3, ok3 = engine.stealth_address_batch(to_mem(jubjub_limbs(r[:1]), mem), mont(G), to_mem(jo.points_mont([A]), mem),
                                                to_mem(jo.points_mont([Bneg]), mem))
    assert host(ok3).all() and jo.points_from_mont(host(pk3)) == [jo.IDENTITY]
    assert host(engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(Bneg), mont(G), R3, pk3)).all()


# 5 ---- invalid items, with canary rows ------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_scan_invalid_items(engine, mem):
    rng = np.random.default_rng(6)
    a, b, A, B = receiver(51)
    r, R, pk = notes(rng, 8, A, B)
    Rp, pkp = jo.points_from_mont(R), jo.points_from_mont(pk)
    Rp[1] = jo.off_curve_point(rng)                               # R off the curve
    Rp[2] = (Rp[2][0] + jo.P, Rp[2][1])                           # R coordinate >= p
    pkp[3] = (pkp[3][0], pkp[3][1] + jo.P)                        # note_pk coordinate >= p
    pkp[4] = jo.off_curve_point(rng)                              # canonical, off the curve: not owned, valid
    n = len(Rp)
    want = np.array([1, 0, 0, 0, 0, 1, 1, 1], dtype=np.uint8)
    big = to_mem(np.full(n + 2, 0xA5, dtype=np.uint8), mem)
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(B), mont(G), to_mem(jo.points_mont(Rp), mem),
                                      to_mem(jo.points_mont(pkp), mem), out=big[1:n + 1])
    bigh = host(big)
    assert np.array_equal(host(owned), want) and bigh[0] == 0xA5 and bigh[n + 1] == 0xA5
    assert engine.last_stealth_owned() == 4 and engine.last_stealth_invalid() == 3
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([jo.R_J]), mem), mont(B), mont(G), to_mem(R, mem),
                                      to_mem(pk, mem))
    assert not host(owned).any() and engine.last_stealth_owned() == 0 and engine.last_stealth_invalid() == 8
    with pytest.raises(pb.InvalidPoint):
        pb.owns(jo.R_J, mont(B), mont(G), R[0], pk[0], engine=engine)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_sender_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(7)
    keys = [receiver(s) for s in (61, 62)]
    n = 12
    r = [jo.random_secret(rng) for _ in range(n)]
    As = [keys[i % 2][2] for i in range(n)]
    Bs = [keys[i % 2][3] for i in range(n)]
    r[1] = jo.R_J                                                 # r >= r_J
    As[2] = jo.off_curve_point(rng)                               # A invalid
    Bs[3] = (Bs[3][0] + jo.P, Bs[3][1])                           # B invalid
    r[4], As[4] = jo.R_J + 3, (As[4][0], As[4][1] + jo.P)         # r and A
    As[5], Bs[5] = jo.off_curve_point(rng), jo.off_curve_point(rng)   # A and B
    r[6], As[6], Bs[6] = (1 << 256) - 1, jo.off_curve_point(rng), (0, 0)   # all three
    bad = np.zeros(n, dtype=bool)
    bad[1:7] = True
    wR, wpk, wok = expect(r, As, Bs)
    assert np.array_equal(wok, (~bad).astype(np.uint8))
    bR = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    bP = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs(r), mem), mont(G), to_mem(jo.points_mont(As), mem),
                                             to_mem(jo.points_mont(Bs), mem), R_out=bR[1:n + 1], out=bP[1:n + 1])
    assert np.array_equal(host(ok), wok) and engine.last_stealth_invalid() == 6
    for big, want in ((host(bR), wR), (host(bP), wpk)):
        assert np.array_equal(big[1:n + 1], want) and (big[0] == CANARY).all() and (big[n + 1] == CANARY).all()
    with pytest.raises(pb.InvalidPoint):
        pb.stealth_address(jo.R_J, mont(G), mont(keys[0][2]), mont(keys[0][3]), engine=engine)


# 6 ---- refused calls ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_bad_G_or_receiver_B_refused_with_nothing_written(engine, mem):
    rng = np.random.default_rng(8)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    a, b, A, B = receiver(71)
    n = 5
    r, R, pk = notes(rng, n, A, B)
    rl, al = to_mem(jubjub_limbs(r), mem), to_mem(jubjub_limbs([a]), mem)
    Am, Bm, Rm, pkm = (to_mem(x, mem) for x in (jo.points_mont([A]), jo.points_mont([B]), R, pk))
    gm, bm = mont(G), mont(B)
    bad_points = [mont(jo.off_curve_point(rng)), mont((G[0] + jo.P, G[1])), mont((B[0], B[1] + jo.P))]
    for bp in bad_points:
        oR = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        opk = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)
        c1, c2 = ctypes.c_size_t(CANARY), ctypes.c_size_t(CANARY)
        before = engine.launch_count
        for nn in (n, 0):
            assert lib.p252_stealth_address_batch(ctx, P_(rl), nn, bp.ctypes.data, P_(Am), P_(Bm), 1, P_(oR), P_(opk),
                                                  P_(ok), ctypes.byref(c1), flags) == 6
            assert lib.p252_stealth_owns_batch(ctx, P_(al), bm.ctypes.data, bp.ctypes.data, P_(Rm), P_(pkm), nn, P_(ok),
                                               ctypes.byref(c1), ctypes.byref(c2), flags) == 6
            assert lib.p252_stealth_owns_batch(ctx, P_(al), bp.ctypes.data, gm.ctypes.data, P_(Rm), P_(pkm), nn, P_(ok),
                                               ctypes.byref(c1), ctypes.byref(c2), flags) == 6
        assert engine.launch_count == before and c1.value == CANARY and c2.value == CANARY
        assert (host(oR) == CANARY).all() and (host(opk) == CANARY).all() and (host(ok) == 0xA5).all()
        with pytest.raises(pb.InvalidPoint):
            engine.stealth_owns_batch(al, bp, gm, Rm, pkm)
    # argument refusals
    ok = to_mem(np.zeros(n, dtype=np.uint8), mem)
    assert lib.p252_stealth_address_batch(ctx, P_(rl), n, None, P_(Am), P_(Bm), 1, P_(Rm), P_(pkm), P_(ok), None, flags) == -1
    assert lib.p252_stealth_address_batch(ctx, P_(rl), n, gm.ctypes.data, P_(Am), None, 1, P_(Rm), P_(pkm), P_(ok), None,
                                          flags) == -1
    assert lib.p252_stealth_address_batch(ctx, P_(rl), n, gm.ctypes.data, P_(Am), P_(Bm), 2, P_(Rm), P_(pkm), P_(ok), None,
                                          flags) == -1
    assert lib.p252_stealth_owns_batch(ctx, P_(al), bm.ctypes.data, gm.ctypes.data, P_(Rm), None, n, P_(ok), None, None,
                                       flags) == -1
    assert lib.p252_stealth_owns_batch(ctx, P_(al), None, gm.ctypes.data, P_(Rm), P_(pkm), n, P_(ok), None, None, flags) == -1
    if mem == "device":
        assert lib.p252_stealth_owns_batch(ctx, P_(al), bm.ctypes.data, gm.ctypes.data, P_(Rm) + 8, P_(pkm), 1, P_(ok), None,
                                           None, flags) == -1
        assert lib.p252_stealth_address_batch(ctx, P_(rl), 1, gm.ctypes.data, P_(Am), P_(Bm), 1, P_(Rm), P_(pkm) + 8, P_(ok),
                                              None, flags) == -1


# 7 ---- batch sizes ----------------------------------------------------------------------------------------------------
def _sizes():
    import torch
    coop = 24 * torch.cuda.get_device_properties(0).multi_processor_count
    return [1, 31, 33, 127, 129, coop - 1, coop, coop + 1, 1 << 18]


def test_batch_sizes(engine):
    rng = np.random.default_rng(9)
    a, b, A, B = receiver(81)
    base_r = [jo.random_secret(rng) for _ in range(8)]
    bR, bpk, _ = expect(base_r, [A] * 8, [B] * 8)
    gm, Am, Bm = mont(G), to_mem(jo.points_mont([A]), "device"), to_mem(jo.points_mont([B]), "device")
    for n in _sizes():
        idx = rng.integers(0, 8, n)
        rl = jubjub_limbs(base_r)[idx]
        R, pk, ok = engine.stealth_address_batch(to_mem(rl, "device"), gm, Am, Bm)
        Rh, pkh = host(R), host(pk)
        rows = rng.choice(n, min(n, 24), replace=False)
        assert host(ok).all() and np.array_equal(Rh[rows], bR[idx[rows]]) and np.array_equal(pkh[rows], bpk[idx[rows]])
        flip = rng.random(n) < 0.25                              # a quarter of the notes tampered: not owned
        pkh[flip, 1, 0] ^= np.uint64(1)
        owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), "device"), mont(B), gm, R, to_mem(pkh, "device"))
        o = host(owned)
        assert engine.last_stealth_invalid() == 0
        assert np.array_equal(o[~flip], np.ones(int((~flip).sum()), np.uint8)) and not o[flip].any()
        assert engine.last_stealth_owned() == int((~flip).sum())


# 8 ---- staging hygiene, injected failures, launches per chunk ---------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_calls(engine, mem):
    rng = np.random.default_rng(10)
    a, b, A, B = receiver(91)
    r, R, pk = notes(rng, 50, A, B)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    engine.stealth_address_batch(to_mem(jubjub_limbs(r), mem), mont(G), to_mem(jo.points_mont([A]), mem),
                                 to_mem(jo.points_mont([B]), mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(B), mont(G), to_mem(R, mem), to_mem(pk, mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(11)
    n = 200000                                                    # several staged chunks
    a, b, A, B = receiver(101)
    base_r = [jo.random_secret(rng) for _ in range(16)]
    bR, bpk, _ = expect(base_r, [A] * 16, [B] * 16)
    idx = rng.integers(0, 16, n)
    rl = jubjub_limbs(base_r)[idx]
    gm, Am, Bm = mont(G), jo.points_mont([A]), jo.points_mont([B])
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    for fail_at in (1, 2):
        assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
        with pytest.raises(pb.EngineError):
            engine.stealth_address_batch(rl, gm, Am, Bm)
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.fixed_base_batch(rl[:1], gm)                           # the table of G is built
    before = engine.launch_count
    R, pk, ok = engine.stealth_address_batch(rl, gm, Am, Bm)      # the retry is correct
    sender_launches = engine.launch_count - before
    assert ok.all() and np.array_equal(R, bR[idx]) and np.array_equal(pk, bpk[idx])
    al = jubjub_limbs([a])
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.stealth_owns_batch(al, mont(B), gm, R, pk)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    before = engine.launch_count
    owned = engine.stealth_owns_batch(al, mont(B), gm, R, pk)
    scan_launches = engine.launch_count - before
    assert owned.all() and engine.last_stealth_owned() == n and engine.last_stealth_invalid() == 0
    # no table rebuild for the repeated G: 4 launches per chunk for the sender, 3 for the scan, over several chunks
    assert sender_launches % 4 == 0 and scan_launches % 3 == 0 and sender_launches > 4 and scan_launches > 3
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


# 9 ---- the C and C++ consumers on the GPU ------------------------------------------------------------------------------
def test_c_stealth_smoke_gpu():
    from test_stealth_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "STEALTH_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_stealth_mirror_gpu():
    from test_stealth_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "stealth mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
