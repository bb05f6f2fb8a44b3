"""Fixed-base JubJub scalar multiplication on the device (p252_fixed_base_batch) and the sender's encrypt batch
(p252_encrypt_batch_ephemeral), against the pure-Python model in jubjub_oracle.py (affine complete addition,
double-and-add: different formulas from the kernel's table walk) and against the variable-base p252_dhke_batch /
p252_encrypt_batch_dhke on the same inputs."""
import ctypes

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs, random_scalars

pytestmark = pytest.mark.gpu

SECRET_EDGES = [0, 1, 7, 8, 9, 15, 16, int("7" * 62, 16), int("8" * 62, 16), int("8" * 63, 16), (1 << 248) - 8,
                jo.R_J - 1, (1 << 251) + 1, (1 << 251) + 0x8888]
CANARY = 0xA5A5A5A5A5A5A5A5


def to_mem(a, mem):
    if mem == "host":
        return a
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(x):
    if isinstance(x, np.ndarray):
        return x
    a = x.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def base_set(rng):
    """a base of every order class: identity, order 2, 4 and 8, the generator, a subgroup and a full-group point"""
    ident, o2, o4, _, o8 = jo.small_order_points(rng)
    return [ident, o2, o4, o8, jo.GENERATOR, jo.random_subgroup_point(rng), jo.random_point(rng)]


def expect(secrets, base):
    want = [jo.dhke(s, base) for s in secrets]
    ok = np.array([w is not None for w in want], dtype=np.uint8)
    rows = jo.points_mont([w if w is not None else (0, 0) for w in want])
    rows[ok == 0] = 0
    return rows, ok


def ok_canary(n, mem):
    if mem == "host":
        return np.full(n, 0xA5, dtype=np.uint8)
    import torch
    return torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")


def mont(pt):
    return jo.points_mont([pt])[0]


def s_int(row):
    return sum(int(row[k]) << (64 * k) for k in range(4))


# 1 ---- edge secrets x every base class, every memory space ---------------------------------------------------------
@pytest.mark.parametrize("mem,async_", [("host", False), ("device", False), ("device", True)])
def test_parity_edges_times_base_classes(engine, mem, async_):
    rng = np.random.default_rng(1)
    secs = SECRET_EDGES + [jo.random_secret(rng) for _ in range(4)]
    for base in base_set(rng):
        want, wok = expect(secs, base)
        out, ok = engine.fixed_base_batch(to_mem(jubjub_limbs(secs), mem), mont(base), async_=async_)
        if async_:
            engine.sync()
        assert np.array_equal(host(ok), wok) and np.array_equal(host(out), want), base
        assert engine.last_dhke_invalid() == 0
    assert jo.points_from_mont([pb.fixed_base(5, mont(jo.GENERATOR), engine=engine)])[0] == jo.mul(5, jo.GENERATOR)


# 2 ---- a large batch against the oracle and the variable-base kernel ------------------------------------------------
def test_large_batch_equals_dhke_n1(engine):
    import torch
    rng = np.random.default_rng(2)
    n = 1 << 18
    secs = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    secs[:, 3] %= np.uint64(jo.R_J >> 192)                    # < r_J
    g = mont(jo.GENERATOR)
    ds = to_mem(secs, "device")
    out, ok = engine.fixed_base_batch(ds, g)
    ref, rok = engine.dhke_batch(ds, to_mem(g[None], "device"))
    torch.cuda.synchronize()
    assert host(ok).all() and host(rok).all() and torch.equal(out, ref)
    rows = rng.choice(n, 32, replace=False)
    want, _ = expect([s_int(secs[i]) for i in rows], jo.GENERATOR)
    assert np.array_equal(host(out)[rows], want)


# 3 ---- invalid secrets, canaries, bad bases ---------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_secrets_and_canaries(engine, mem):
    rng = np.random.default_rng(3)
    secs = [jo.random_secret(rng), jo.R_J, 3, (1 << 256) - 1, jo.R_J + 5, jo.R_J - 1, 1 << 252]
    n = len(secs)
    base = jo.random_point(rng)
    want, wok = expect(secs, base)
    assert list(wok) == [1, 0, 1, 0, 0, 1, 0]
    big = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    _, ok = engine.fixed_base_batch(to_mem(jubjub_limbs(secs), mem), mont(base), out=big[1:n + 1])
    big = host(big)
    assert np.array_equal(host(ok), wok) and np.array_equal(big[1:n + 1], want)
    assert (big[0] == CANARY).all() and (big[n + 1] == CANARY).all()
    assert engine.last_dhke_invalid() == 4
    with pytest.raises(pb.InvalidPoint):
        pb.fixed_base(jo.R_J, mont(jo.GENERATOR), engine=engine)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_bad_base_refused_with_nothing_written(engine, mem):
    rng = np.random.default_rng(4)
    lib, ctx = _native.lib(), engine._ctx
    g = jo.GENERATOR
    bad_bases = [jo.points_mont([jo.off_curve_point(rng)])[0], jo.points_mont([(g[0] + jo.P, g[1])])[0],
                 jo.points_mont([(g[0], g[1] + jo.P)])[0]]
    n, L = 5, 2
    s = to_mem(jubjub_limbs([jo.random_secret(rng) for _ in range(n)]), mem)
    msg, non = to_mem(random_scalars(rng, (n, L)), mem), to_mem(random_scalars(rng, n), mem)
    pk = to_mem(jo.points_mont([jo.mul(7, g)]), mem)
    P_ = engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    for b in bad_bases:
        out = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        cip = to_mem(np.full((n, L + 1, 4), CANARY, dtype=np.uint64), mem)
        ok = ok_canary(n, mem)
        cnt = ctypes.c_size_t(CANARY)
        before = engine.launch_count
        assert lib.p252_fixed_base_batch(ctx, b.ctypes.data, P_(s), n, P_(out), P_(ok), ctypes.byref(cnt), flags) == 6
        assert lib.p252_fixed_base_batch(ctx, b.ctypes.data, None, 0, None, None, ctypes.byref(cnt), flags) == 6
        assert lib.p252_encrypt_batch_ephemeral(ctx, P_(msg), n, L, P_(s), b.ctypes.data, P_(pk), 1, P_(non), P_(cip),
                                                P_(out), P_(ok), ctypes.byref(cnt), flags) == 6
        assert engine.launch_count == before and cnt.value == CANARY
        assert (host(out) == CANARY).all() and (host(cip) == CANARY).all() and (host(ok) == 0xA5).all()
        with pytest.raises(pb.InvalidPoint):
            engine.fixed_base_batch(s, b)
    # argument refusals
    gb = mont(g)
    assert lib.p252_fixed_base_batch(ctx, None, P_(s), n, P_(out), P_(ok), None, flags) == -1
    assert lib.p252_fixed_base_batch(ctx, gb.ctypes.data, None, n, P_(out), P_(ok), None, flags) == -1
    assert lib.p252_fixed_base_batch(ctx, gb.ctypes.data, P_(s), n, P_(out), None, None, flags) == -1
    assert lib.p252_encrypt_batch_ephemeral(ctx, P_(msg), n, L, P_(s), gb.ctypes.data, P_(pk), 2, P_(non), P_(cip),
                                            P_(out), P_(ok), None, flags) == -1
    assert lib.p252_encrypt_batch_ephemeral(ctx, P_(msg), n, L, P_(s), gb.ctypes.data, P_(pk), 1, P_(non), P_(cip),
                                            None, P_(ok), None, flags) == -1
    assert lib.p252_encrypt_batch_ephemeral(ctx, P_(msg), n, 0, P_(s), gb.ctypes.data, P_(pk), 1, P_(non), P_(cip),
                                            P_(out), P_(ok), None, flags) == 2
    if mem == "device":
        assert lib.p252_fixed_base_batch(ctx, gb.ctypes.data, P_(s) + 8, 1, P_(out), P_(ok), None, flags) == -1
        assert lib.p252_fixed_base_batch(ctx, gb.ctypes.data, P_(s), 1, P_(out) + 8, P_(ok), None, flags) == -1


# 4 ---- the table cache -----------------------------------------------------------------------------------------------
def test_cache_one_launch_for_a_repeated_base_and_alternating_bases(engine):
    rng = np.random.default_rng(5)
    secs = [jo.random_secret(rng) for _ in range(20)]
    b1, b2 = jo.GENERATOR, jo.random_point(rng)
    s = jubjub_limbs(secs)
    engine.fixed_base_batch(s, mont(b1))
    before = engine.launch_count
    out, _ = engine.fixed_base_batch(s, mont(b1))
    assert engine.launch_count == before + 1                  # the cached table: k_fixed_base only
    assert np.array_equal(out, expect(secs, b1)[0])
    for k in range(4):
        b = (b2, b1)[k % 2]                                   # every call changes the base
        before = engine.launch_count
        out, ok = engine.fixed_base_batch(s, mont(b))
        assert engine.launch_count == before + 2              # a new base: the table build, then k_fixed_base
        assert np.array_equal(out, expect(secs, b)[0]) and ok.all()


def test_async_calls_with_different_bases_back_to_back(engine):
    rng = np.random.default_rng(6)
    secs = [jo.random_secret(rng) for _ in range(300)]
    bases = [jo.random_point(rng), jo.GENERATOR, jo.random_subgroup_point(rng)]
    s = to_mem(jubjub_limbs(secs), "device")
    outs = [engine.fixed_base_batch(s, mont(b), async_=True) for b in bases]
    engine.sync()
    rows = rng.choice(len(secs), 12, replace=False)
    for (out, ok), b in zip(outs, bases):
        want, _ = expect([secs[i] for i in rows], b)
        assert host(ok).all() and np.array_equal(host(out)[rows], want)


# 5 ---- the sender's fused call -----------------------------------------------------------------------------------------
def sender_batch(rng, n, L, per_note_keys):
    a = [jo.random_secret(rng) for _ in range(n if per_note_keys else 1)]
    pk = [jo.mul(x, jo.GENERATOR) for x in a]
    r = [jo.random_secret(rng) for _ in range(n)]
    return a, pk, r, random_scalars(rng, (n, L)), random_scalars(rng, n)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("per_note_keys", [False, True])
def test_fused_equals_separate_calls_and_round_trips(engine, coracle, mem, per_note_keys):
    rng = np.random.default_rng(10 + per_note_keys)
    n, L = 45, 2
    a, pk, r, msgs, nonce = sender_batch(rng, n, L, per_note_keys)
    g, rl, pkm = mont(jo.GENERATOR), jubjub_limbs(r), jo.points_mont(pk)
    cip, R, ok = engine.encrypt_batch_ephemeral(to_mem(msgs, mem), to_mem(rl, mem), g, to_mem(pkm, mem), to_mem(nonce, mem))
    cip, R, ok = host(cip), host(R), host(ok)
    assert ok.all() and engine.last_dhke_invalid() == 0
    R1, _ = engine.fixed_base_batch(rl, g)
    assert np.array_equal(R, R1)
    assert np.array_equal(R, jo.points_mont([jo.mul(x, jo.GENERATOR) for x in r]))
    c2, ok2 = engine.encrypt_batch_dhke(msgs, rl, pkm, nonce)
    assert np.array_equal(cip, c2) and ok2.all()
    tag = np.zeros(4, dtype=np.uint64)
    _native.lib().p252_encryption_tag(L, tag.ctypes.data)
    uv = jo.points_mont([jo.mul(x, pk[0 if len(pk) == 1 else i]) for i, x in enumerate(r)])
    assert np.array_equal(cip, coracle.encrypt(tag, msgs, L, uv, nonce))
    # the receiver: decrypt_batch_dhke(a, R) restores every message (the reference example's round trip)
    msg, okd = engine.decrypt_batch_dhke(to_mem(cip, mem), to_mem(jubjub_limbs(a), mem), to_mem(R, mem), to_mem(nonce, mem))
    assert host(okd).all() and np.array_equal(host(msg), msgs)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_fused_invalid_items_zeroed_and_counted(engine, mem):
    rng = np.random.default_rng(20)
    n, L = 14, 3
    a, pk, r, msgs, nonce = sender_batch(rng, n, L, True)
    pts = list(pk)
    pts[3] = jo.off_curve_point(rng)                          # public key off the curve
    pts[5] = (jo.GENERATOR[0] + jo.P, jo.GENERATOR[1])        # u >= p
    rr = list(r)
    rr[8] = jo.R_J                                            # r >= r_J
    rr[5] = jo.R_J + 1                                        # both invalid: counted once
    bad = np.zeros(n, dtype=bool)
    bad[[3, 5, 8]] = True
    big_c = to_mem(np.full((n + 2, L + 1, 4), CANARY, dtype=np.uint64), mem)
    big_r = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    cip, R, ok = engine.encrypt_batch_ephemeral(to_mem(msgs, mem), to_mem(jubjub_limbs(rr), mem), mont(jo.GENERATOR),
                                                to_mem(jo.points_mont(pts), mem), to_mem(nonce, mem), out=big_c[1:n + 1],
                                                R_out=big_r[1:n + 1])
    big_c, big_r, ok = host(big_c), host(big_r), host(ok)
    assert np.array_equal(ok, (~bad).astype(np.uint8)) and engine.last_dhke_invalid() == 3
    assert not big_c[1:n + 1][bad].any() and not big_r[1:n + 1][bad].any()
    for arr in (big_c, big_r):
        assert (arr[0] == CANARY).all() and (arr[n + 1] == CANARY).all()
    good = ~bad
    want_r = jo.points_mont([jo.mul(x, jo.GENERATOR) for x in r])
    assert np.array_equal(big_r[1:n + 1][good], want_r[good])
    c2, _ = engine.encrypt_batch_dhke(msgs, jubjub_limbs(r), jo.points_mont(pk), nonce)
    assert np.array_equal(big_c[1:n + 1][good], c2[good])


def test_async_fused_count_after_sync(engine):
    rng = np.random.default_rng(21)
    n, L = 9, 2
    a, pk, r, msgs, nonce = sender_batch(rng, n, L, False)
    rr = list(r)
    rr[4] = jo.R_J
    cip, R, ok = engine.encrypt_batch_ephemeral(to_mem(msgs, "device"), to_mem(jubjub_limbs(rr), "device"),
                                                mont(jo.GENERATOR), to_mem(jo.points_mont(pk), "device"),
                                                to_mem(nonce, "device"), async_=True)
    engine.sync()
    assert engine.last_dhke_invalid() == 1 and host(ok).sum() == n - 1


# 6 ---- staging hygiene -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_calls(engine, mem):
    rng = np.random.default_rng(30)
    a, pk, r, msgs, nonce = sender_batch(rng, 50, 2, False)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    g = mont(jo.GENERATOR)
    engine.encrypt_batch_ephemeral(to_mem(msgs, mem), to_mem(jubjub_limbs(r), mem), g, to_mem(jo.points_mont(pk), mem),
                                   to_mem(nonce, mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.fixed_base_batch(to_mem(jubjub_limbs(r), mem), g)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_and_retry(engine):
    rng = np.random.default_rng(31)
    n, L = 200000, 2                                          # several staged chunks
    a = jo.random_secret(rng)
    pk = jo.points_mont([jo.mul(a, jo.GENERATOR)])
    base_r = [jo.random_secret(rng) for _ in range(16)]
    idx = rng.integers(0, 16, n)
    rs = jubjub_limbs(base_r)[idx]
    R_want = jo.points_mont([jo.mul(x, jo.GENERATOR) for x in base_r])[idx]
    msgs = rng.integers(0, 1 << 62, (n, L, 4), dtype=np.uint64)
    nonce = rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64)
    g = mont(jo.GENERATOR)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    for fail_at in (1, 2):
        assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
        with pytest.raises(pb.EngineError):
            engine.encrypt_batch_ephemeral(msgs, rs, g, pk, nonce)
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    cip, R, ok = engine.encrypt_batch_ephemeral(msgs, rs, g, pk, nonce)      # the retry is correct
    assert ok.all() and np.array_equal(R, R_want)
    c2, _ = engine.encrypt_batch_dhke(msgs, rs, pk, nonce)
    assert np.array_equal(cip, c2)
    msg, okd = engine.decrypt_batch_dhke(cip, jubjub_limbs([a]), R, nonce)
    assert okd.all() and np.array_equal(msg, msgs)
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.fixed_base_batch(rs, g)
    out, ok = engine.fixed_base_batch(rs, g)
    assert ok.all() and np.array_equal(out, R_want)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
