"""Schnorr signatures on the device (p252_schnorr_sign_batch / p252_schnorr_verify_batch) against the model of
schnorr_oracle.py (affine complete addition, double-and-add, the Python Hades, big-integer arithmetic modulo r_J), against
the existing calls signing is built from (fixed_base_batch, hash_batch_truncated), and verification against signing."""
import ctypes
import functools

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import poseidon252_b200 as pb
import schnorr_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_gpu_stealth import CANARY, _sizes, classes, host, mont, s_int, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
SK_EDGES = [0, 1, 2, N - 1, 0x0b3f6a5c1d2e3f405162738495a6b7c8d9eafb0c1d2e3f4051627384950a1b2c]
R_EDGES = [0, 1, N - 1, 0x0123456789abcdeffedcba98765432100f1e2d3c4b5a69788796a5b4c3d2e1f0]
M_EDGES = [0, 1, P - 1, 0x2c3e8f1a9b7d6e5f4a3b2c1d0e9f8a7b6c5d4e3f2a1b0c9d8e7f6a5b4c3d2e1f]


def fr_rows(ms):
    """field elements -> (n, 4) BlsScalar.0 limbs; a value >= p is passed through raw, so that the device sees it"""
    out = np.zeros((len(ms), 4), dtype=np.uint64)
    for i, m in enumerate(ms):
        v = m * ho.R % P if m < P else m
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & ((1 << 64) - 1)
    return out


def ints(rows):
    return [s_int(r) for r in host(rows)]


@functools.lru_cache(maxsize=None)
def mul(k, pt):
    return jo.mul(k, pt)


@functools.lru_cache(maxsize=None)
def model_sign(sk, r, m):
    """(u, R, ok) as the device writes them: zeroed rows for an invalid item"""
    if not (0 <= sk < N and 0 <= r < N and 0 <= m < P):
        return 0, (0, 0), 0
    R = mul(r, G)
    return (r - so.challenge(R, m) * sk) % N, R, 1


@functools.lru_cache(maxsize=None)
def model_verify(pk, u, R, m):
    """1 / 0 / None (invalid), with the model's scalar multiplications cached"""
    if not (0 <= u < N and 0 <= m < P and all(0 <= x < P for x in R) and jo.on_curve(pk)):
        return None
    return int(jo.add(mul(u, G), mul(so.challenge(R, m), pk)) == tuple(R))


def expect_sign(sks, rs, ms):
    rows = [model_sign(sk, r, m) for sk, r, m in zip(sks, rs, ms)]
    R = jo.points_mont([x[1] for x in rows])
    ok = np.array([x[2] for x in rows], dtype=np.uint8)
    R[ok == 0] = 0
    return [x[0] for x in rows], R, ok


@functools.lru_cache(maxsize=None)
def signer(seed):
    rng = np.random.default_rng(seed)
    sk = jo.random_secret(rng)
    return sk, mul(sk, G)


def random_r(rng, n):
    r = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    r[:, 3] %= np.uint64(N >> 192)
    return r


def random_m(rng, n):
    m = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    m[:, 3] %= np.uint64(P >> 192)
    return m


# 1 ---- signing against the model: edge sk x r x m ------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", [("host", False), ("device", False), ("device", True)])
@pytest.mark.parametrize("n_secret", ["one", "n"])
def test_sign_against_model(engine, mem, async_, n_secret):
    gm = mont(G)
    grid = [(sk, r, m) for sk in SK_EDGES for r in R_EDGES for m in M_EDGES]
    if n_secret == "n":
        calls = [grid]
    else:
        calls = [[x for x in grid if x[0] == sk] for sk in SK_EDGES]
    for items in calls:
        sks, rs, ms = zip(*items)
        wu, wR, wok = expect_sign(sks, rs, ms)
        k = 1 if n_secret == "one" else len(sks)
        u, R, ok = engine.schnorr_sign_batch(to_mem(jubjub_limbs(sks[:k]), mem), to_mem(jubjub_limbs(rs), mem),
                                             to_mem(fr_rows(ms), mem), gm, async_=async_)
        if async_:
            engine.sync()
        assert np.array_equal(host(ok), wok) and np.array_equal(host(R), wR) and ints(u) == wu
        assert engine.last_schnorr_invalid() == 0
    u1, R1 = pb.schnorr_sign(SK_EDGES[4], R_EDGES[3], fr_rows([M_EDGES[3]])[0], gm, engine=engine)
    w = model_sign(SK_EDGES[4], R_EDGES[3], M_EDGES[3])
    assert s_int(u1) == w[0] and jo.points_from_mont(R1[None]) == [w[1]]
    pk = mont(mul(SK_EDGES[4], G))
    assert pb.schnorr_verify(pk, u1, R1, fr_rows([M_EDGES[3]])[0], gm, engine=engine) is True
    assert pb.schnorr_verify(pk, u1, R1, fr_rows([M_EDGES[2]])[0], gm, engine=engine) is False


# 2 ---- signing against the calls it is built from ---------------------------------------------------------------------
def test_sign_equals_fixed_base_and_truncated_hash(engine):
    import torch
    rng = np.random.default_rng(2)
    n = 1 << 12
    sk, _ = signer(1)
    r, m = random_r(rng, n), random_m(rng, n)
    dr, dm, gm = to_mem(r, "device"), to_mem(m, "device"), mont(G)
    u, R, ok = engine.schnorr_sign_batch(to_mem(jubjub_limbs([sk]), "device"), dr, dm, gm)
    R1, ok1 = engine.fixed_base_batch(dr, gm)
    rows = torch.cat([R.reshape(n, 2, 4), dm.reshape(n, 1, 4)], dim=1).contiguous()
    c = engine.hash_batch_truncated(pb.Domain.Other, rows)
    torch.cuda.synchronize()
    assert host(ok).all() and host(ok1).all() and torch.equal(R, R1)
    for i, (ui, ci) in enumerate(zip(ints(u), ints(c.reshape(n, 4)))):
        assert ui == (s_int(r[i]) - ci * sk) % N
    for i in rng.choice(n, 3, replace=False):
        m_int = s_int(m[i]) * pow(ho.R, -1, P) % P
        assert model_sign(sk, s_int(r[i]), m_int)[0] == ints(u)[i]


# 3 ---- every signature of a large device-signed batch verifies ---------------------------------------------------------
def test_large_batch_round_trip(engine):
    rng = np.random.default_rng(3)
    n = 1 << 18
    keys = [signer(s) for s in (11, 12, 13)]
    pick = rng.integers(0, 3, n)
    sks = jubjub_limbs([k[0] for k in keys])[pick]
    pks = jo.points_mont([k[1] for k in keys])
    r, m, gm = to_mem(random_r(rng, n), "device"), to_mem(random_m(rng, n), "device"), mont(G)
    u, R, ok = engine.schnorr_sign_batch(to_mem(sks, "device"), r, m, gm)
    assert host(ok).all() and engine.last_schnorr_invalid() == 0
    v = engine.schnorr_verify_batch(to_mem(pks[pick], "device"), u, R, m, gm)
    assert host(v).all() and engine.last_schnorr_verified() == n and engine.last_schnorr_invalid() == 0
    # one key for the whole batch, n_secret = n_public = 1; under it only that key's signatures verify
    u1, R1, ok1 = engine.schnorr_sign_batch(to_mem(sks[:1], "device"), r, m, gm)
    v1 = engine.schnorr_verify_batch(to_mem(pks[pick[:1]], "device"), u1, R1, m, gm)
    assert host(ok1).all() and host(v1).all() and engine.last_schnorr_verified() == n
    v2 = engine.schnorr_verify_batch(to_mem(pks[pick[:1]], "device"), u, R, m, gm)
    assert np.array_equal(host(v2), (pick == pick[0]).astype(np.uint8))
    # signatures made by the model verify on the device
    sk, pk = keys[0]
    rs = [jo.random_secret(rng) for _ in range(6)]
    ms = [int(rng.integers(0, 1 << 62)) << 190 | i for i in range(6)]
    mu, mR, _ = expect_sign([sk] * 6, rs, ms)
    v3 = engine.schnorr_verify_batch(jo.points_mont([pk]), jubjub_limbs(mu), mR, fr_rows(ms), gm)
    assert v3.all() and engine.last_schnorr_verified() == 6


# 4 ---- tampered signatures and keys of every order class, each compared with the model ----------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_tampered_against_model(engine, mem):
    rng = np.random.default_rng(4)
    ident, o2, o4, o8, _, _, full = classes()
    sk, pk0 = signer(21)
    _, other = signer(22)
    cases = []
    for T in (ident, o2, o4, o8, full):
        # a key with the torsion component of T's class: [sk] G + (T's torsion part; full: a random full-order key)
        pk = jo.add(pk0, T) if T != full else full
        r = jo.random_secret(rng)
        m = int(rng.integers(0, 1 << 62)) << 190 | 77
        u, R, ok = model_sign(sk, r, m)
        assert ok
        cases += [(pk, u, R, m), (pk, u, R, m + 1), (pk, (u + 1) % N, R, m), (pk, u, jo.neg(R), m),
                  (pk, u, (R[1], R[0]), m), (pk, u, jo.IDENTITY, m), (other, u, R, m), (jo.neg(pk), u, R, m),
                  (jo.add(pk, o2), u, R, m), (jo.add(pk, o4), u, R, m), (jo.add(pk, o8), u, R, m)]
    want = np.array([model_verify(*c) for c in cases], dtype=np.uint8)
    assert want[0] == 1                                             # the untampered signature under [sk] G
    v = engine.schnorr_verify_batch(to_mem(jo.points_mont([c[0] for c in cases]), mem),
                                    to_mem(jubjub_limbs([c[1] for c in cases]), mem),
                                    to_mem(jo.points_mont([c[2] for c in cases]), mem),
                                    to_mem(fr_rows([c[3] for c in cases]), mem), mont(G))
    assert np.array_equal(host(v), want) and engine.last_schnorr_invalid() == 0
    assert engine.last_schnorr_verified() == int(want.sum())


# 5 ---- invalid items, with canary rows and both counts ----------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_sign_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(5)
    n = 10
    sks = [signer(31 + i % 2)[0] for i in range(n)]
    rs = [jo.random_secret(rng) for _ in range(n)]
    ms = [int(rng.integers(0, 1 << 62)) for _ in range(n)]
    sks[1] = N                                                     # sk >= r_J
    rs[2] = N + 5                                                  # r >= r_J
    ms[3] = P                                                      # m >= p
    sks[4], rs[4], ms[4] = (1 << 256) - 1, (1 << 256) - 1, (1 << 256) - 1   # all three
    bad = np.zeros(n, dtype=bool)
    bad[1:5] = True
    wu, wR, wok = expect_sign(sks, rs, ms)
    assert np.array_equal(wok, (~bad).astype(np.uint8))
    bu = to_mem(np.full((n + 2, 4), CANARY, dtype=np.uint64), mem)
    bR = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    u, R, ok = engine.schnorr_sign_batch(to_mem(jubjub_limbs(sks), mem), to_mem(jubjub_limbs(rs), mem),
                                         to_mem(fr_rows(ms), mem), mont(G), u_out=bu[1:n + 1], R_out=bR[1:n + 1])
    assert np.array_equal(host(ok), wok) and engine.last_schnorr_invalid() == 4
    hu, hR = host(bu), host(bR)
    assert ints(hu[1:n + 1]) == wu and np.array_equal(hR[1:n + 1], wR)
    for big in (hu, hR):
        assert (big[0] == CANARY).all() and (big[n + 1] == CANARY).all()
    with pytest.raises(pb.InvalidPoint):
        pb.schnorr_sign(N, 5, fr_rows([1])[0], mont(G), engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.schnorr_sign(5, 5, fr_rows([P])[0], mont(G), engine=engine)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_verify_invalid_items(engine, mem):
    rng = np.random.default_rng(6)
    sk, pk = signer(41)
    n = 9
    rs = [jo.random_secret(rng) for _ in range(n)]
    ms = [int(rng.integers(0, 1 << 62)) for _ in range(n)]
    sig = [model_sign(sk, r, m) for r, m in zip(rs, ms)]
    us, Rs, pks = [s[0] for s in sig], [s[1] for s in sig], [pk] * n
    us[1] = N                                                      # u >= r_J
    Rs[2] = (Rs[2][0] + P, Rs[2][1])                               # an R coordinate >= p
    pks[3] = jo.off_curve_point(rng)                               # PK off the curve
    pks[4] = (pk[0], pk[1] + P)                                    # a PK coordinate >= p
    ms[5] = P + 1                                                  # m >= p
    Rs[6] = jo.off_curve_point(rng)                                # canonical R off the curve: valid, not verified
    want = np.array([1, 0, 0, 0, 0, 0, 0, 1, 1], dtype=np.uint8)
    assert [model_verify(*c) for c in zip(pks, us, Rs, ms)] == [1, None, None, None, None, None, 0, 1, 1]
    big = to_mem(np.full(n + 2, 0xA5, dtype=np.uint8), mem)
    v = engine.schnorr_verify_batch(to_mem(jo.points_mont(pks), mem), to_mem(jubjub_limbs(us), mem),
                                    to_mem(jo.points_mont(Rs), mem), to_mem(fr_rows(ms), mem), mont(G), out=big[1:n + 1])
    bigh = host(big)
    assert np.array_equal(host(v), want) and bigh[0] == 0xA5 and bigh[n + 1] == 0xA5
    assert engine.last_schnorr_verified() == 3 and engine.last_schnorr_invalid() == 5
    # a broadcast PK off the curve makes every item invalid
    v = engine.schnorr_verify_batch(to_mem(jo.points_mont([pks[3]]), mem), to_mem(jubjub_limbs(us), mem),
                                    to_mem(jo.points_mont(Rs), mem), to_mem(fr_rows(ms), mem), mont(G))
    assert not host(v).any() and engine.last_schnorr_verified() == 0 and engine.last_schnorr_invalid() == n
    with pytest.raises(pb.InvalidPoint):
        pb.schnorr_verify(mont(pk), N, mont(Rs[0]), fr_rows([ms[0]])[0], mont(G), engine=engine)


# 6 ---- refused calls ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing_and_launch_nothing(engine, mem):
    rng = np.random.default_rng(7)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    sk, pk = signer(51)
    n = 5
    rs = [jo.random_secret(rng) for _ in range(n)]
    ms = list(range(n))
    wu, wR, _ = expect_sign([sk] * n, rs, ms)
    skl, rl, ml = (to_mem(x, mem) for x in (jubjub_limbs([sk]), jubjub_limbs(rs), fr_rows(ms)))
    ul, Rl, pkl = to_mem(jubjub_limbs(wu), mem), to_mem(wR, mem), to_mem(jo.points_mont([pk]), mem)
    gm = mont(G)
    for bp in [mont(jo.off_curve_point(rng)), mont((G[0] + P, G[1])), mont((G[0], G[1] + P))]:
        ou = to_mem(np.full((n, 4), CANARY, dtype=np.uint64), mem)
        oR = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)
        c1, c2 = ctypes.c_size_t(CANARY), ctypes.c_size_t(CANARY)
        before = engine.launch_count
        for nn in (n, 0):
            assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 1, P_(rl), P_(ml), nn, bp.ctypes.data, P_(ou), P_(oR), P_(ok),
                                               ctypes.byref(c1), flags) == 6
            assert lib.p252_schnorr_verify_batch(ctx, P_(pkl), 1, P_(ul), P_(Rl), P_(ml), nn, bp.ctypes.data, P_(ok),
                                                 ctypes.byref(c1), ctypes.byref(c2), flags) == 6
        assert engine.launch_count == before and c1.value == CANARY and c2.value == CANARY
        assert (host(ou) == CANARY).all() and (host(oR) == CANARY).all() and (host(ok) == 0xA5).all()
        with pytest.raises(pb.InvalidPoint):
            engine.schnorr_verify_batch(pkl, ul, Rl, ml, bp)
    # argument refusals
    ok = to_mem(np.zeros(n, dtype=np.uint8), mem)
    ou, oR = to_mem(np.zeros((n, 4), np.uint64), mem), to_mem(np.zeros((n, 2, 4), np.uint64), mem)
    g = gm.ctypes.data
    before = engine.launch_count
    assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 1, P_(rl), P_(ml), n, None, P_(ou), P_(oR), P_(ok), None, flags) == -1
    assert lib.p252_schnorr_sign_batch(ctx, None, 1, P_(rl), P_(ml), n, g, P_(ou), P_(oR), P_(ok), None, flags) == -1
    assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 1, P_(rl), None, n, g, P_(ou), P_(oR), P_(ok), None, flags) == -1
    assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 1, P_(rl), P_(ml), n, g, P_(ou), P_(oR), None, None, flags) == -1
    assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 2, P_(rl), P_(ml), n, g, P_(ou), P_(oR), P_(ok), None, flags) == -1
    assert lib.p252_schnorr_verify_batch(ctx, P_(pkl), 2, P_(ul), P_(Rl), P_(ml), n, g, P_(ok), None, None, flags) == -1
    assert lib.p252_schnorr_verify_batch(ctx, P_(pkl), 1, P_(ul), None, P_(ml), n, g, P_(ok), None, None, flags) == -1
    assert lib.p252_schnorr_verify_batch(ctx, None, 1, P_(ul), P_(Rl), P_(ml), n, g, P_(ok), None, None, flags) == -1
    if mem == "device":
        assert lib.p252_schnorr_sign_batch(ctx, P_(skl), 1, P_(rl), P_(ml), 1, g, P_(ou) + 8, P_(oR), P_(ok), None,
                                           flags) == -1
        assert lib.p252_schnorr_verify_batch(ctx, P_(pkl), 1, P_(ul), P_(Rl) + 8, P_(ml), 1, g, P_(ok), None, None,
                                             flags) == -1
    assert engine.launch_count == before and (host(ou) == 0).all() and (host(ok) == 0).all()


# 7 ---- batch sizes ----------------------------------------------------------------------------------------------------
def test_batch_sizes(engine):
    rng = np.random.default_rng(8)
    sk, pk = signer(61)
    base_r = [jo.random_secret(rng) for _ in range(8)]
    base_m = [int(rng.integers(0, 1 << 62)) for _ in range(8)]
    bu, bR, _ = expect_sign([sk] * 8, base_r, base_m)
    bu = jubjub_limbs(bu)
    gm, skl, pkl = mont(G), to_mem(jubjub_limbs([sk]), "device"), to_mem(jo.points_mont([pk]), "device")
    for n in _sizes():
        idx = rng.integers(0, 8, n)
        m = to_mem(fr_rows(base_m)[idx], "device")
        u, R, ok = engine.schnorr_sign_batch(skl, to_mem(jubjub_limbs(base_r)[idx], "device"), m, gm)
        uh, Rh = host(u), host(R)
        rows = rng.choice(n, min(n, 24), replace=False)
        assert host(ok).all() and np.array_equal(uh[rows], bu[idx[rows]]) and np.array_equal(Rh[rows], bR[idx[rows]])
        flip = rng.random(n) < 0.25                              # a quarter of the signatures tampered: not verified
        uh[flip, 0] ^= np.uint64(1)
        v = host(engine.schnorr_verify_batch(pkl, to_mem(uh, "device"), R, m, gm))
        assert engine.last_schnorr_invalid() == 0
        assert v[~flip].all() and not v[flip].any() and engine.last_schnorr_verified() == int((~flip).sum())


# 8 ---- staging hygiene, injected failures, launches per chunk ---------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_signing(engine, mem):
    rng = np.random.default_rng(9)
    sk, pk = signer(71)
    rs = [jo.random_secret(rng) for _ in range(50)]
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    u, R, ok = engine.schnorr_sign_batch(to_mem(jubjub_limbs([sk]), mem), to_mem(jubjub_limbs(rs), mem),
                                         to_mem(fr_rows(list(range(50))), mem), mont(G))
    assert host(ok).all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(10)
    n = 200000                                                    # several staged chunks
    sk, pk = signer(81)
    base_r = [jo.random_secret(rng) for _ in range(16)]
    base_m = [int(rng.integers(0, 1 << 62)) for _ in range(16)]
    bu, bR, _ = expect_sign([sk] * 16, base_r, base_m)
    idx = rng.integers(0, 16, n)
    rl, ml = jubjub_limbs(base_r)[idx], fr_rows(base_m)[idx]
    gm, skl, pkl = mont(G), jubjub_limbs([sk]), jo.points_mont([pk])
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    for fail_at in (1, 2):
        assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
        with pytest.raises(pb.EngineError):
            engine.schnorr_sign_batch(skl, rl, ml, gm)
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.fixed_base_batch(rl[:1], gm)                           # the table of G is built
    before = engine.launch_count
    u, R, ok = engine.schnorr_sign_batch(skl, rl, ml, gm)         # the retry is correct
    sign_launches = engine.launch_count - before
    assert ok.all() and ints(u) == [bu[i] for i in idx] and np.array_equal(R, bR[idx])
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    # verification stages public data only (signatures, keys, messages, challenges): no wipe is asked of it
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.schnorr_verify_batch(pkl, u, R, ml, gm)
    before = engine.launch_count
    v = engine.schnorr_verify_batch(pkl, u, R, ml, gm)
    verify_launches = engine.launch_count - before
    assert v.all() and engine.last_schnorr_verified() == n and engine.last_schnorr_invalid() == 0
    # no table rebuild for the repeated G: 4 launches per chunk for signing, 3 for verification, over several chunks
    assert sign_launches % 4 == 0 and verify_launches % 3 == 0 and sign_launches > 4 and verify_launches > 3


# 9 ---- the C and C++ consumers on the GPU ------------------------------------------------------------------------------
def test_c_schnorr_smoke_gpu():
    from test_schnorr_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "SCHNORR_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_schnorr_mirror_gpu():
    from test_schnorr_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "schnorr mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
