"""JubJub key exchange on the device (p252_dhke_batch) and the encrypt / decrypt batches that derive their shared secret
with it (p252_encrypt_batch_dhke / p252_decrypt_batch_dhke), against the pure-Python model in jubjub_oracle.py (affine
complete addition, double-and-add: different formulas from the kernel's) and the C oracle of the sponge."""
import ctypes

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs, random_scalars

pytestmark = pytest.mark.gpu

SECRET_EDGES = [0, 1, 2, 15, 16, jo.R_J - 1, 1 << 251]


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


def point_set(rng):
    """every order class: the small-order points, the generator, random subgroup and random full-group points"""
    return (jo.small_order_points(rng) + [jo.GENERATOR] + [jo.random_subgroup_point(rng) for _ in range(3)] +
            [jo.random_point(rng) for _ in range(3)])


def expect(secrets, points):
    """oracle rows (n, 2, 4) and ok (n,) for paired secrets / points"""
    want = [jo.dhke(s, p) for s, p in zip(secrets, points)]
    ok = np.array([w is not None for w in want], dtype=np.uint8)
    rows = jo.points_mont([w if w is not None else (0, 0) for w in want])
    rows[ok == 0] = 0
    return rows, ok


def run(engine, mem, secrets, points, async_=False):
    s, p = jubjub_limbs(secrets), jo.points_mont(points)
    out, ok = engine.dhke_batch(to_mem(s, mem), to_mem(p, mem), async_=async_)
    if async_:
        engine.sync()
    return host(out), host(ok)


# 1 ---- every edge secret against every point class, every memory space ------------------------------------------
@pytest.mark.parametrize("mem,async_", [("host", False), ("device", False), ("device", True)])
def test_parity_edges_times_point_classes(engine, mem, async_):
    rng = np.random.default_rng(1)
    pts = point_set(rng)
    secs = SECRET_EDGES + [jo.random_secret(rng) for _ in range(3)]
    S = [s for s in secs for _ in pts]
    Pt = [p for _ in secs for p in pts]
    want, wok = expect(S, Pt)
    assert wok.all()
    got, ok = run(engine, mem, S, Pt, async_)
    assert np.array_equal(ok, wok) and np.array_equal(got, want)
    assert engine.last_dhke_invalid() == 0


def test_known_small_order_results(engine):
    rng = np.random.default_rng(2)
    o2, o4, o8 = (0, jo.P - 1), (jo.SQRT_M1, 0), jo.order8_point(rng)
    got, ok = run(engine, "host", [2, 4, 8, 3, 5], [o2, o4, o8, o2, o4])
    assert ok.all()
    assert jo.points_from_mont(got) == [jo.IDENTITY, jo.IDENTITY, jo.IDENTITY, o2, o4]
    # a torsion component passes through: [s](G + T8) = [s]G + [s]T8
    s = jo.random_secret(rng)
    got, ok = run(engine, "host", [s], [jo.add(jo.GENERATOR, o8)])
    assert ok[0] == 1 and jo.points_from_mont(got)[0] == jo.add(jo.mul(s, jo.GENERATOR), jo.mul(s, o8))


# 2 ---- shapes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 129, 1000])
@pytest.mark.parametrize("shape", ["1n", "n1", "nn"])
def test_shapes(engine, n, shape):
    rng = np.random.default_rng(n)
    base = point_set(rng)
    secs = [jo.random_secret(rng) for _ in range(n if shape != "1n" else 1)]
    pts = [base[i % len(base)] for i in range(n if shape != "n1" else 1)]
    for mem in ("host", "device"):
        out, ok = engine.dhke_batch(to_mem(jubjub_limbs(secs), mem), to_mem(jo.points_mont(pts), mem))
        out, ok = host(out), host(ok)
        assert out.shape == (n, 2, 4) and ok.all()
        rows = sorted(set(rng.choice(n, min(n, 24), replace=False).tolist()) | {0, n - 1})
        want, _ = expect([secs[0 if len(secs) == 1 else i] for i in rows], [pts[0 if len(pts) == 1 else i] for i in rows])
        assert np.array_equal(out[rows], want)


def test_large_batch_sampled(engine):
    import torch
    rng = np.random.default_rng(3)
    n = 1 << 18
    base = point_set(rng) + [jo.random_point(rng) for _ in range(20)]
    pts = jo.points_mont(base)[rng.integers(0, len(base), n)]
    secs = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    secs[:, 3] %= np.uint64(jo.R_J >> 192)                    # < r_J
    out, ok = engine.dhke_batch(to_mem(secs, "device"), to_mem(pts, "device"))
    torch.cuda.synchronize()
    out, ok = host(out), host(ok)
    assert ok.all() and engine.last_dhke_invalid() == 0
    rows = rng.choice(n, 48, replace=False)
    want, _ = expect([sum(int(secs[i, k]) << (64 * k) for k in range(4)) for i in rows],
                     jo.points_from_mont(pts[rows]))
    assert np.array_equal(out[rows], want)
    # the view-key scan shape on the same points
    out1, ok1 = engine.dhke_batch(to_mem(secs[:1], "device"), to_mem(pts, "device"))
    out1 = host(out1)
    want1, _ = expect([sum(int(secs[0, k]) << (64 * k) for k in range(4))] * len(rows), jo.points_from_mont(pts[rows]))
    assert np.array_equal(out1[rows], want1) and host(ok1).all()


# 3 ---- invalid items ------------------------------------------------------------------------------------------------
def invalid_batch(rng):
    """(secrets, points, valid): valid and invalid items interleaved"""
    g = jo.GENERATOR
    u_big = (g[0] + jo.P, g[1])                                 # u >= p (same residue as a curve point)
    v_big = (g[0], g[1] + jo.P)
    cases = [(jo.random_secret(rng), jo.off_curve_point(rng), False), (5, u_big, False), (5, v_big, False),
             (jo.R_J, g, False), ((1 << 256) - 1, g, False), (jo.R_J + 3, jo.IDENTITY, False)]
    secs, pts, valid = [], [], []
    for s, p, v in cases:
        secs += [jo.random_secret(rng), s]
        pts += [jo.random_subgroup_point(rng), p]
        valid += [True, v]
    secs.append(7)
    pts.append(g)
    valid.append(True)
    return secs, pts, np.array(valid, dtype=np.uint8)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_items_and_canaries(engine, mem):
    rng = np.random.default_rng(4)
    secs, pts, valid = invalid_batch(rng)
    n = len(secs)
    want, wok = expect(secs, pts)
    assert np.array_equal(wok, valid)
    canary = np.full((n + 2, 2, 4), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    big = to_mem(canary, mem)
    out, ok = engine.dhke_batch(to_mem(jubjub_limbs(secs), mem), to_mem(jo.points_mont(pts), mem), out=big[1:n + 1])
    big = host(big)
    assert np.array_equal(host(ok), valid) and np.array_equal(big[1:n + 1], want)
    assert (big[0] == 0xA5A5A5A5A5A5A5A5).all() and (big[n + 1] == 0xA5A5A5A5A5A5A5A5).all()
    assert engine.last_dhke_invalid() == int((valid == 0).sum())
    with pytest.raises(pb.InvalidPoint):
        pb.dhke(jo.R_J, jo.points_mont([jo.GENERATOR])[0], engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.dhke(3, jo.points_mont([jo.off_curve_point(rng)])[0], engine=engine)
    assert jo.points_from_mont([pb.dhke(3, jo.points_mont([jo.GENERATOR])[0], engine=engine)])[0] == jo.mul(3, jo.GENERATOR)


# 4 ---- batch checks -------------------------------------------------------------------------------------------------
def test_batch_check_refusals(engine):
    import torch
    lib, ctx = _native.lib(), engine._ctx
    s = np.zeros((3, 4), dtype=np.uint64)
    p = jo.points_mont([jo.GENERATOR] * 3)
    out = np.zeros((3, 2, 4), dtype=np.uint64)
    ok = np.zeros(3, dtype=np.uint8)
    msg = np.zeros((3, 2, 4), dtype=np.uint64)
    cip = np.zeros((3, 3, 4), dtype=np.uint64)
    non = np.zeros((3, 4), dtype=np.uint64)
    P_ = lambda a: a.ctypes.data                              # noqa: E731
    nz = ctypes.c_size_t(9)
    assert lib.p252_dhke_batch(ctx, P_(s), 2, P_(p), 3, 3, P_(out), P_(ok), None, 0) == -1
    assert lib.p252_dhke_batch(ctx, P_(s), 3, P_(p), 2, 3, P_(out), P_(ok), None, 0) == -1
    assert lib.p252_dhke_batch(ctx, None, 1, P_(p), 3, 3, P_(out), P_(ok), None, 0) == -1
    assert lib.p252_dhke_batch(ctx, P_(s), 1, P_(p), 1, 3, None, P_(ok), None, 0) == -1
    assert lib.p252_dhke_batch(ctx, P_(s), 1, P_(p), 1, 3, P_(out), None, None, 0) == -1
    assert lib.p252_dhke_batch(ctx, None, 0, None, 0, 0, None, None, ctypes.byref(nz), 0) == 0 and nz.value == 0
    for fn, a, b in ((lib.p252_encrypt_batch_dhke, msg, cip), (lib.p252_decrypt_batch_dhke, cip, msg)):
        assert fn(ctx, P_(a), 3, 2, P_(s), 2, P_(p), 1, P_(non), P_(b), P_(ok), None, 0) == -1
        assert fn(ctx, P_(a), 3, 2, P_(s), 1, P_(p), 1, None, P_(b), P_(ok), None, 0) == -1
        assert fn(ctx, P_(a), 3, 2, P_(s), 1, P_(p), 1, P_(non), P_(b), None, None, 0) == -1
        assert fn(ctx, P_(a), 3, 0, P_(s), 1, P_(p), 1, P_(non), P_(b), P_(ok), None, 0) == 2     # L == 0
    # DEVICE buffers must be 16-byte aligned (ok is a byte array and may sit anywhere)
    ds, dp, do = (torch.zeros(64, dtype=torch.int64, device="cuda") for _ in range(3))
    dok = torch.zeros(16, dtype=torch.uint8, device="cuda")
    assert lib.p252_dhke_batch(ctx, ds.data_ptr() + 8, 1, dp.data_ptr(), 1, 1, do.data_ptr(), dok.data_ptr(), None, 1) == -1
    assert lib.p252_dhke_batch(ctx, ds.data_ptr(), 1, dp.data_ptr() + 8, 1, 1, do.data_ptr(), dok.data_ptr(), None, 1) == -1
    assert lib.p252_dhke_batch(ctx, ds.data_ptr(), 1, dp.data_ptr(), 1, 1, do.data_ptr() + 8, dok.data_ptr(), None, 1) == -1
    assert lib.p252_dhke_batch(ctx, ds.data_ptr(), 1, dp.data_ptr(), 1, 1, do.data_ptr(), dok.data_ptr() + 1, None, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.dhke_batch(s[:2], p)                           # 2 secrets for 3 points


# 5 ---- fused calls ----------------------------------------------------------------------------------------------------
def scan_batch(rng, n, L, view=None):
    """a wallet scan: notes encrypted to view key `view` (or per-note keys) with ephemeral keys R_i = [r_i] G"""
    a = view if view is not None else jo.random_secret(rng)
    pk = jo.mul(a, jo.GENERATOR)
    r = [jo.random_secret(rng) for _ in range(n)]
    R = [jo.mul(ri, jo.GENERATOR) for ri in r]
    msgs = random_scalars(rng, (n, L))
    nonce = random_scalars(rng, n)
    uv = jo.points_mont([jo.mul(ri, pk) for ri in r])       # sender's shared secrets
    return a, pk, r, R, msgs, nonce, uv


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("L", [1, 2, 5])
def test_fused_equals_separate_calls(engine, coracle, mem, L):
    rng = np.random.default_rng(10 + L)
    n = 37
    a, pk, r, R, msgs, nonce, uv = scan_batch(rng, n, L)
    tag = np.zeros(4, dtype=np.uint64)
    _native.lib().p252_encryption_tag(L, tag.ctypes.data)
    # sender: encrypt with dhke(r_i, pk) fused == encrypt_batch with oracle-derived secrets == C oracle
    cip, ok = engine.encrypt_batch_dhke(to_mem(msgs, mem), to_mem(jubjub_limbs(r), mem), to_mem(jo.points_mont([pk]), mem),
                                        to_mem(nonce, mem))
    cip, ok = host(cip), host(ok)
    assert ok.all() and engine.last_dhke_invalid() == 0
    want = coracle.encrypt(tag, msgs, L, uv, nonce)
    assert np.array_equal(cip, want)
    assert np.array_equal(cip, engine.encrypt_batch(msgs, uv, nonce))
    # receiver: one view key against every R_i; fused == dhke_batch + decrypt_batch
    sk = to_mem(jubjub_limbs([a]), mem)
    msg, ok = engine.decrypt_batch_dhke(to_mem(cip, mem), sk, to_mem(jo.points_mont(R), mem), to_mem(nonce, mem))
    assert host(ok).all() and engine.last_decrypt_failures() == 0 and np.array_equal(host(msg), msgs)
    shared, sok = engine.dhke_batch(sk, to_mem(jo.points_mont(R), mem))
    assert np.array_equal(host(shared), uv) and host(sok).all()
    m2, ok2 = engine.decrypt_batch(to_mem(cip, mem), shared, to_mem(nonce, mem))
    assert np.array_equal(host(m2), host(msg)) and np.array_equal(host(ok2), host(ok))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_round_trip_wrong_key_tamper_and_invalid(engine, mem):
    rng = np.random.default_rng(20)
    n, L = 12, 3
    a, pk, r, R, msgs, nonce, uv = scan_batch(rng, n, L)
    cip, ok = engine.encrypt_batch_dhke(to_mem(msgs, mem), to_mem(jubjub_limbs(r), mem), to_mem(jo.points_mont([pk]), mem),
                                        to_mem(nonce, mem))
    cip = host(cip).copy()
    cip[4, 1, 2] ^= np.uint64(1)                              # tampered cipher
    pts = list(R)
    pts[7] = jo.off_curve_point(rng)                          # invalid item: counted once, zeroed
    msg, ok = engine.decrypt_batch_dhke(to_mem(cip, mem), to_mem(jubjub_limbs([a]), mem), to_mem(jo.points_mont(pts), mem),
                                        to_mem(nonce, mem))
    msg, ok = host(msg), host(ok)
    bad = np.zeros(n, dtype=bool)
    bad[[4, 7]] = True
    assert np.array_equal(ok, (~bad).astype(np.uint8)) and engine.last_decrypt_failures() == 2
    assert np.array_equal(msg[~bad], msgs[~bad]) and not msg[bad].any()
    # a wrong view key fails every item
    msg, ok = engine.decrypt_batch_dhke(to_mem(cip, mem), to_mem(jubjub_limbs([a ^ 1]), mem),
                                        to_mem(jo.points_mont(R), mem), to_mem(nonce, mem))
    assert not host(ok).any() and not host(msg).any() and engine.last_decrypt_failures() == n
    # encrypt: an invalid secret gives ok = 0 and a zeroed cipher row, the rest unchanged
    rr = list(r)
    rr[2] = jo.R_J
    cip2, ok2 = engine.encrypt_batch_dhke(to_mem(msgs, mem), to_mem(jubjub_limbs(rr), mem),
                                          to_mem(jo.points_mont([pk]), mem), to_mem(nonce, mem))
    cip2, ok2 = host(cip2), host(ok2)
    assert ok2[2] == 0 and ok2.sum() == n - 1 and not cip2[2].any() and engine.last_dhke_invalid() == 1
    good = np.arange(n) != 2
    want = engine.encrypt_batch(msgs, uv, nonce)
    assert np.array_equal(cip2[good], want[good])


def test_async_fused_counts_after_sync(engine):
    rng = np.random.default_rng(21)
    n, L = 9, 2
    a, pk, r, R, msgs, nonce, uv = scan_batch(rng, n, L)
    cip = engine.encrypt_batch(msgs, uv, nonce)
    cip[0, 0, 0] ^= np.uint64(1)
    msg, ok = engine.decrypt_batch_dhke(to_mem(cip, "device"), to_mem(jubjub_limbs([a]), "device"),
                                        to_mem(jo.points_mont(R), "device"), to_mem(nonce, "device"), async_=True)
    engine.sync()
    assert engine.last_decrypt_failures() == 1 and host(ok).sum() == n - 1


# 6 ---- staging hygiene -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_fused_calls(engine, mem):
    rng = np.random.default_rng(30)
    a, pk, r, R, msgs, nonce, uv = scan_batch(rng, 50, 2)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    cip, _ = engine.encrypt_batch_dhke(to_mem(msgs, mem), to_mem(jubjub_limbs(r), mem), to_mem(jo.points_mont([pk]), mem),
                                       to_mem(nonce, mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.decrypt_batch_dhke(cip, to_mem(jubjub_limbs([a]), mem), to_mem(jo.points_mont(R), mem), to_mem(nonce, mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.dhke_batch(to_mem(jubjub_limbs(r), mem), to_mem(jo.points_mont([pk]), mem))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_and_retry(engine):
    rng = np.random.default_rng(31)
    n, L = 200000, 2                                          # 65536-item chunks after a ramp-up: several chunks
    a = jo.random_secret(rng)
    pk = jo.mul(a, jo.GENERATOR)
    base_r = [jo.random_secret(rng) for _ in range(16)]
    idx = rng.integers(0, 16, n)
    R = jo.points_mont([jo.mul(x, jo.GENERATOR) for x in base_r])[idx]
    uv = jo.points_mont([jo.mul(x, pk) for x in base_r])[idx]
    msgs = rng.integers(0, 1 << 62, (n, L, 4), dtype=np.uint64)
    nonce = rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64)
    cip = engine.encrypt_batch(msgs, uv, nonce)
    sk = jubjub_limbs([a])
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    assert lib.p252_debug_fail_chunk(ctx, 2) == 0
    with pytest.raises(pb.EngineError):
        engine.decrypt_batch_dhke(cip, sk, R, nonce)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    msg, ok = engine.decrypt_batch_dhke(cip, sk, R, nonce)    # the retry is correct
    assert ok.all() and np.array_equal(msg, msgs) and engine.last_decrypt_failures() == 0
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    # the same for the sender's fused call and the plain dhke batch
    rs = jubjub_limbs(base_r)[idx]
    assert lib.p252_debug_fail_chunk(ctx, 1) == 0
    with pytest.raises(pb.EngineError):
        engine.encrypt_batch_dhke(msgs, rs, jo.points_mont([pk]), nonce)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    c2, ok2 = engine.encrypt_batch_dhke(msgs, rs, jo.points_mont([pk]), nonce)
    assert ok2.all() and np.array_equal(c2, cip)
    shared, sok = engine.dhke_batch(rs, jo.points_mont([pk]))
    assert sok.all() and np.array_equal(shared, uv)
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
