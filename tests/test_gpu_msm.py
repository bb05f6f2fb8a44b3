"""Multi-scalar multiplication and all-or-nothing Schnorr verification on the device (p252_jubjub_msm /
p252_schnorr_verify_all) against the models of msm_oracle.py, and at device scale against an identity that does not use
the bucket code: for P_i = [k_i] G from fixed_base_batch, sum [s_i] P_i = [sum s_i k_i mod r_J] G."""
import ctypes

import numpy as np
import pytest

import jubjub_oracle as jo
import msm_oracle as mo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
import schnorr_oracle as so
from test_gpu_schnorr import fr_rows, random_m, random_r, signer
from test_gpu_stealth import host, mont, s_int, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
CHUNK = 1 << 17          # the staged chunk of an MSM batch (96 bytes per item)
SPACES = [("host", False), ("device", False), ("device", True)]


def run_msm(engine, sc, pts, mem, async_=False):
    out = engine.jubjub_msm(to_mem(sc, mem), to_mem(pts, mem), async_=async_)
    if async_:
        engine.sync()
    return jo.points_from_mont(host(out).reshape(1, 2, 4))[0]


def limbs_raw(vals):
    """ints < 2^256 -> (n, 4) rows, also for values >= r_J (jubjub_limbs may refuse those)"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & ((1 << 64) - 1)
    return out


# 1 ---- parity with the model on random, edge and small-order points ---------------------------------------------------
@pytest.mark.parametrize("mem,async_", SPACES)
@pytest.mark.parametrize("n", [1, 2, 3, 127, 128, 129])
def test_random_points_against_model(engine, mem, async_, n):
    rng = np.random.default_rng(n)
    pts = [jo.random_point(rng) for _ in range(n)]
    sc = [jo.random_secret(rng) for _ in range(n)]
    assert run_msm(engine, limbs_raw(sc), jo.points_mont(pts), mem, async_) == mo.msm(sc, pts)
    assert engine.last_msm_invalid() == 0


@pytest.mark.parametrize("mem,async_", SPACES)
def test_edge_and_small_order_points(engine, mem, async_):
    rng = np.random.default_rng(7)
    pts = list(mo.edge_points()) + jo.small_order_points(rng) + [jo.IDENTITY, G, jo.neg(G)]
    sc = mo.edge_scalars()
    sc = (sc * (len(pts) // len(sc) + 1))[:len(pts)]
    assert run_msm(engine, limbs_raw(sc), jo.points_mont(pts), mem, async_) == mo.msm(sc, pts)
    # P and -P under the same scalar cancel
    p = jo.random_point(rng)
    s = jo.random_secret(rng)
    assert run_msm(engine, limbs_raw([s, s]), jo.points_mont([p, jo.neg(p)]), mem, async_) == jo.IDENTITY
    assert run_msm(engine, np.zeros((0, 4), np.uint64), np.zeros((0, 2, 4), np.uint64), mem, async_) == jo.IDENTITY


def test_thousand_points_against_model(engine):
    rng = np.random.default_rng(1000)
    pts = [jo.random_point(rng) for _ in range(1000)]
    sc = [jo.random_secret(rng) for _ in range(1000)]
    assert run_msm(engine, limbs_raw(sc), jo.points_mont(pts), "host") == mo.msm(sc, pts)


# 2 ---- device scale: points [k_i] G, checked through fixed_base_batch ----------------------------------------------------
def generated(engine, rng, n):
    k = [int(x) for x in rng.integers(1, 1 << 62, n)]
    pts, ok = engine.fixed_base_batch(to_mem(jubjub_limbs(k), "device"), mont(G))
    assert host(ok).all()
    return k, pts


def expect_fb(engine, total):
    out, ok = engine.fixed_base_batch(jubjub_limbs([total % N]), mont(G))
    return jo.points_from_mont(out)[0]


@pytest.mark.parametrize("kind,n", [("random", CHUNK - 1), ("random", CHUNK + 1), ("random", 3 * CHUNK + 5),
                                    ("equal", 3 * CHUNK + 5), ("zero", CHUNK + 1), ("one", CHUNK + 1),
                                    ("random", 1 << 20)])
def test_chunks_and_skew_against_fixed_base(engine, kind, n):
    rng = np.random.default_rng(n)
    k, pts = generated(engine, rng, n)
    if kind == "random":
        s = [jo.random_secret(rng) for _ in range(n)]
    else:
        s = [{"equal": N - 12345, "zero": 0, "one": 1}[kind]] * n
    want = expect_fb(engine, sum(a * b for a, b in zip(s, k)))
    sc, hp = limbs_raw(s), host(pts)
    for mem in ("host", "device"):
        got = run_msm(engine, sc, hp, mem)
        assert got == want, (kind, n, mem)
    if kind == "zero":
        assert want == jo.IDENTITY


# 3 ---- invalid items are skipped and counted ------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", SPACES)
def test_invalid_items_skipped_and_counted(engine, mem, async_):
    rng = np.random.default_rng(3)
    n = 40
    pts = [jo.random_point(rng) for _ in range(n)]
    sc = [jo.random_secret(rng) for _ in range(n)]
    rows = jo.points_mont(pts)
    srows = limbs_raw(sc)
    bad = {3: "scalar", 9: "scalar_max", 17: "u", 23: "v", 31: "off"}
    for i, what in bad.items():
        if what == "scalar":
            srows[i] = limbs_raw([N])[0]
        elif what == "scalar_max":
            srows[i] = limbs_raw([(1 << 256) - 1])[0]
        elif what == "u":
            rows[i, 0] = limbs_raw([P])[0]
        elif what == "v":
            rows[i, 1] = limbs_raw([(1 << 256) - 1])[0]
        else:
            rows[i] = jo.points_mont([jo.off_curve_point(rng)])[0]
    want = mo.msm([s for i, s in enumerate(sc) if i not in bad], [p for i, p in enumerate(pts) if i not in bad])
    assert run_msm(engine, srows, rows, mem, async_) == want
    assert engine.last_msm_invalid() == len(bad)


# 4 ---- refused calls and injected chunk failures -------------------------------------------------------------------------
def test_refused_calls(engine):
    lib, ctx = _native.lib(), engine._ctx
    sc, pts, out = np.zeros((4, 4), np.uint64), jo.points_mont([G] * 4), np.zeros((2, 4), np.uint64)
    ptr = lambda a: a.ctypes.data
    assert lib.p252_jubjub_msm(ctx, None, ptr(pts), 4, ptr(out), None, 0) != 0
    assert lib.p252_jubjub_msm(ctx, ptr(sc), ptr(pts), 4, None, None, 0) != 0
    import torch
    d = torch.zeros(4 * 4 + 2, dtype=torch.int64, device="cuda")
    dp = torch.zeros(4 * 8, dtype=torch.int64, device="cuda")
    do = torch.zeros(8, dtype=torch.int64, device="cuda")
    assert lib.p252_jubjub_msm(ctx, d.data_ptr() + 8, dp.data_ptr(), 4, do.data_ptr(), None, _native.MEM_DEVICE) != 0
    # verify_all: NULL answer, n_public not 1 or n, off-curve base (also for n == 0)
    u, R, m, w = np.zeros((4, 4), np.uint64), jo.points_mont([G] * 4), np.zeros((4, 4), np.uint64), np.ones((4, 4), np.uint64)
    ans = ctypes.c_uint8(9)
    gm = mont(G)
    assert lib.p252_schnorr_verify_all(ctx, ptr(pts), 4, ptr(u), ptr(R), ptr(m), ptr(w), 4, ptr(gm), None, None, 0) != 0
    assert lib.p252_schnorr_verify_all(ctx, ptr(pts), 2, ptr(u), ptr(R), ptr(m), ptr(w), 4, ptr(gm), ctypes.byref(ans),
                                       None, 0) != 0
    off = jo.points_mont([jo.off_curve_point(np.random.default_rng(1))])[0]
    rc = lib.p252_schnorr_verify_all(ctx, ptr(pts), 1, ptr(u), ptr(R), ptr(m), ptr(w), 0, ptr(off), ctypes.byref(ans), None, 0)
    assert rc != 0 and ans.value == 9
    rc = lib.p252_schnorr_verify_all(ctx, ptr(pts), 1, ptr(u), ptr(R), ptr(m), ptr(w), 0, ptr(gm), ctypes.byref(ans), None, 0)
    assert rc == 0 and ans.value == 1


def test_injected_chunk_failure_then_retry(engine):
    rng = np.random.default_rng(5)
    n = 2 * CHUNK + 77
    k, pts = generated(engine, rng, n)
    s = [int(x) for x in rng.integers(0, 1 << 62, n)]
    want = expect_fb(engine, sum(a * b for a, b in zip(s, k)))
    hp = host(pts)
    for chunk in (0, 2):
        _native.lib().p252_debug_fail_chunk(engine._ctx, chunk)
        with pytest.raises(pb.EngineError):
            engine.jubjub_msm(limbs_raw(s), hp)
        assert run_msm(engine, limbs_raw(s), hp, "host") == want


# 5 ---- all-or-nothing verification -------------------------------------------------------------------------------------
def signed_batch(engine, n, seed, one_key):
    rng = np.random.default_rng(seed)
    keys = [signer(s) for s in (21, 22, 23)]
    pick = np.zeros(n, dtype=np.int64) if one_key else rng.integers(0, 3, n)
    sks = jubjub_limbs([kk[0] for kk in keys])[pick]
    pks = jo.points_mont([kk[1] for kk in keys])
    r, m = to_mem(random_r(rng, n), "device"), to_mem(random_m(rng, n), "device")
    u, R, ok = engine.schnorr_sign_batch(to_mem(sks[:1] if one_key else sks, "device"), r, m, mont(G))
    assert host(ok).all()
    pk = to_mem(pks[:1] if one_key else pks[pick], "device")
    return pk, u, R, m


@pytest.mark.parametrize("one_key", [True, False])
def test_verify_all_large_batch_and_tampering(engine, one_key):
    import torch
    n = 1 << 18
    pk, u, R, m = signed_batch(engine, n, 31 if one_key else 32, one_key)
    gm = mont(G)
    assert engine.schnorr_verify_all(pk, u, R, m, gm) is True
    assert engine.last_schnorr_invalid() == 0
    assert host(engine.schnorr_verify_batch(pk, u, R, m, gm)).all()
    for i in (0, n // 2, n - 1):
        for what in ("u", "msg", "R"):
            uu, mm, RR = u.clone(), m.clone(), R.clone()
            if what == "u":
                uu[i, 0] ^= 1
            elif what == "msg":
                mm[i, 0] ^= 1
            else:
                RR[i] = R[(i + 1) % n]
            assert engine.schnorr_verify_all(pk, uu, RR, mm, gm) is False, (i, what)
            assert engine.last_schnorr_invalid() == 0
    # async on device buffers: the answer after sync
    assert engine.schnorr_verify_all(pk, u, R, m, gm, async_=True) is None
    engine.sync()
    assert engine.last_verify_all() is True
    # host buffers
    hpk = host(pk) if one_key else host(pk)[:4096]
    assert engine.schnorr_verify_all(hpk, host(u)[:4096], host(R)[:4096], host(m)[:4096], gm) is True
    del torch


def test_verify_all_invalid_and_off_curve(engine):
    n = 5000
    pk, u, R, m = signed_batch(engine, n, 33, False)
    gm = mont(G)
    uu = host(u).copy()
    uu[17] = limbs_raw([N])[0]
    assert engine.schnorr_verify_all(host(pk), uu, host(R), host(m), gm) is False
    assert engine.last_schnorr_invalid() == 1
    w = np.ones((n, 4), dtype=np.uint64)
    w[99] = limbs_raw([N])[0]
    assert engine.schnorr_verify_all(host(pk), host(u), host(R), host(m), gm, weights=w) is False
    assert engine.last_schnorr_invalid() == 1
    RR = host(R).copy()
    RR[4321] = jo.points_mont([jo.off_curve_point(np.random.default_rng(2))])[0]
    assert engine.schnorr_verify_all(host(pk), host(u), RR, host(m), gm) is False
    assert engine.last_schnorr_invalid() == 0


def test_verify_all_equals_and_of_per_item(engine):
    rng = np.random.default_rng(6)
    n = 3000
    pk, u, R, m = signed_batch(engine, n, 34, False)
    gm = mont(G)
    for trial in range(4):
        uu = host(u).copy()
        for i in rng.choice(n, trial, replace=False):
            uu[i, 0] ^= 2
        per = host(engine.schnorr_verify_batch(pk, to_mem(uu, "device"), R, m, gm))
        assert engine.schnorr_verify_all(pk, to_mem(uu, "device"), R, m, gm) == bool(per.all())


def test_verify_all_is_cofactored(engine):
    """R + T for an order-8 T: the per-item call rejects the signature, the cofactored batch equation accepts it"""
    rng = np.random.default_rng(9)
    sk, pk = signer(21)
    t = jo.small_order_points(rng)[4]
    ms = [int(x) for x in rng.integers(1, 1 << 62, 8)]
    us, Rs = [], []
    for i, mi in enumerate(ms):
        r = jo.random_secret(rng)
        Rp = jo.mul(r, G) if i != 5 else jo.add(jo.mul(r, G), t)
        us.append((r - so.challenge(Rp, mi) * sk) % N)
        Rs.append(Rp)
    assert mo.verify_all([pk], us, Rs, ms, [1] * 8) is True and mo.verify_all([pk], us, Rs, ms, [1] * 8, cofactor=1) is False
    args = (jo.points_mont([pk]), jubjub_limbs(us), jo.points_mont(Rs), fr_rows(ms), mont(G))
    assert list(engine.schnorr_verify_batch(*args)) == [1] * 5 + [0] + [1] * 2
    assert engine.schnorr_verify_all(*args) is True
    us[5] = (us[5] + 1) % N
    args = (jo.points_mont([pk]), jubjub_limbs(us), jo.points_mont(Rs), fr_rows(ms), mont(G))
    assert engine.schnorr_verify_all(*args) is False


# 6 ---- verify_all: injected chunk failures, refused device buffers, default weights, the C and C++ programs -----------------
VERIFY_CHUNK = 45056     # a staged verify_all chunk with n_public = n: 24 MiB over the ~560 staged bytes of an item


def test_verify_all_injected_chunk_failure_then_retry(engine):
    n = 3 * VERIFY_CHUNK + 5
    pk, u, R, m = signed_batch(engine, n, 36, False)
    gm = mont(G)
    hpk, hu, hR, hm = host(pk), host(u), host(R), host(m)
    w = limbs_raw([(0x9e3779b97f4a7c15 * (i + 1)) % (1 << 128) or 1 for i in range(n)])
    for chunk in (0, 2, 4):
        _native.lib().p252_debug_fail_chunk(engine._ctx, chunk)
        with pytest.raises(pb.EngineError):
            engine.schnorr_verify_all(hpk, hu, hR, hm, gm, weights=w)
        assert engine.schnorr_verify_all(hpk, hu, hR, hm, gm, weights=w) is True
        assert engine.last_schnorr_invalid() == 0
    hu2 = hu.copy()
    hu2[n - 3, 1] ^= 4                                  # a failure in the last chunk after a retry
    _native.lib().p252_debug_fail_chunk(engine._ctx, 1)
    with pytest.raises(pb.EngineError):
        engine.schnorr_verify_all(hpk, hu2, hR, hm, gm, weights=w)
    assert engine.schnorr_verify_all(hpk, hu2, hR, hm, gm, weights=w) is False
    # device buffers go through the same pipeline
    _native.lib().p252_debug_fail_chunk(engine._ctx, 0)
    with pytest.raises(pb.EngineError):
        engine.schnorr_verify_all(pk, u, R, m, gm)
    assert engine.schnorr_verify_all(pk, u, R, m, gm) is True     # DEVICE, synchronous, weights drawn by the engine


def test_verify_all_refuses_misaligned_device_buffers(engine):
    import torch
    n = 8
    pk, u, R, m = signed_batch(engine, n, 37, False)
    w = to_mem(np.ones((n, 4), np.uint64), "device")
    gm = mont(G)
    lib, ctx = _native.lib(), engine._ctx
    flat = {name: torch.zeros(t.numel() + 2, dtype=torch.int64, device="cuda") for name, t in
            (("pk", pk), ("u", u), ("R", R), ("m", m), ("w", w))}
    for name, t in (("pk", pk), ("u", u), ("R", R), ("m", m), ("w", w)):
        flat[name][1:1 + t.numel()] = t.reshape(-1)
    torch.cuda.synchronize()
    ptrs = {name: t.data_ptr() for name, t in (("pk", pk), ("u", u), ("R", R), ("m", m), ("w", w))}
    ans, cnt = ctypes.c_uint8(9), ctypes.c_size_t(7)
    for bad in ptrs:
        p = dict(ptrs)
        p[bad] = flat[bad].data_ptr() + 8                   # 8-byte aligned, not 16
        rc = lib.p252_schnorr_verify_all(ctx, p["pk"], n, p["u"], p["R"], p["m"], p["w"], n, gm.ctypes.data,
                                         ctypes.byref(ans), ctypes.byref(cnt), _native.MEM_DEVICE)
        assert rc != 0 and ans.value == 9 and cnt.value == 7, bad
    rc = lib.p252_schnorr_verify_all(ctx, ptrs["pk"], n, ptrs["u"], ptrs["R"], ptrs["m"], ptrs["w"], n, gm.ctypes.data,
                                     ctypes.byref(ans), ctypes.byref(cnt), _native.MEM_DEVICE)
    assert rc == 0 and ans.value == 1 and cnt.value == 0


def test_c_msm_smoke_gpu():
    from test_msm_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "MSM_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_msm_mirror_gpu():
    from test_msm_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "msm mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
