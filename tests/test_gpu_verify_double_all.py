"""All-or-nothing verification of double-key signatures on the device (p252_schnorr_verify_double_all) against the model
of verify_double_all_oracle.py and against the AND of the per-item call p252_schnorr_verify_double_batch: genuine batches
of every size and shape, note spends, tampering in every chunk, invalid items, the cofactor, the two independent weight
arrays, edge weights, n == 0, refused calls, injected chunk failures, the table cache and the C and C++ programs."""
import ctypes

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
import schnorr_double_oracle as sdo
import stealth_oracle as so
import verify_double_all_oracle as vo
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_gpu_msm import limbs_raw
from test_gpu_schnorr import fr_rows, random_m, random_r
from test_gpu_schnorr_double import g_prime, key_pair
from test_gpu_stealth import CANARY, host, mont, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
MEMS = [("host", False), ("device", False), ("device", True)]
# staged chunks (DESIGN.md section 4): HOST buffers with n_public = n, DEVICE buffers with n_public = n
CHUNK_HOST, CHUNK_DEVICE = 25856, 42624


def signed(engine, n, seed, one_pair):
    """n signatures of schnorr_sign_double_batch on the device, under one key pair or one per item:
    (pk, pk', u, R, R', msg), all device tensors"""
    rng = np.random.default_rng(seed)
    gm, gpm = mont(G), mont(g_prime())
    sk = to_mem(random_r(rng, 1 if one_pair else n), "device")
    pk, ok1 = engine.fixed_base_batch(sk, gm)
    pkp, ok2 = engine.fixed_base_batch(sk, gpm)
    m = to_mem(random_m(rng, n), "device")
    u, R, Rp, ok = engine.schnorr_sign_double_batch(sk, to_mem(random_r(rng, n), "device"), m, gm, gpm)
    assert host(ok1).all() and host(ok2).all() and host(ok).all()
    return pk, pkp, u, R, Rp, m


def weights(n, seed):
    rng = np.random.default_rng(seed)
    w = rng.integers(1, 1 << 63, (2, n, 4), dtype=np.uint64)
    w[:, :, 2:] = 0                                              # 128-bit weights
    return w[0].copy(), w[1].copy()


def verify_all(engine, args, mem="device", async_=False, w=None, wp=None):
    """the answer of schnorr_verify_double_all on args (pk, pk', u, R, R', msg) moved to `mem`"""
    a = [to_mem(host(x), mem) for x in args]
    w = None if w is None else to_mem(w, mem)
    wp = None if wp is None else to_mem(wp, mem)
    got = engine.schnorr_verify_double_all(*a, mont(G), mont(g_prime()), weights=w, weights_p=wp, async_=async_)
    if async_:
        assert got is None
        engine.sync()
        return engine.last_verify_double_all()
    assert got == engine.last_verify_double_all()
    return got


def per_item_and(engine, args):
    return bool(host(engine.schnorr_verify_double_batch(*args, mont(G), mont(g_prime()))).all())


def rows_of(pks, pkps, us, Rs, Rps, ms):
    """model values -> host arrays (coordinates >= p and scalars >= r_J are passed through raw)"""
    return points(pks), points(pkps), limbs_raw(us), points(Rs), points(Rps), fr_rows(ms)


def points(pts):
    out = np.zeros((len(pts), 2, 4), dtype=np.uint64)
    for i, p in enumerate(pts):
        out[i] = jo.points_mont([p])[0] if all(0 <= x < P for x in p) else limbs_raw(list(p))
    return out


def ints(rows):
    return [sum(int(r[k]) << (64 * k) for k in range(4)) for r in rows]


# 1 ---- genuine batches: every size, both shapes, every memory space, against the AND of the per-item call ----------------
@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("one_pair", [True, False])
def test_genuine_batches_of_every_size(engine, mem, async_, one_pair):
    for n in (1, 31, 33, 127, 129):
        args = signed(engine, n, 1000 + n, one_pair)
        assert per_item_and(engine, args)
        assert verify_all(engine, args, mem, async_) is True, n
        assert engine.last_schnorr_double_invalid() == 0


@pytest.mark.parametrize("one_pair", [True, False])
def test_three_chunks_plus_5_and_2_18(engine, one_pair):
    for n, mems in ((3 * CHUNK_HOST + 5, ("host", "device")), (1 << 18, ("device",))):
        args = signed(engine, n, 1100 + n, one_pair)
        assert per_item_and(engine, args)
        w, wp = weights(n, 7)
        for mem in mems:
            assert verify_all(engine, args, mem, w=w, wp=wp) is True, (n, mem)
            assert engine.last_schnorr_double_invalid() == 0


def test_note_spends_verify_under_note_keys(engine):
    """spend signatures of note_sign_double_batch verify under (note_pk of stealth_address_batch, pk')"""
    rng = np.random.default_rng(1200)
    n = 4096
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    gm, gpm = mont(G), mont(g_prime())
    Rn, note_pk, okn = engine.stealth_address_batch(to_mem(random_r(rng, n), "device"), gm,
                                                   to_mem(jo.points_mont([A]), "device"), to_mem(jo.points_mont([B]), "device"))
    m = to_mem(random_m(rng, n), "device")
    u, R, Rp, pkp, ok = engine.note_sign_double_batch(to_mem(jubjub_limbs([a]), "device"), to_mem(jubjub_limbs([b]), "device"),
                                                      Rn, to_mem(random_r(rng, n), "device"), m, gm, gpm)
    assert host(okn).all() and host(ok).all()
    args = (note_pk, pkp, u, R, Rp, m)
    assert verify_all(engine, args) is True and per_item_and(engine, args)
    m[n // 3, 0] ^= 1
    assert verify_all(engine, args) is False and engine.last_schnorr_double_invalid() == 0


# 2 ---- tampering: every component, in the first, a middle and the last chunk -------------------------------------------
@pytest.mark.parametrize("one_pair", [True, False])
def test_tampering_in_every_chunk(engine, one_pair):
    import torch
    n = 1 << 18
    args = signed(engine, n, 1300, one_pair)
    w, wp = weights(n, 8)
    assert verify_all(engine, args, w=w, wp=wp) is True
    parts = ("u", "msg", "R", "R'") + (() if one_pair else ("PK", "PK'"))
    for i in (0, n // 2, n - 1):
        for what in parts:
            t = [x.clone() for x in args]
            k = {"PK": 0, "PK'": 1, "u": 2, "R": 3, "R'": 4, "msg": 5}[what]
            if what in ("u", "msg"):
                t[k][i, 0] ^= 2
            else:
                t[k][i] = args[k][(i + 1) % n]                  # another curve point
            torch.cuda.synchronize()
            assert verify_all(engine, t, w=w, wp=wp) is False, (i, what)
            assert engine.last_schnorr_double_invalid() == 0
            assert not per_item_and(engine, t)


def _small(seed, n=6):
    """n model signatures under n key pairs: lists (pks, pkps, us, Rs, Rps, ms)"""
    rng = np.random.default_rng(seed)
    cols = [[] for _ in range(6)]
    for i in range(n):
        sk = jo.random_secret(rng)
        u, R, Rp = sdo.sign_double(sk, jo.random_secret(rng), 11 * i + 3, g_prime())
        for c, v in zip(cols, key_pair(sk) + (u, R, Rp, 11 * i + 3)):
            c.append(v)
    return cols


def _model(cols, w, wp):
    return vo.verify_double_all(*cols, ints(w), ints(wp), g_prime())


@pytest.mark.parametrize("mem,async_", MEMS)
def test_tampering_against_model(engine, mem, async_):
    cols = _small(1400)
    w, wp = weights(6, 9)
    assert _model(cols, w, wp) is True and verify_all(engine, rows_of(*cols), mem, async_, w, wp) is True
    for what in ("u+1", "m+1", "R", "R'", "swap", "PK", "PK'=PK"):
        c = [list(x) for x in cols]
        if what == "u+1":
            c[2][3] = (c[2][3] + 1) % N
        elif what == "m+1":
            c[5][3] += 1
        elif what == "R":
            c[3][3] = jo.add(c[3][3], G)
        elif what == "R'":
            c[4][3] = jo.add(c[4][3], g_prime())
        elif what == "swap":
            c[3][3], c[4][3] = c[4][3], c[3][3]
        elif what == "PK":
            c[0][3] = jo.add(c[0][3], G)
        else:
            c[1][3] = c[0][3]
        assert _model(c, w, wp) is False, what
        assert verify_all(engine, rows_of(*c), mem, async_, w, wp) is False, what
        assert engine.last_schnorr_double_invalid() == 0


# 3 ---- invalid items and off-curve R --------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_items_counted_once(engine, mem):
    rng = np.random.default_rng(1500)
    cols = _small(1501)
    w, wp = weights(6, 10)
    base = rows_of(*cols)
    cases = {"u": (2, limbs_raw([N])[0]), "msg": (5, limbs_raw([P])[0]), "R.u": (3, None), "R'.v": (4, None),
             "PK": (0, jo.points_mont([jo.off_curve_point(rng)])[0]), "PK'": (1, jo.points_mont([jo.off_curve_point(rng)])[0])}
    for what, (k, val) in cases.items():
        a = [x.copy() for x in base]
        if what == "R.u":
            a[3][2, 0] = limbs_raw([P + 3])[0]
        elif what == "R'.v":
            a[4][2, 1] = limbs_raw([(1 << 256) - 1])[0]
        else:
            a[k][2] = val
        assert verify_all(engine, a, mem, w=w, wp=wp) is False, what
        assert engine.last_schnorr_double_invalid() == 1, what
    for which in (0, 1):                                       # a weight >= r_J
        ww = [w.copy(), wp.copy()]
        ww[which][4] = limbs_raw([N + which])[0]
        assert verify_all(engine, base, mem, w=ww[0], wp=ww[1]) is False
        assert engine.last_schnorr_double_invalid() == 1
    a = [x.copy() for x in base]                               # several items, one of them invalid three times over
    a[2][0] = limbs_raw([N])[0]
    a[5][0] = limbs_raw([P])[0]
    a[0][0] = jo.points_mont([jo.off_curve_point(rng)])[0]
    a[2][5] = limbs_raw([N + 7])[0]
    ww = wp.copy()
    ww[3] = limbs_raw([(1 << 256) - 1])[0]
    assert verify_all(engine, a, mem, w=w, wp=ww) is False and engine.last_schnorr_double_invalid() == 3
    for k in (3, 4):                                           # a canonical R or R' off the curve: False, not counted
        a = [x.copy() for x in base]
        a[k][1] = jo.points_mont([jo.off_curve_point(rng)])[0]
        assert verify_all(engine, a, mem, w=w, wp=wp) is False and engine.last_schnorr_double_invalid() == 0


# 4 ---- the cofactor, the two weight arrays, edge weights ----------------------------------------------------------------
def test_torsion_shifted_R_passes(engine):
    rng = np.random.default_rng(1600)
    T = jo.order8_point(rng)
    cols = _small(1601, 4)
    sk = jo.random_secret(rng)
    pk, pkp = key_pair(sk)
    for i, which in ((1, "R"), (2, "R'")):
        r, m = jo.random_secret(rng), 1000 + i
        R, Rp = jo.mul(r, G), jo.mul(r, g_prime())
        R, Rp = (jo.add(R, T), Rp) if which == "R" else (R, jo.add(Rp, T))
        u = (r - sdo.challenge2(R, Rp, m) * sk) % N
        for c, v in zip(cols, (pk, pkp, u, R, Rp, m)):
            c[i] = v
    w, wp = weights(4, 11)
    assert _model(cols, w, wp) is True
    assert vo.verify_double_all(*cols, ints(w), ints(wp), g_prime(), cofactor=1) is False
    a = rows_of(*cols)
    assert list(host(engine.schnorr_verify_double_batch(*a, mont(G), mont(g_prime())))) == [1, 0, 0, 1]
    for mem in ("host", "device"):
        assert verify_all(engine, a, mem, w=w, wp=wp) is True


def test_equal_weights_accept_a_cancelling_signature(engine):
    """R = [r] G + D, R' = [r] G' - D: passes with weights_p == weights, fails with independent weights"""
    rng = np.random.default_rng(1700)
    cols = _small(1701, 4)
    sk = jo.random_secret(rng)
    pk, pkp = key_pair(sk)
    u, R, Rp = vo.cancelling_signature(sk, jo.random_secret(rng), 42, jo.random_subgroup_point(rng), g_prime())
    for c, v in zip(cols, (pk, pkp, u, R, Rp, 42)):
        c[2] = v
    w, wp = weights(4, 12)
    assert _model(cols, w, w) is True and _model(cols, w, wp) is False
    a = rows_of(*cols)
    assert list(host(engine.schnorr_verify_double_batch(*a, mont(G), mont(g_prime())))) == [1, 1, 0, 1]
    for mem in ("host", "device"):
        assert verify_all(engine, a, mem, w=w, wp=w) is True
        assert verify_all(engine, a, mem, w=w, wp=wp) is False
        assert verify_all(engine, a, mem) is False               # fresh weights drawn by the engine


def test_edge_weights_equal_the_model(engine):
    cols = _small(1800, 4)
    bad = [list(x) for x in cols]
    bad[2][1] = (bad[2][1] + 1) % N
    for z in (1, N - 1, (1 << 128) - 1):
        for zp in (1, N - 1, (1 << 128) - 1):
            w, wp = limbs_raw([z] * 4), limbs_raw([zp] * 4)
            for c in (cols, bad):
                want = _model(c, w, wp)
                assert verify_all(engine, rows_of(*c), "device", w=w, wp=wp) is want, (z, zp)
    # a zero weight leaves its equation unchecked
    pkbad = [list(x) for x in cols]
    pkbad[0][1] = jo.add(pkbad[0][1], G)                       # only item 1's first equation fails
    w, wp = weights(4, 13)
    w[1] = 0
    assert _model(pkbad, w, wp) is True and verify_all(engine, rows_of(*pkbad), "host", w=w, wp=wp) is True
    w, wp = weights(4, 13)
    wp[1] = 0
    assert _model(pkbad, w, wp) is False and verify_all(engine, rows_of(*pkbad), "host", w=w, wp=wp) is False


# 5 ---- n == 0 and refused calls: nothing written, nothing launched ---------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_n_zero_and_refused_calls(engine, mem):
    rng = np.random.default_rng(1900)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 4
    gm, gpm = mont(G), mont(g_prime())
    sc = to_mem(jubjub_limbs([3] * n), mem)
    pts = to_mem(jo.points_mont([G] * n), mem)
    m = to_mem(fr_rows([1] * n), mem)
    ans, cnt = ctypes.c_uint8(9), ctypes.c_size_t(CANARY)

    def call(g=gm.ctypes.data, gp=gpm.ctypes.data, pk=pts, pkp=pts, npub=n, u=sc, R=pts, Rp=pts, msg=m, w=sc, wp=sc,
             nn=n, answer=True):
        p = lambda x: None if x is None else (x if isinstance(x, int) else P_(x))
        return lib.p252_schnorr_verify_double_all(ctx, p(pk), p(pkp), npub, p(u), p(R), p(Rp), p(msg), p(w), p(wp), nn,
                                                  g, gp, ctypes.byref(ans) if answer else None, ctypes.byref(cnt), flags)

    before = engine.launch_count
    assert call(nn=0, npub=1) == 0 and ans.value == 1 and cnt.value == 0
    assert engine.schnorr_verify_double_all(pts[:0], pts[:0], sc[:0], pts[:0], pts[:0], m[:0], gm, gpm) is True
    assert engine.launch_count == before                       # n == 0: no launch
    ans.value, cnt.value = 9, CANARY
    for bad in [mont(jo.off_curve_point(rng)), mont((G[0] + P, G[1])), mont((G[0], G[1] + P))]:
        for nn, npub in ((n, n), (0, 1)):
            assert call(g=bad.ctypes.data, nn=nn, npub=npub) == 6 and call(gp=bad.ctypes.data, nn=nn, npub=npub) == 6
        with pytest.raises(pb.InvalidPoint):
            engine.schnorr_verify_double_all(pts, pts, sc, pts, pts, m, gm, bad)
    assert call(g=None) == -1 and call(gp=None) == -1 and call(answer=False) == -1
    for name in ("pk", "pkp", "u", "R", "Rp", "msg", "w", "wp"):
        assert call(**{name: None}) == -1, name
    assert call(npub=2) == -1 and call(npub=0) == -1
    if mem == "device":                                          # misaligned DEVICE rows
        for name in ("pk", "pkp", "u", "R", "Rp", "msg", "w", "wp"):
            base = {"pk": pts, "pkp": pts, "u": sc, "R": pts, "Rp": pts, "msg": m, "w": sc, "wp": sc}[name]
            assert call(**{name: P_(base) + 8}) == -1, name
    assert ans.value == 9 and cnt.value == CANARY
    assert engine.launch_count == before


# 6 ---- injected chunk failures, the table cache, the C and C++ programs ------------------------------------------------
def _chunks(n, chunk):
    """the chunk count of the staged pipeline (first chunks chunk / 8, / 4, / 2 for batches over two chunks)"""
    cur = max(1024, chunk // 8 // 128 * 128) if n > 2 * chunk else chunk
    k = off = 0
    while off < n:
        off += min(cur, n - off)
        k += 1
        cur = min(chunk, cur * 2)
    return k


@pytest.mark.parametrize("mem,chunk", [("host", CHUNK_HOST), ("device", CHUNK_DEVICE)])
def test_injected_chunk_failures_then_retry(engine, mem, chunk):
    n = 3 * chunk + 5
    args = signed(engine, n, 2000, False)
    w, wp = weights(n, 14)
    a = [to_mem(host(x), mem) for x in args]
    wm, wpm = to_mem(w, mem), to_mem(wp, mem)
    last = _chunks(n, chunk) - 1
    assert last >= 3
    for fail_at in (0, 2, last):
        assert _native.lib().p252_debug_fail_chunk(engine._ctx, fail_at) == 0
        with pytest.raises(pb.EngineError):
            engine.schnorr_verify_double_all(*a, mont(G), mont(g_prime()), weights=wm, weights_p=wpm)
        assert engine.schnorr_verify_double_all(*a, mont(G), mont(g_prime()), weights=wm, weights_p=wpm) is True
        assert engine.last_schnorr_double_invalid() == 0
    u = host(args[2]).copy()
    u[n - 2, 1] ^= 4                                           # a wrong u in the last chunk, after a failed call
    a[2] = to_mem(u, mem)
    _native.lib().p252_debug_fail_chunk(engine._ctx, 1)
    with pytest.raises(pb.EngineError):
        engine.schnorr_verify_double_all(*a, mont(G), mont(g_prime()), weights=wm, weights_p=wpm)
    assert engine.schnorr_verify_double_all(*a, mont(G), mont(g_prime()), weights=wm, weights_p=wpm) is False


def test_table_cache_by_launch_count(engine):
    """after schnorr_verify_double_batch with the same G, G' the call builds no table, and it does not evict the
    single-base slot"""
    n = 300
    args = [host(x) for x in signed(engine, n, 2100, False)]
    w, wp = weights(n, 15)
    third = mont(jo.mul(12345, G))
    sl = jubjub_limbs([5, 6, 7])

    def launches(call):
        before = engine.launch_count
        call()
        return engine.launch_count - before

    once = lambda: verify_all(engine, args, "host", w=w, wp=wp)
    launches(once)
    L = launches(once)                                           # no table built
    assert launches(once) == L
    engine.fixed_base_batch(sl, mont(jo.mul(777, G)))            # the single-base slot takes another base
    assert launches(lambda: engine.schnorr_verify_double_batch(*args, mont(G), mont(g_prime()))) == 3
    assert launches(once) == L
    engine.fixed_base_batch(sl, third)
    assert launches(once) == L
    assert launches(lambda: engine.fixed_base_batch(sl, third)) == 1   # the single-base slot is not evicted
    engine.schnorr_sign_double_batch(sl, sl, fr_rows([1, 2, 3]), mont(G), mont(g_prime()))
    assert launches(once) == L


def test_c_verify_double_all_smoke_gpu():
    from test_verify_double_all_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "VERIFY_DOUBLE_ALL_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_verify_double_all_mirror_gpu():
    from test_verify_double_all_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "verify double all mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
