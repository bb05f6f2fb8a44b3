"""Double-key Schnorr signatures on the device (p252_schnorr_sign_double_batch, p252_schnorr_verify_double_batch,
p252_note_sign_double_batch) against the model of schnorr_double_oracle.py (affine complete addition, double-and-add, the
Python Hades, big-integer arithmetic modulo r_J), against the existing calls they are built from (fixed_base_batch,
hash_batch_truncated, stealth_address_batch, nullifier_batch), and the calls' own plumbing: invalid items, refused calls,
batch sizes, staging wipes, injected chunk failures, launches per chunk and the two-generator table cache."""
import ctypes
import functools

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_edges as je
import jubjub_oracle as jo
import nullifier_oracle as no
import poseidon252_b200 as pb
import schnorr_double_oracle as sdo
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs, to_mont
from test_gpu_schnorr import M_EDGES, R_EDGES, SK_EDGES, fr_rows, ints, random_m, random_r
from test_gpu_stealth import CANARY, _sizes, host, mont, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
MEMS = [("host", False), ("device", False), ("device", True)]


@functools.lru_cache(maxsize=None)
def g_prime():
    """a random point of the prime-order subgroup as G' (GENERATOR_NUMS is not pinned here)"""
    return jo.random_subgroup_point(np.random.default_rng(800))


@functools.lru_cache(maxsize=None)
def mul(k, pt):
    return jo.mul(k, pt)


@functools.lru_cache(maxsize=None)
def model_sign(sk, r, m):
    """(u, R, R', ok) as the device writes them: zeroed rows for an invalid item"""
    s = sdo.sign_double(sk, r, m, g_prime())
    return (0, (0, 0), (0, 0), 0) if s is None else s + (1,)


@functools.lru_cache(maxsize=None)
def model_note(a, b, R_note, r, m):
    """(u, R, R', pk', ok) as the device writes them"""
    s = sdo.note_sign_double(a, b, R_note, r, m, g_prime())
    return (0, (0, 0), (0, 0), (0, 0), 0) if s is None else s[0] + (s[1], 1)


@functools.lru_cache(maxsize=None)
def model_verify(pk, pkp, u, R, Rp, m):
    """1 / 0 / None (invalid), with the model's scalar multiplications cached"""
    Gp = g_prime()
    if sdo.verify_double(pk, pkp, u, R, Rp, m, Gp) is None:
        return None
    c = sdo.challenge2(R, Rp, m)
    return int(jo.add(mul(u, G), mul(c, pk)) == tuple(R) and jo.add(mul(u, Gp), mul(c, pkp)) == tuple(Rp))


def rows_of(points, ok):
    out = jo.points_mont(points)
    out[ok == 0] = 0
    return out


def expect(rows):
    """the model's rows -> (u (n, 4), point arrays..., ok)"""
    ok = np.array([x[-1] for x in rows], dtype=np.uint8)
    u = jubjub_limbs([x[0] for x in rows])
    return (u,) + tuple(rows_of([x[k] for x in rows], ok) for k in range(1, len(rows[0]) - 1)) + (ok,)


def key_pair(sk):
    return mul(sk, G), mul(sk, g_prime())


def done(engine, async_):
    if async_:
        engine.sync()


# 1 ---- signing against the model: edge sk x r x m ------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("n_secret", ["one", "n"])
def test_sign_against_model(engine, mem, async_, n_secret):
    grid = [(sk, r, m) for sk in SK_EDGES for r in R_EDGES for m in M_EDGES]
    if n_secret == "one":
        grid = [(SK_EDGES[-1], r, m) for _, r, m in grid]
    sks, rs, ms = zip(*grid)
    want = expect([model_sign(*x) for x in grid])
    assert want[-1].all()
    k = 1 if n_secret == "one" else len(grid)
    got = engine.schnorr_sign_double_batch(to_mem(jubjub_limbs(sks[:k]), mem), to_mem(jubjub_limbs(rs), mem),
                                           to_mem(fr_rows(ms), mem), mont(G), mont(g_prime()), async_=async_)
    done(engine, async_)
    for g, w in zip(got, want):
        assert np.array_equal(host(g), w)
    assert engine.last_schnorr_double_invalid() == 0
    u, R, Rp = pb.schnorr_sign_double(sks[5], rs[5], fr_rows([ms[5]])[0], mont(G), mont(g_prime()), engine=engine)
    assert np.array_equal(u, want[0][5]) and np.array_equal(R, want[1][5]) and np.array_equal(Rp, want[2][5])


# 2 ---- note signing against the model: edge R_note, a, b, r, m --------------------------------------------------------
@functools.lru_cache(maxsize=None)
def edge_R():
    """R_note at the field's edges: one prime-subgroup point of every class, the first point of every class, G and the
    small-order points"""
    rng = np.random.default_rng(801)
    pts = [e.pt for e in je.subgroup_edges()] + [je.edges(k)[0].pt for k in je.KINDS] + [G]
    return tuple(dict.fromkeys(pts + jo.small_order_points(rng)))


@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("n_secret", ["one", "n"])
def test_note_sign_against_model(engine, mem, async_, n_secret):
    Rs = list(edge_R())
    n = len(Rs)
    A_EDGES = [1, 2, N - 1] + list(je.OUTPUT_SECRETS)
    B_EDGES = [0, 1, N - 1, (1 << 250) + 3]
    if n_secret == "n":
        a_s = [A_EDGES[i % len(A_EDGES)] for i in range(n)]
        b_s = [B_EDGES[(3 * i) % len(B_EDGES)] for i in range(n)]
        b_s[0] = N - so.hash_point(mul(a_s[0], Rs[0]))              # note_sk = 0: pk' = the identity, u = r
    else:
        a_s, b_s = [A_EDGES[4]] * n, [N - 1] * n                     # h + b wraps for every h > 0
    rs = [R_EDGES[i % len(R_EDGES)] for i in range(n)]
    ms = [M_EDGES[i % len(M_EDGES)] for i in range(n)]
    rows = [model_note(a, b, R, r, m) for a, b, R, r, m in zip(a_s, b_s, Rs, rs, ms)]
    want = expect(rows)
    assert want[-1].all()
    if n_secret == "n":
        assert rows[0][3] == jo.IDENTITY and rows[0][0] == rs[0]
    k = 1 if n_secret == "one" else n
    got = engine.note_sign_double_batch(to_mem(jubjub_limbs(a_s[:k]), mem), to_mem(jubjub_limbs(b_s[:k]), mem),
                                        to_mem(jo.points_mont(Rs), mem), to_mem(jubjub_limbs(rs), mem),
                                        to_mem(fr_rows(ms), mem), mont(G), mont(g_prime()), async_=async_)
    done(engine, async_)
    for g, w in zip(got, want):
        assert np.array_equal(host(g), w)
    assert engine.last_schnorr_double_invalid() == 0


# 3 ---- verification against the model: genuine, tampered and torsion-shifted signatures, edge keys ---------------------
def _verify_cases(rng):
    """(PK, PK', u, R, R', m) rows: genuine signatures, then every forgery of the model tests, edge keys and a PK' with a
    small-order component"""
    Gp = g_prime()
    out = []
    T = jo.order8_point(rng)
    for sk in SK_EDGES:
        pk, pkp = key_pair(sk)
        for r, m in zip(R_EDGES, M_EDGES):
            u, R, Rp, _ = model_sign(sk, r, m)
            out += [(pk, pkp, u, R, Rp, m), (pk, pkp, u, R, mul(r + 1, Gp), m), (pk, mul(sk + 1, Gp), u, R, Rp, m),
                    (pk, pkp, u, Rp, R, m), (pk, pkp, (u + 1) % N, R, Rp, m), (pk, pkp, (u - 1) % N, R, Rp, m),
                    (pk, pkp, u, R, Rp, (m + 1) % P), (pk, pk, u, R, Rp, m), (pk, jo.add(pkp, T), u, R, Rp, m)]
    for e in je.subgroup_edges() + tuple(je.edges(k)[0] for k in je.KINDS):
        u, R, Rp, _ = model_sign(SK_EDGES[-1], R_EDGES[-1], 5)
        out += [(e.pt, key_pair(SK_EDGES[-1])[1], u, R, Rp, 5), (key_pair(SK_EDGES[-1])[0], e.pt, u, R, Rp, 5)]
    return out


@pytest.mark.parametrize("mem,async_", MEMS)
def test_verify_against_model(engine, mem, async_):
    cases = _verify_cases(np.random.default_rng(802))
    want = np.array([model_verify(*c) for c in cases], dtype=np.uint8)
    assert want.sum() >= len(SK_EDGES) * len(R_EDGES) and not (want == 1).all()
    pk, pkp, u, R, Rp, m = zip(*cases)
    got = engine.schnorr_verify_double_batch(to_mem(jo.points_mont(pk), mem), to_mem(jo.points_mont(pkp), mem),
                                             to_mem(jubjub_limbs(u), mem), to_mem(jo.points_mont(R), mem),
                                             to_mem(jo.points_mont(Rp), mem), to_mem(fr_rows(m), mem), mont(G),
                                             mont(g_prime()), async_=async_)
    done(engine, async_)
    assert np.array_equal(host(got), want)
    assert engine.last_schnorr_double_verified() == int(want.sum()) and engine.last_schnorr_double_invalid() == 0


@pytest.mark.parametrize("mem", ["host", "device"])
def test_verify_one_key_pair_for_the_batch(engine, mem):
    """n_public = 1: one (PK, PK') for every signature; a signature of another key does not verify"""
    rng = np.random.default_rng(803)
    sk, sk2 = jo.random_secret(rng), jo.random_secret(rng)
    n = 40
    rs, ms = ints(random_r(rng, n)), [int(x) for x in rng.integers(0, 1 << 62, n)]
    sigs = [model_sign(sk2 if i % 5 == 3 else sk, r, m) for i, (r, m) in enumerate(zip(rs, ms))]
    pk, pkp = key_pair(sk)
    got = engine.schnorr_verify_double_batch(to_mem(jo.points_mont([pk]), mem), to_mem(jo.points_mont([pkp]), mem),
                                             to_mem(jubjub_limbs([s[0] for s in sigs]), mem),
                                             to_mem(jo.points_mont([s[1] for s in sigs]), mem),
                                             to_mem(jo.points_mont([s[2] for s in sigs]), mem), to_mem(fr_rows(ms), mem),
                                             mont(G), mont(g_prime()))
    want = np.array([0 if i % 5 == 3 else 1 for i in range(n)], dtype=np.uint8)
    assert np.array_equal(host(got), want) and engine.last_schnorr_double_verified() == int(want.sum())
    assert pb.schnorr_verify_double(mont(pk), mont(pkp), sigs[0][0], mont(sigs[0][1]), mont(sigs[0][2]),
                                    fr_rows([ms[0]])[0], mont(G), mont(g_prime()), engine=engine)


# 4 ---- against the existing calls ------------------------------------------------------------------------------------
def test_sign_equals_existing_calls(engine):
    """R = fixed_base_batch(r, G), R' = fixed_base_batch(r, G'), c = hash_batch_truncated of [R.u, R.v, R'.u, R'.v, m],
    u = (r - c sk) mod r_J"""
    import torch
    rng = np.random.default_rng(810)
    n = 4096
    sks, r, m = random_r(rng, n), random_r(rng, n), random_m(rng, n)
    gm, gpm = mont(G), mont(g_prime())
    u, R, Rp, ok = engine.schnorr_sign_double_batch(to_mem(sks, "device"), to_mem(r, "device"), to_mem(m, "device"), gm, gpm)
    R1, _ = engine.fixed_base_batch(to_mem(r, "device"), gm)
    R2, _ = engine.fixed_base_batch(to_mem(r, "device"), gpm)
    rows = torch.cat([R.reshape(n, 2, 4), Rp.reshape(n, 2, 4), to_mem(m, "device").reshape(n, 1, 4)], dim=1).contiguous()
    c = engine.hash_batch_truncated(pb.Domain.Other, rows)
    torch.cuda.synchronize()
    assert host(ok).all() and torch.equal(R, R1) and torch.equal(Rp, R2)
    cs, ss, rr, us = ints(host(c).reshape(n, 4)), ints(sks), ints(r), ints(u)
    assert all(us[i] == (rr[i] - cs[i] * ss[i]) % N for i in range(n))


def test_note_sign_equals_stealth_and_nullifier_calls(engine):
    """for notes made by stealth_address_batch: the signature verifies under (note_pk, pk'), and
    Hash::digest(Other, [pk'.u, pk'.v, pos]) is nullifier_batch's nullifier of the same (a, b, R_note, pos)"""
    import torch
    rng = np.random.default_rng(811)
    n = 4096
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    gm, gpm = mont(G), mont(g_prime())
    Rn, note_pk, okn = engine.stealth_address_batch(to_mem(random_r(rng, n), "device"), gm,
                                                   to_mem(jo.points_mont([A]), "device"), to_mem(jo.points_mont([B]), "device"))
    al, bl = to_mem(jubjub_limbs([a]), "device"), to_mem(jubjub_limbs([b]), "device")
    m = to_mem(random_m(rng, n), "device")
    u, R, Rp, pkp, ok = engine.note_sign_double_batch(al, bl, Rn, to_mem(random_r(rng, n), "device"), m, gm, gpm)
    ver = engine.schnorr_verify_double_batch(note_pk, pkp, u, R, Rp, m, gm, gpm)
    pos = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    nul, oknul = engine.nullifier_batch(al, bl, gpm, Rn, to_mem(pos, "device"))
    rows = torch.cat([pkp.reshape(n, 2, 4), to_mem(to_mont([int(x) for x in pos]), "device").reshape(n, 1, 4)], dim=1)
    want = engine.hash_batch(pb.Domain.Other, rows.contiguous())
    torch.cuda.synchronize()
    assert host(okn).all() and host(ok).all() and host(oknul).all() and host(ver).all()
    assert engine.last_schnorr_double_verified() == n
    assert torch.equal(nul.reshape(n, 4), want.reshape(n, 4))
    i = int(rng.integers(0, n))
    Ri = jo.points_from_mont(host(Rn)[i:i + 1])[0]
    assert np.array_equal(host(pkp)[i], jo.points_mont([mul(no.note_sk(a, b, Ri), g_prime())])[0])


# 5 ---- 2^18 round trips ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_public", ["one", "n"])
def test_round_trip_2_18(engine, n_public):
    import torch
    rng = np.random.default_rng(820)
    n = 1 << 18
    gm, gpm = mont(G), mont(g_prime())
    sks = random_r(rng, 1 if n_public == "one" else n)
    sk_d = to_mem(sks, "device")
    pk, _ = engine.fixed_base_batch(sk_d, gm)
    pkp, _ = engine.fixed_base_batch(sk_d, gpm)
    m = to_mem(random_m(rng, n), "device")
    u, R, Rp, ok = engine.schnorr_sign_double_batch(sk_d, to_mem(random_r(rng, n), "device"), m, gm, gpm)
    ver = engine.schnorr_verify_double_batch(pk, pkp, u, R, Rp, m, gm, gpm)
    torch.cuda.synchronize()
    assert host(ok).all() and host(ver).all() and engine.last_schnorr_double_verified() == n
    m[7, 0] ^= 1                                                  # one message changed after signing
    ver = engine.schnorr_verify_double_batch(pk, pkp, u, R, Rp, m, gm, gpm)
    torch.cuda.synchronize()
    assert engine.last_schnorr_double_verified() == n - 1 and host(ver)[7] == 0


# 6 ---- invalid items, with canaries around every output, counted once -----------------------------------------------
def _canary(mem, n, shape, byte=False):
    return to_mem(np.full((n + 2,) + shape, 0xA5 if byte else CANARY, dtype=np.uint8 if byte else np.uint64), mem)


def _inner(buf, n):
    h = host(buf)
    canary = 0xA5 if h.dtype == np.uint8 else CANARY
    assert (h[0] == canary).all() and (h[n + 1] == canary).all()
    return h[1:n + 1]


@pytest.mark.parametrize("mem", ["host", "device"])
def test_sign_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(830)
    n = 10
    sks = [jo.random_secret(rng) for _ in range(n)]
    rs = [jo.random_secret(rng) for _ in range(n)]
    ms = [int(x) for x in rng.integers(0, 1 << 62, n)]
    sks[1], rs[2], ms[3] = N, N, P                                 # each alone
    sks[4], rs[4], ms[4] = N + 1, (1 << 256) - 1, P + 7             # all three
    want = expect([model_sign(*x) for x in zip(sks, rs, ms)])
    assert want[-1].sum() == n - 4
    lib, P_ = _native.lib(), engine._ptr
    u, R, Rp, ok = _canary(mem, n, (4,)), _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    sl, rl, ml = to_mem(jubjub_limbs(sks), mem), to_mem(jubjub_limbs(rs), mem), to_mem(fr_rows(ms), mem)
    assert lib.p252_schnorr_sign_double_batch(engine._ctx, P_(sl), n, P_(rl), P_(ml), n, mont(G).ctypes.data,
                                              mont(g_prime()).ctypes.data, P_(u) + 32, P_(R) + 64, P_(Rp) + 64, P_(ok) + 1,
                                              ctypes.byref(cnt), flags) == 0
    for g, w in zip((u, R, Rp, ok), want):
        assert np.array_equal(_inner(g, n), w)
    assert cnt.value == 4
    with pytest.raises(pb.InvalidPoint):
        pb.schnorr_sign_double(N, 1, fr_rows([0])[0], mont(G), mont(g_prime()), engine=engine)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_note_sign_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(831)
    n = 10
    a_s = [jo.random_secret(rng) for _ in range(n)]
    b_s = [jo.random_secret(rng) for _ in range(n)]
    Rs = [mul(jo.random_secret(rng), G) for _ in range(n)]
    rs = [jo.random_secret(rng) for _ in range(n)]
    ms = [int(x) for x in rng.integers(0, 1 << 62, n)]
    a_s[1], b_s[2], rs[3], ms[4] = N, N, N, P
    Rs[5] = (Rs[5][0] + P, Rs[5][1])                              # an R_note coordinate >= p
    Rs[6] = jo.off_curve_point(rng)
    a_s[7], b_s[7], Rs[7], rs[7], ms[7] = N + 5, N + 1, (0, 0), N, P   # everything
    want = expect([model_note(*x) for x in zip(a_s, b_s, Rs, rs, ms)])
    assert want[-1].sum() == n - 7
    lib, P_ = _native.lib(), engine._ptr
    outs = (_canary(mem, n, (4,)), _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)),
            _canary(mem, n, (), True))
    cnt = ctypes.c_size_t(CANARY)
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    ins = [to_mem(jubjub_limbs(a_s), mem), to_mem(jubjub_limbs(b_s), mem), to_mem(jo.points_mont(Rs), mem),
           to_mem(jubjub_limbs(rs), mem), to_mem(fr_rows(ms), mem)]
    assert lib.p252_note_sign_double_batch(engine._ctx, P_(ins[0]), P_(ins[1]), n, P_(ins[2]), P_(ins[3]), P_(ins[4]), n,
                                           mont(G).ctypes.data, mont(g_prime()).ctypes.data, P_(outs[0]) + 32,
                                           P_(outs[1]) + 64, P_(outs[2]) + 64, P_(outs[3]) + 64, P_(outs[4]) + 1,
                                           ctypes.byref(cnt), flags) == 0
    for g, w in zip(outs, want):
        assert np.array_equal(_inner(g, n), w)
    assert cnt.value == 7


@pytest.mark.parametrize("mem", ["host", "device"])
def test_verify_invalid_items_counted_once(engine, mem):
    rng = np.random.default_rng(832)
    n = 10
    sk = jo.random_secret(rng)
    pk, pkp = key_pair(sk)
    cases = []
    for i in range(n):
        u, R, Rp, _ = model_sign(sk, jo.random_secret(rng), i)
        cases.append([pk, pkp, u, R, Rp, i])
    cases[1][2] = N                                               # u >= r_J
    cases[2][5] = P                                               # m >= p
    cases[3][3] = (cases[3][3][0] + P, cases[3][3][1])            # R coordinate >= p
    cases[4][4] = (cases[4][4][0], cases[4][4][1] + P)            # R' coordinate >= p
    cases[5][0] = jo.off_curve_point(rng)                         # PK off the curve
    cases[6][1] = jo.off_curve_point(rng)                         # PK' off the curve
    cases[7][0], cases[7][1], cases[7][2] = jo.off_curve_point(rng), jo.off_curve_point(rng), N + 1   # both sides
    cases[8][2] = (cases[8][2] + 1) % N                           # valid, does not verify
    want = [model_verify(*[tuple(x) if isinstance(x, tuple) else x for x in c]) for c in cases]
    assert want.count(None) == 7 and want.count(1) == 2
    pk_, pkp_, u_, R_, Rp_, m_ = zip(*cases)
    ver = engine.schnorr_verify_double_batch(to_mem(jo.points_mont(pk_), mem), to_mem(jo.points_mont(pkp_), mem),
                                             to_mem(jubjub_limbs(u_), mem), to_mem(jo.points_mont(R_), mem),
                                             to_mem(jo.points_mont(Rp_), mem), to_mem(fr_rows(m_), mem), mont(G),
                                             mont(g_prime()))
    assert np.array_equal(host(ver), np.array([1 if w == 1 else 0 for w in want], dtype=np.uint8))
    assert engine.last_schnorr_double_invalid() == 7 and engine.last_schnorr_double_verified() == 2
    with pytest.raises(pb.InvalidPoint):
        pb.schnorr_verify_double(mont(pk), mont(pkp), N, mont(G), mont(G), fr_rows([0])[0], mont(G), mont(g_prime()),
                                 engine=engine)


# 7 ---- refused calls --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing_and_launch_nothing(engine, mem):
    rng = np.random.default_rng(840)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 4
    gm, gpm = mont(G), mont(g_prime())
    sc = to_mem(jubjub_limbs([3] * n), mem)
    pts = to_mem(jo.points_mont([G] * n), mem)
    m = to_mem(fr_rows([1] * n), mem)
    o4, o24, o24b, o24c = (to_mem(np.full(s, CANARY, dtype=np.uint64), mem) for s in ((n, 4), (n, 2, 4), (n, 2, 4), (n, 2, 4)))
    ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)

    def sign(g, gp, sk=sc, ns=n, nn=n, r=sc, ms=m, outs=(o4, o24, o24b), okb=ok, cnt=None):
        return lib.p252_schnorr_sign_double_batch(ctx, P_(sk) if sk is not None else None, ns, P_(r) if r is not None else None,
                                                  P_(ms), nn, g, gp, *[P_(o) if o is not None else None for o in outs],
                                                  P_(okb), cnt, flags)

    def verify(g, gp, pk=pts, npub=n, nn=n, u=sc, outs=(o24, o24b), cnt=None):
        return lib.p252_schnorr_verify_double_batch(ctx, P_(pk) if pk is not None else None, P_(pts), npub,
                                                    P_(u) if u is not None else None, *[P_(o) for o in outs], P_(m), nn,
                                                    g, gp, P_(ok), cnt, cnt, flags)

    def note(g, gp, a=sc, ns=n, nn=n, Rn=pts, cnt=None):
        return lib.p252_note_sign_double_batch(ctx, P_(a) if a is not None else None, P_(sc), ns,
                                               P_(Rn) if Rn is not None else None, P_(sc), P_(m), nn, g, gp, P_(o4), P_(o24),
                                               P_(o24b), P_(o24c), P_(ok), cnt, flags)

    def unchanged():
        assert all((host(x) == CANARY).all() for x in (o4, o24, o24b, o24c)) and (host(ok) == 0xA5).all()

    before = engine.launch_count
    for bad in [mont(jo.off_curve_point(rng)), mont((G[0] + P, G[1])), mont((G[0], G[1] + P))]:
        c = ctypes.c_size_t(CANARY)
        for nn in (n, 0):
            for g, gp in ((bad, gpm), (gm, bad)):
                assert sign(g.ctypes.data, gp.ctypes.data, ns=1, nn=nn, cnt=ctypes.byref(c)) == 6
                assert verify(g.ctypes.data, gp.ctypes.data, npub=1, nn=nn, cnt=ctypes.byref(c)) == 6
                assert note(g.ctypes.data, gp.ctypes.data, ns=1, nn=nn, cnt=ctypes.byref(c)) == 6
        assert c.value == CANARY
        with pytest.raises(pb.InvalidPoint):
            engine.schnorr_sign_double_batch(sc, sc, m, gm, bad)
    g, gp = gm.ctypes.data, gpm.ctypes.data
    assert sign(None, gp) == -1 and sign(g, None) == -1 and verify(None, gp) == -1 and note(g, None) == -1
    assert sign(g, gp, sk=None) == -1 and sign(g, gp, r=None) == -1 and sign(g, gp, outs=(o4, None, o24b)) == -1
    assert verify(g, gp, pk=None) == -1 and verify(g, gp, u=None) == -1 and note(g, gp, a=None) == -1
    assert note(g, gp, Rn=None) == -1
    assert sign(g, gp, ns=2) == -1 and sign(g, gp, ns=0) == -1 and note(g, gp, ns=3) == -1
    assert verify(g, gp, npub=2) == -1 and verify(g, gp, npub=0) == -1
    if mem == "device":                                           # misaligned DEVICE rows
        mis = P_(sc) + 8
        assert lib.p252_schnorr_sign_double_batch(ctx, mis, 1, P_(sc), P_(m), 1, g, gp, P_(o4), P_(o24), P_(o24b), P_(ok),
                                                  None, flags) == -1
        assert lib.p252_schnorr_sign_double_batch(ctx, P_(sc), 1, P_(sc), P_(m), 1, g, gp, P_(o4), P_(o24) + 8, P_(o24b),
                                                  P_(ok), None, flags) == -1
        assert lib.p252_schnorr_verify_double_batch(ctx, P_(pts), P_(pts) + 8, 1, P_(sc), P_(o24), P_(o24b), P_(m), 1, g, gp,
                                                    P_(ok), None, None, flags) == -1
        assert lib.p252_note_sign_double_batch(ctx, P_(sc), P_(sc), 1, P_(pts), P_(sc), P_(m), 1, g, gp, P_(o4), P_(o24),
                                               P_(o24b), P_(o24c) + 8, P_(ok), None, flags) == -1
    assert engine.launch_count == before
    unchanged()


# 8 ---- plumbing: batch sizes, staging, injected failures, launches per chunk, the table cache ------------------------
@functools.lru_cache(maxsize=None)
def pool(k=8):
    """k items (sk, r, m) and their model signatures"""
    rng = np.random.default_rng(850)
    items = [(jo.random_secret(rng), jo.random_secret(rng), int(rng.integers(0, 1 << 62))) for _ in range(k)]
    return items, expect([model_sign(*x) for x in items])


def test_batch_sizes(engine):
    rng = np.random.default_rng(851)
    items, want = pool()
    sks, rs, ms = zip(*items)
    sl, rl, ml = jubjub_limbs(sks), jubjub_limbs(rs), fr_rows(ms)
    for n in _sizes():
        sel = rng.integers(0, len(items), n)
        got = engine.schnorr_sign_double_batch(to_mem(sl[sel], "device"), to_mem(rl[sel], "device"),
                                               to_mem(ml[sel], "device"), mont(G), mont(g_prime()))
        rows = rng.choice(n, min(n, 32), replace=False)
        for g, w in zip(got, want):
            assert np.array_equal(host(g)[rows], w[sel[rows]])
        pk = to_mem(jo.points_mont([key_pair(s)[0] for s in sks])[sel], "device")
        pkp = to_mem(jo.points_mont([key_pair(s)[1] for s in sks])[sel], "device")
        ver = engine.schnorr_verify_double_batch(pk, pkp, got[0], got[1], got[2], to_mem(ml[sel], "device"), mont(G),
                                                 mont(g_prime()))
        assert host(ver).all() and engine.last_schnorr_double_verified() == n


@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_signing(engine, mem):
    items, want = pool()
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    sks, rs, ms = zip(*items)
    got = engine.schnorr_sign_double_batch(to_mem(jubjub_limbs(sks), mem), to_mem(jubjub_limbs(rs), mem),
                                           to_mem(fr_rows(ms), mem), mont(G), mont(g_prime()))
    assert np.array_equal(host(got[0]), want[0])
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    Rn = jo.points_mont([G] * len(items))
    got = engine.note_sign_double_batch(to_mem(jubjub_limbs(sks[:1]), mem), to_mem(jubjub_limbs(rs[:1]), mem),
                                        to_mem(Rn, mem), to_mem(jubjub_limbs(rs), mem), to_mem(fr_rows(ms), mem), mont(G),
                                        mont(g_prime()))
    assert host(got[-1]).all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(852)
    n = 200000                                                    # several staged chunks
    items, want = pool()
    sks, rs, ms = zip(*items)
    sel = rng.integers(0, len(items), n)
    sl, rl, ml = jubjub_limbs(sks)[sel], jubjub_limbs(rs)[sel], fr_rows(ms)[sel]
    gm, gpm = mont(G), mont(g_prime())
    Rn = jo.points_mont([G])[np.zeros(n, dtype=np.int64)]
    pk = jo.points_mont([key_pair(s)[0] for s in sks])[sel]
    pkp = jo.points_mont([key_pair(s)[1] for s in sks])[sel]
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    calls = {"sign": (lambda: engine.schnorr_sign_double_batch(sl, rl, ml, gm, gpm), 5),
             "note": (lambda: engine.note_sign_double_batch(sl[:1], rl[:1], Rn, rl, ml, gm, gpm), 7),
             "verify": (lambda: engine.schnorr_verify_double_batch(pk, pkp, want[0][sel], want[1][sel], want[2][sel], ml,
                                                                   gm, gpm), 3)}
    for name, (call, per_chunk) in calls.items():
        for fail_at in (1, 2):
            assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
            with pytest.raises(pb.EngineError):
                call()
            if name != "verify":                                  # verification stages public data only: no wipe
                assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
        call()                                                    # both tables built
        before = engine.launch_count
        res = call()                                              # the retry is correct
        launches = engine.launch_count - before
        assert launches % per_chunk == 0 and launches > per_chunk, (name, launches)
        if name == "sign":
            for g, w in zip(res, want):
                assert np.array_equal(g, w[sel])
        elif name == "verify":
            assert res.all() and engine.last_schnorr_double_verified() == n
        else:
            assert res[-1].all()
        if name != "verify":
            assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_two_generator_cache_by_launch_count(engine):
    """repeated double calls build no table; a fixed_base_batch with a third base evicts neither double slot; a double
    call does not evict the single-base slot"""
    items, want = pool()
    sks, rs, ms = zip(*items)
    sl, rl, ml = jubjub_limbs(sks), jubjub_limbs(rs), fr_rows(ms)
    gm, gpm = mont(G), mont(g_prime())
    third = mont(mul(12345, G))

    def double():
        before = engine.launch_count
        got = engine.schnorr_sign_double_batch(sl, rl, ml, gm, gpm)
        assert np.array_equal(got[0], want[0])
        return engine.launch_count - before

    double()                                                      # both double slots filled
    assert double() == 5 and double() == 5                        # no table built: 5 launches in one chunk
    engine.fixed_base_batch(sl, third)                            # the single-base slot takes a third base
    assert double() == 5                                          # neither double slot evicted
    before = engine.launch_count
    engine.fixed_base_batch(sl, third)
    assert engine.launch_count - before == 1                      # the double call did not evict the single-base slot
    engine.fixed_base_batch(sl, gpm)                              # single-base slot: G'
    assert double() == 5
    before = engine.launch_count
    engine.fixed_base_batch(sl, gpm)
    assert engine.launch_count - before == 1


# 9 ---- the C and C++ consumers on the GPU ---------------------------------------------------------------------------
def test_c_schnorr_double_smoke_gpu():
    from test_schnorr_double_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "SCHNORR_DOUBLE_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_schnorr_double_mirror_gpu():
    from test_schnorr_double_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "schnorr double mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
