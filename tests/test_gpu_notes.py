"""Note values on the device (p252_value_commit_batch, p252_note_create_batch, p252_note_open_batch) against the model of
note_oracle.py (affine complete addition, double-and-add, the Python Hades), against the existing calls they are built
from (stealth_address_batch, encrypt_batch_ephemeral, fixed_base_batch, jubjub_msm, stealth_owns_batch, dhke_batch +
encrypt_batch), and the calls' own plumbing: invalid items, refused calls, batch sizes, staging wipes, injected chunk
failures, launches per chunk and the two-generator table cache."""
import ctypes
import functools

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import note_oracle as nto
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_gpu_schnorr import fr_rows, ints
from test_gpu_stealth import CANARY, R_EDGES, _sizes, classes, host, mont, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
MEMS = [("host", False), ("device", False), ("device", True)]
V_EDGES = [0, 1, 15, 16, int("7" * 16, 16), int("8" * 16, 16), 1 << 63, (1 << 64) - 1]
B_EDGES = [0, 1, N - 1]


@functools.lru_cache(maxsize=None)
def g_prime():
    """a random point of the prime-order subgroup as G' (GENERATOR_NUMS is not pinned here)"""
    return jo.random_subgroup_point(np.random.default_rng(900))


@functools.lru_cache(maxsize=None)
def mul(k, pt):
    return jo.mul(k, pt)


@functools.lru_cache(maxsize=None)
def commit(v, b, Gp):
    return None if not 0 <= b < N else jo.add(mul(v, G), mul(b, Gp))


@functools.lru_cache(maxsize=None)
def model_create(r, v, b, nonce, A, B, Gp):
    """(R, note_pk, C, cipher, ok) as the device writes them: zeroed rows for an invalid item"""
    if not (0 <= r < N) or not (0 <= b < N) or not jo.on_curve(A) or not jo.on_curve(B):
        return (0, 0), (0, 0), (0, 0), (0, 0, 0), 0
    S = mul(r, A)
    pk = jo.add(mul(so.hash_point(S), G), B)
    return mul(r, G), pk, commit(v, b, Gp), tuple(ho.encrypt([v, b], list(S), nonce)), 1


def model_open(a, R, nonce, cipher, C, Gp):
    """(v, blinder, ok) as the device writes them"""
    if not nto.valid_opening(a, R) or not all(0 <= c < P for c in C):
        return 0, 0, 0
    m = nto.decrypt_rows(a, R, nonce, cipher)
    if m is None or not (0 <= m[0] < 1 << 64 and 0 <= m[1] < N) or commit(m[0], m[1], Gp) != tuple(C):
        return 0, 0, 0
    return m[0], m[1], 1


def pts(points, ok=None):
    out = jo.points_mont(points)
    if ok is not None:
        out[ok == 0] = 0
    return out


def ciphers(rows):
    return fr_rows([x for row in rows for x in row]).reshape(len(rows), 3, 4)


def values(vs):
    return np.array([int(v) for v in vs], dtype=np.uint64)


def done(engine, async_):
    if async_:
        engine.sync()


@functools.lru_cache(maxsize=None)
def wallet(seed):
    rng = np.random.default_rng(seed)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    return (a, b) + so.keys(a, b)


# 1 ---- commitments against the model: edge v x edge blinder, G' = G and a random G' -----------------------------------
@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("gp", ["random", "G"])
def test_commit_against_model(engine, mem, async_, gp):
    Gp = g_prime() if gp == "random" else G
    grid = [(v, b) for v in V_EDGES for b in B_EDGES]
    vs, bs = zip(*grid)
    want = pts([commit(v, b, Gp) for v, b in grid])
    C, ok = engine.value_commit_batch(to_mem(values(vs), mem), to_mem(jubjub_limbs(bs), mem), mont(G), mont(Gp),
                                      async_=async_)
    done(engine, async_)
    assert host(ok).all() and np.array_equal(host(C), want) and engine.last_note_invalid() == 0
    assert np.array_equal(pb.value_commit(vs[4], bs[4], mont(G), mont(Gp), engine=engine), want[4])


# 2 ---- creation against the model: edge v, blinder and r, receivers of every order class -------------------------------
def _create_grid(n_public):
    cls = classes()
    rs = [r for r in R_EDGES if r < N]
    items = []
    for i, (v, b) in enumerate((v, b) for v in V_EDGES for b in B_EDGES):
        A = cls[(i + 4) % len(cls)] if n_public == "n" else cls[5]
        B = cls[(3 * i + 1) % len(cls)] if n_public == "n" else cls[6]
        items.append((rs[i % len(rs)], v, b, 1000 + i, A, B))
    return items


@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("n_public", ["one", "n"])
def test_create_against_model(engine, mem, async_, n_public):
    items = _create_grid(n_public)
    rows = [model_create(*x, g_prime()) for x in items]
    ok = np.array([x[4] for x in rows], dtype=np.uint8)
    assert ok.all()
    r, v, b, nonce, A, B = zip(*items)
    k = 1 if n_public == "one" else len(items)
    got = engine.note_create_batch(to_mem(jubjub_limbs(r), mem), to_mem(values(v), mem), to_mem(jubjub_limbs(b), mem),
                                   to_mem(fr_rows(nonce), mem), mont(G), mont(g_prime()), to_mem(pts(A[:k]), mem),
                                   to_mem(pts(B[:k]), mem), async_=async_)
    done(engine, async_)
    want = (pts([x[0] for x in rows]), pts([x[1] for x in rows]), pts([x[2] for x in rows]), ciphers([x[3] for x in rows]), ok)
    for g, w in zip(got, want):
        assert np.array_equal(host(g), w)
    assert engine.last_note_invalid() == 0
    one = pb.note_create(r[3], v[3], b[3], fr_rows([nonce[3]])[0], mont(G), mont(g_prime()), mont(A[3]), mont(B[3]),
                         engine=engine)
    for g, w in zip(one, want):
        assert np.array_equal(g, w[3])


# 3 ---- opening against the model: genuine notes, every tampering, n_secret 1 and n -------------------------------------
def _open_cases(n_secret):
    """(a, R, nonce, cipher, C) rows: notes of edge values for one or several wallets, and each of them tampered"""
    rng = np.random.default_rng(910)
    Gp = g_prime()
    out, vb = [], [(v, b) for v in V_EDGES for b in B_EDGES]
    for i, (v, b) in enumerate(vb):
        a, _, A, B = wallet(911 if n_secret == "one" else 912 + i % 3)
        r = jo.random_secret(rng)
        R, _, C, cipher, _ = model_create(r, v, b, 7 * i, A, B, Gp)
        out.append((a, R, 7 * i, cipher, C))
    genuine = list(out)
    for k, (a, R, nonce, cipher, C) in enumerate(genuine[:6]):
        a2, R2, _, _, C2 = genuine[k + 1]
        out += [(a, R, nonce, cipher, commit(vb[k][0] + 1, vb[k][1], Gp)),   # C of v + 1
                (a, R, nonce, cipher, C2),                                 # another note's C
                (a, R, nonce, (cipher[0], (cipher[1] + 1) % P, cipher[2]), C),
                (a, R, nonce + 1, cipher, C), (a, R2, nonce, cipher, C)]
        if n_secret == "n":
            out.append(((a + 1) % N, R, nonce, cipher, C))               # another view key
    a, R, nonce, _, C = genuine[1]                                       # (v, blinder) = (0, 1): m0 and m1 swapped
    out.append((a, R, nonce, tuple(ho.encrypt([1, 0], list(mul(a, R)), nonce)), C))
    return out


@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("n_secret", ["one", "n"])
def test_open_against_model(engine, mem, async_, n_secret):
    cases = _open_cases(n_secret)
    want = [model_open(*c, g_prime()) for c in cases]
    n_genuine = len(V_EDGES) * len(B_EDGES)
    assert all(w[2] for w in want[:n_genuine]) and not any(w[2] for w in want[n_genuine:])
    a_all, R, nonce, cipher, C = zip(*cases)
    a = a_all
    if n_secret == "one":
        assert len(set(a)) == 1
        a = a[:1]
    v, b, ok = engine.note_open_batch(to_mem(jubjub_limbs(a), mem), to_mem(pts(R), mem), to_mem(fr_rows(nonce), mem),
                                      to_mem(ciphers(cipher), mem), to_mem(pts(C), mem), mont(G), mont(g_prime()),
                                      async_=async_)
    done(engine, async_)
    assert np.array_equal(host(v), values([w[0] for w in want]))
    assert np.array_equal(host(b), jubjub_limbs([w[1] for w in want]))
    assert np.array_equal(host(ok), np.array([w[2] for w in want], dtype=np.uint8))
    assert engine.last_note_failed() == len(cases) - n_genuine
    i = n_genuine - 1
    v1, b1 = pb.note_open(a[0] if n_secret == "one" else a[i], pts([R[i]])[0], fr_rows([nonce[i]])[0],
                          ciphers([cipher[i]])[0], pts([C[i]])[0], mont(G), mont(g_prime()), engine=engine)
    assert v1 == want[i][0] and np.array_equal(b1, jubjub_limbs([want[i][1]])[0])
    with pytest.raises(pb.DecryptionFailed):
        pb.note_open(a_all[-1], pts([R[-1]])[0], fr_rows([nonce[-1]])[0], ciphers([cipher[-1]])[0], pts([C[-1]])[0], mont(G),
                     mont(g_prime()), engine=engine)


# 4 ---- against the existing calls ------------------------------------------------------------------------------------
def test_create_equals_existing_calls(engine):
    """R and note_pk = stealth_address_batch's, cipher = encrypt_batch_ephemeral's on [v, blinder], C = fixed_base_batch(v,
    G) + fixed_base_batch(blinder, G') and jubjub_msm of those rows; the notes are owned by stealth_owns_batch and open
    under the receiver's a and under no other key"""
    import torch
    rng = np.random.default_rng(920)
    n = 4096
    a, b, A, B = wallet(921)
    gm, gpm = mont(G), mont(g_prime())
    r = to_mem(jubjub_limbs([jo.random_secret(rng) for _ in range(n)]), "device")
    vs = rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2 + (rng.integers(0, 2, n, dtype=np.uint64))
    bl = [jo.random_secret(rng) for _ in range(n)]
    v_d, b_d = to_mem(vs, "device"), to_mem(jubjub_limbs(bl), "device")
    nonce = to_mem(fr_rows([int(x) for x in rng.integers(0, 1 << 62, n)]), "device")
    Ad, Bd = to_mem(pts([A]), "device"), to_mem(pts([B]), "device")
    R, pk, C, cipher, ok = engine.note_create_batch(r, v_d, b_d, nonce, gm, gpm, Ad, Bd)
    R1, pk1, ok1 = engine.stealth_address_batch(r, gm, Ad, Bd)
    msg = to_mem(fr_rows([x for i in range(n) for x in (int(vs[i]), bl[i])]).reshape(n, 2, 4), "device")
    cipher1, R2, ok2 = engine.encrypt_batch_ephemeral(msg, r, gm, Ad, nonce)
    vrows = to_mem(jubjub_limbs([int(x) for x in vs]), "device")
    CV, _ = engine.fixed_base_batch(vrows, gm)
    CB, _ = engine.fixed_base_batch(b_d, gpm)
    C1, okc = engine.value_commit_batch(v_d, b_d, gm, gpm)
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), "device"), pts([B])[0], gm, R, pk)
    v_o, b_o, ok_o = engine.note_open_batch(to_mem(jubjub_limbs([a]), "device"), R, nonce, cipher, C, gm, gpm)
    _, _, ok_x = engine.note_open_batch(to_mem(jubjub_limbs([b]), "device"), R, nonce, cipher, C, gm, gpm)
    torch.cuda.synchronize()
    assert host(ok).all() and host(ok1).all() and host(ok2).all() and host(okc).all() and host(ok_o).all()
    assert torch.equal(R, R1) and torch.equal(pk, pk1) and torch.equal(R, R2) and torch.equal(cipher, cipher1)
    assert torch.equal(C, C1) and host(owned).all() and engine.last_stealth_owned() == n
    assert np.array_equal(host(v_o), vs) and np.array_equal(host(b_o), jubjub_limbs(bl))
    assert not host(ok_x).any() and engine.last_note_failed() == n
    hv, hb, hc = jo.points_from_mont(host(CV)), jo.points_from_mont(host(CB)), jo.points_from_mont(host(C))
    for i in rng.choice(n, 64, replace=False):
        assert jo.add(hv[i], hb[i]) == hc[i]
    for i in rng.choice(n, 4, replace=False):
        sc = to_mem(np.stack([host(vrows)[i], jubjub_limbs([bl[i]])[0]]), "device")
        pt = to_mem(np.stack([pts([G])[0], gpm]), "device")
        assert np.array_equal(host(engine.jubjub_msm(sc, pt)), host(C)[i])


@pytest.mark.parametrize("mem", ["host", "device"])
def test_crafted_out_of_range_plaintexts_do_not_open(engine, mem):
    """openings with m0 >= 2^64 or m1 >= r_J, encrypted with dhke_batch + encrypt_batch under commitments that match them,
    do not open; the in-range opening of the same commitment does"""
    rng = np.random.default_rng(930)
    a, _, A, _ = wallet(931)
    Gp = g_prime()
    crafted = [((1 << 64), 3), (5, N), ((1 << 64) + 9, N + 2), (5, 0), (P - 1, 1)]
    n = len(crafted)
    R = [mul(jo.random_secret(rng), G) for _ in range(n)]
    C = [jo.add(mul(m0, G), mul(m1, Gp)) for m0, m1 in crafted]
    assert C[1] == C[3]                                            # [r_J] G' is the identity
    S, okd = engine.dhke_batch(jubjub_limbs([a]), pts(R))
    msg = fr_rows([x for m in crafted for x in m]).reshape(n, 2, 4)
    nonce = fr_rows(list(range(n)))
    cipher = engine.encrypt_batch(msg, S, nonce)
    assert okd.all()
    v, b, ok = engine.note_open_batch(to_mem(jubjub_limbs([a]), mem), to_mem(pts(R), mem), to_mem(nonce, mem),
                                      to_mem(cipher, mem), to_mem(pts(C), mem), mont(G), mont(Gp))
    assert np.array_equal(host(ok), np.array([0, 0, 0, 1, 0], dtype=np.uint8))
    assert np.array_equal(host(v), values([0, 0, 0, 5, 0])) and not host(b).any()
    assert engine.last_note_failed() == 4


# 5 ---- invalid items, with canaries around every output, counted once -----------------------------------------------
def _canary(mem, n, shape, byte=False):
    return to_mem(np.full((n + 2,) + shape, 0xA5 if byte else CANARY, dtype=np.uint8 if byte else np.uint64), mem)


def _inner(buf, n):
    h = host(buf)
    canary = 0xA5 if h.dtype == np.uint8 else CANARY
    assert (h[0] == canary).all() and (h[n + 1] == canary).all()
    return h[1:n + 1]


@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(940)
    lib, P_ = _native.lib(), engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    gm, gpm = mont(G), mont(g_prime())
    n = 10
    _, _, A, B = wallet(941)
    rs = [jo.random_secret(rng) for _ in range(n)]
    vs = [int(x) for x in rng.integers(0, 1 << 63, n)]
    bs = [jo.random_secret(rng) for _ in range(n)]
    As, Bs = [A] * n, [B] * n
    rs[1], bs[2] = N, N                                             # each alone
    As[3], Bs[4] = jo.off_curve_point(rng), (B[0] + P, B[1])
    rs[5], bs[5], As[5], Bs[5] = (1 << 256) - 1, N + 1, (0, 0), jo.off_curve_point(rng)   # everything
    rows = [model_create(rs[i], vs[i], bs[i], i, As[i], Bs[i], g_prime()) for i in range(n)]
    ok_w = np.array([x[4] for x in rows], dtype=np.uint8)
    assert ok_w.sum() == n - 5
    # commit: only the blinder
    C, ok = _canary(mem, n, (2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    vl, bl = to_mem(values(vs), mem), to_mem(jubjub_limbs(bs), mem)
    assert lib.p252_value_commit_batch(engine._ctx, P_(vl), P_(bl), n, gm.ctypes.data, gpm.ctypes.data, P_(C) + 64,
                                       P_(ok) + 1, ctypes.byref(cnt), flags) == 0
    okc = np.array([int(b < N) for b in bs], dtype=np.uint8)
    assert np.array_equal(_inner(ok, n), okc) and cnt.value == 2
    assert np.array_equal(_inner(C, n), pts([commit(v, b, g_prime()) or (0, 0) for v, b in zip(vs, bs)], okc))
    # create
    outs = (_canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (3, 4)),
            _canary(mem, n, (), True))
    ins = [to_mem(jubjub_limbs(rs), mem), vl, bl, to_mem(fr_rows(list(range(n))), mem), to_mem(pts(As), mem),
           to_mem(pts(Bs), mem)]
    cnt = ctypes.c_size_t(CANARY)
    assert lib.p252_note_create_batch(engine._ctx, P_(ins[0]), P_(ins[1]), P_(ins[2]), P_(ins[3]), n, gm.ctypes.data,
                                      gpm.ctypes.data, P_(ins[4]), P_(ins[5]), n, P_(outs[0]) + 64, P_(outs[1]) + 64,
                                      P_(outs[2]) + 64, P_(outs[3]) + 96, P_(outs[4]) + 1, ctypes.byref(cnt), flags) == 0
    want = (pts([x[0] for x in rows], ok_w), pts([x[1] for x in rows], ok_w), pts([x[2] or (0, 0) for x in rows], ok_w),
            ciphers([x[3] for x in rows]), ok_w)
    for g, w in zip(outs, want):
        assert np.array_equal(_inner(g, n), w)
    assert cnt.value == 5
    # open: a >= r_J, R off the curve, R with a coordinate >= p, and notes that do not open
    good = [i for i in range(n) if ok_w[i]]
    a, _, _, _ = wallet(941)
    a_s = [a] * n
    Rs = [rows[i][0] if ok_w[i] else mul(7, G) for i in range(n)]
    Cs = [rows[i][2] if ok_w[i] else mul(9, G) for i in range(n)]
    cph = ciphers([rows[i][3] for i in range(n)])
    a_s[good[0]], Rs[good[1]] = N, jo.off_curve_point(rng)
    Rs[good[2]] = (Rs[good[2]][0] + P, Rs[good[2]][1])
    vo, bo, oko = _canary(mem, n, ()), _canary(mem, n, (4,)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    ins = [to_mem(jubjub_limbs(a_s), mem), to_mem(pts(Rs), mem), to_mem(fr_rows(list(range(n))), mem), to_mem(cph, mem),
           to_mem(pts(Cs), mem)]
    assert lib.p252_note_open_batch(engine._ctx, P_(ins[0]), n, P_(ins[1]), P_(ins[2]), P_(ins[3]), P_(ins[4]), n,
                                    gm.ctypes.data, gpm.ctypes.data, P_(vo) + 8, P_(bo) + 32, P_(oko) + 1,
                                    ctypes.byref(cnt), flags) == 0
    opened = [i for i in good[3:]]
    want_ok = np.array([int(i in opened) for i in range(n)], dtype=np.uint8)
    assert np.array_equal(_inner(oko, n), want_ok) and cnt.value == n - len(opened)
    assert np.array_equal(_inner(vo, n), values([vs[i] if i in opened else 0 for i in range(n)]))
    assert np.array_equal(_inner(bo, n), jubjub_limbs([bs[i] if i in opened else 0 for i in range(n)]))
    with pytest.raises(pb.InvalidPoint):
        pb.value_commit(1, N, gm, gpm, engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.note_open(N, pts([Rs[good[3]]])[0], fr_rows([good[3]])[0], cph[good[3]], pts([Cs[good[3]]])[0], gm, gpm,
                     engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.note_create(N, 1, 1, fr_rows([0])[0], gm, gpm, mont(A), mont(B), engine=engine)


# 6 ---- refused calls --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing_and_launch_nothing(engine, mem):
    rng = np.random.default_rng(950)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 4
    gm, gpm = mont(G), mont(g_prime())
    sc = to_mem(jubjub_limbs([3] * n), mem)
    vl = to_mem(values([5] * n), mem)
    pt = to_mem(pts([G] * n), mem)
    f3 = to_mem(fr_rows([1] * (3 * n)).reshape(n, 3, 4), mem)
    o24a, o24b, o24c, o34, o4 = (to_mem(np.full(s, CANARY, dtype=np.uint64), mem)
                                 for s in ((n, 2, 4), (n, 2, 4), (n, 2, 4), (n, 3, 4), (n, 4)))
    ov = to_mem(np.full(n, CANARY, dtype=np.uint64), mem)
    ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)

    def p(x):
        return P_(x) if x is not None else None

    def commit_(g, gp, nn=n, v=vl, b=sc, out=o24a, cnt=None):
        return lib.p252_value_commit_batch(ctx, p(v), p(b), nn, g, gp, p(out), P_(ok), cnt, flags)

    def create(g, gp, nn=n, r=sc, v=vl, npub=n, A=pt, outs=(o24a, o24b, o24c, o34), cnt=None):
        return lib.p252_note_create_batch(ctx, p(r), p(v), P_(sc), P_(sc), nn, g, gp, p(A), P_(pt), npub,
                                          *[p(o) for o in outs], P_(ok), cnt, flags)

    def open_(g, gp, nn=n, a=sc, ns=n, R=pt, cipher=f3, v=ov, b=o4, cnt=None):
        return lib.p252_note_open_batch(ctx, p(a), ns, p(R), P_(sc), p(cipher), P_(pt), nn, g, gp, p(v), p(b), P_(ok), cnt,
                                        flags)

    def unchanged():
        assert all((host(x) == CANARY).all() for x in (o24a, o24b, o24c, o34, o4, ov)) and (host(ok) == 0xA5).all()

    before = engine.launch_count
    for bad in [mont(jo.off_curve_point(rng)), mont((G[0] + P, G[1])), mont((G[0], G[1] + P))]:
        c = ctypes.c_size_t(CANARY)
        for nn in (n, 0):
            for g, gp in ((bad, gpm), (gm, bad)):
                assert commit_(g.ctypes.data, gp.ctypes.data, nn=nn, cnt=ctypes.byref(c)) == 6
                assert create(g.ctypes.data, gp.ctypes.data, nn=nn, npub=1, cnt=ctypes.byref(c)) == 6
                assert open_(g.ctypes.data, gp.ctypes.data, nn=nn, ns=1, cnt=ctypes.byref(c)) == 6
        assert c.value == CANARY
        with pytest.raises(pb.InvalidPoint):
            engine.value_commit_batch(vl, sc, gm, bad)
    g, gp = gm.ctypes.data, gpm.ctypes.data
    assert commit_(None, gp) == -1 and create(g, None) == -1 and open_(None, gp) == -1
    assert commit_(g, gp, v=None) == -1 and commit_(g, gp, b=None) == -1 and commit_(g, gp, out=None) == -1
    assert create(g, gp, r=None) == -1 and create(g, gp, v=None) == -1 and create(g, gp, A=None) == -1
    assert create(g, gp, outs=(o24a, o24b, o24c, None)) == -1
    assert open_(g, gp, a=None) == -1 and open_(g, gp, R=None) == -1 and open_(g, gp, cipher=None) == -1
    assert open_(g, gp, v=None) == -1 and open_(g, gp, b=None) == -1
    assert create(g, gp, npub=2) == -1 and create(g, gp, npub=0) == -1
    assert open_(g, gp, ns=3) == -1 and open_(g, gp, ns=0) == -1
    if mem == "device":                                           # misaligned DEVICE rows: value to 8, the rest to 16
        assert lib.p252_value_commit_batch(ctx, P_(vl) + 4, P_(sc), 1, g, gp, P_(o24a), P_(ok), None, flags) == -1
        assert lib.p252_value_commit_batch(ctx, P_(vl), P_(sc) + 8, 1, g, gp, P_(o24a), P_(ok), None, flags) == -1
        assert lib.p252_note_create_batch(ctx, P_(sc), P_(vl), P_(sc), P_(sc), 1, g, gp, P_(pt), P_(pt), 1, P_(o24a),
                                          P_(o24b), P_(o24c) + 8, P_(o34), P_(ok), None, flags) == -1
        assert lib.p252_note_open_batch(ctx, P_(sc), 1, P_(pt), P_(sc), P_(f3), P_(pt), 1, g, gp, P_(ov) + 4, P_(o4),
                                        P_(ok), None, flags) == -1
        assert lib.p252_note_open_batch(ctx, P_(sc), 1, P_(pt), P_(sc), P_(f3) + 8, P_(pt), 1, g, gp, P_(ov), P_(o4),
                                        P_(ok), None, flags) == -1
    assert engine.launch_count == before
    unchanged()


# 7 ---- plumbing: batch sizes, staging, injected failures, launches per chunk, the table cache ------------------------
def _random_notes(rng, n, A, B):
    """device inputs of n notes for (A, B): r, v, blinder, nonce"""
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(min(n, 64))])[rng.integers(0, min(n, 64), n)]
    v = rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2 + rng.integers(0, 2, n, dtype=np.uint64)
    b = jubjub_limbs([jo.random_secret(rng) for _ in range(min(n, 64))])[rng.integers(0, min(n, 64), n)]
    nonce = rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64)
    nonce[:, 3] = 0
    return r, v, b, nonce


def test_batch_sizes_round_trip(engine):
    """create -> open at every size, 2^18 included; sampled rows against the model"""
    rng = np.random.default_rng(960)
    a, _, A, B = wallet(961)
    gm, gpm = mont(G), mont(g_prime())
    ad, Ad, Bd = to_mem(jubjub_limbs([a]), "device"), to_mem(pts([A]), "device"), to_mem(pts([B]), "device")
    for n in _sizes():
        r, v, b, nonce = (to_mem(x, "device") for x in _random_notes(rng, n, A, B))
        R, pk, C, cipher, ok = engine.note_create_batch(r, v, b, nonce, gm, gpm, Ad, Bd)
        vo, bo, oko = engine.note_open_batch(ad, R, nonce, cipher, C, gm, gpm)
        assert host(ok).all() and host(oko).all() and engine.last_note_failed() == 0
        assert np.array_equal(host(vo), host(v)) and np.array_equal(host(bo), host(b))
        for i in rng.choice(n, min(n, 2), replace=False):
            ri, bi = ints(host(r)[i:i + 1])[0], ints(host(b)[i:i + 1])[0]
            mi = ints(host(nonce)[i:i + 1])[0] * pow(ho.R, -1, P) % P
            want = model_create(ri, int(host(v)[i]), bi, mi, A, B, g_prime())
            assert np.array_equal(host(C)[i], pts([want[2]])[0]) and np.array_equal(host(R)[i], pts([want[0]])[0])
            assert np.array_equal(host(cipher)[i], ciphers([want[3]])[0])


@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_every_call(engine, mem):
    rng = np.random.default_rng(970)
    a, _, A, B = wallet(971)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    gm, gpm = mont(G), mont(g_prime())
    r, v, b, nonce = (to_mem(x, mem) for x in _random_notes(rng, 8, A, B))
    C, ok = engine.value_commit_batch(v, b, gm, gpm)
    assert host(ok).all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    R, pk, C, cipher, ok = engine.note_create_batch(r, v, b, nonce, gm, gpm, to_mem(pts([A]), mem), to_mem(pts([B]), mem))
    assert host(ok).all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    vo, bo, ok = engine.note_open_batch(to_mem(jubjub_limbs([a]), mem), R, nonce, cipher, C, gm, gpm)
    assert host(ok).all() and np.array_equal(host(vo), host(v))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(980)
    n = 200000                                                    # several staged chunks
    a, _, A, B = wallet(981)
    gm, gpm = mont(G), mont(g_prime())
    r, v, b, nonce = _random_notes(rng, n, A, B)
    R, pk, C, cipher, ok = engine.note_create_batch(r, v, b, nonce, gm, gpm, pts([A]), pts([B]))
    assert ok.all()
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    al = jubjub_limbs([a])
    v3, b3 = np.tile(v, 3), np.tile(b, (3, 1))                  # a commitment item stages fewer bytes: more items
    calls = {"commit": (lambda: engine.value_commit_batch(v3, b3, gm, gpm), 1),
             "create": (lambda: engine.note_create_batch(r, v, b, nonce, gm, gpm, pts([A]), pts([B])), 8),
             "open": (lambda: engine.note_open_batch(al, R, nonce, cipher, C, gm, gpm), 3)}
    for name, (call, per_chunk) in calls.items():
        for fail_at in (1, 2):
            assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
            with pytest.raises(pb.EngineError):
                call()
            assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
        before = engine.launch_count
        res = call()                                              # the retry is correct
        launches = engine.launch_count - before
        assert launches % per_chunk == 0 and launches > per_chunk, (name, launches)
        assert res[-1].all()
        if name == "commit":
            assert np.array_equal(res[0], np.tile(C, (3, 1, 1)))
        elif name == "create":
            for g, w in zip(res, (R, pk, C, cipher)):
                assert np.array_equal(g, w)
        else:
            assert np.array_equal(res[0], v) and np.array_equal(res[1], b) and engine.last_note_failed() == 0
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_table_cache_by_launch_count(engine):
    """after a double-key call the note calls build no table, and they do not evict the single-base slot"""
    rng = np.random.default_rng(990)
    a, _, A, B = wallet(991)
    gm, gpm = mont(G), mont(g_prime())
    third = mont(mul(12345, G))
    r, v, b, nonce = _random_notes(rng, 8, A, B)
    engine.schnorr_sign_double_batch(r[:1], r, fr_rows([1] * 8), gm, gpm)   # both double slots: G, G'
    engine.fixed_base_batch(r, third)                                        # the single-base slot: a third base

    def launches(call):
        before = engine.launch_count
        res = call()
        assert res[-1].all()
        return engine.launch_count - before

    created = []
    assert launches(lambda: created.append(engine.note_create_batch(r, v, b, nonce, gm, gpm, pts([A]), pts([B])))
                    or created[0]) == 8
    R, pk, C, cipher, ok = created[0]
    assert launches(lambda: engine.value_commit_batch(v, b, gm, gpm)) == 1
    assert launches(lambda: engine.note_open_batch(jubjub_limbs([a]), R, nonce, cipher, C, gm, gpm)) == 3
    assert launches(lambda: engine.fixed_base_batch(r, third)) == 1          # the single-base slot is still the third base


# 8 ---- the C and C++ consumers on the GPU ---------------------------------------------------------------------------
def test_c_notes_smoke_gpu():
    from test_notes_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "NOTES_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_notes_mirror_gpu():
    from test_notes_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "notes mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
