"""Every JubJub kernel on the field-edge points of jubjub_edges.py: coordinates, Niels components and products at p - 1,
at p's top limb, at all-ones limbs and across the conditional subtraction of a sum or the borrow of a difference, placed
on the kernels' inputs, on fixed-base table entries and on their results; and raw coordinates p, p + 1, 2p - 1, 2p,
2p + 1 and 2^256 - 1 next to their canonical twins at every site that checks them.  Expected values come from
jubjub_oracle.py / stealth_oracle.py (affine complete addition, double-and-add); a placed result must also equal the
constructed point."""
import ctypes
import functools

import numpy as np
import pytest

import jubjub_edges as je
import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs, random_scalars

pytestmark = pytest.mark.gpu

CANARY = 0xA5A5A5A5A5A5A5A5
G = jo.GENERATOR
SECRETS = ([0, 1, 2, 15, 16, je.R_J - 1, 1 << 251, int("f" * 62, 16), int("8" * 62, 16), int("7" * 62, 16)]
           + [je.R_J - (1 << k) for k in (1, 4, 32, 128, 250)])
MEMS = [("host", False), ("device", False)]
MEMS_ASYNC = MEMS + [("device", True)]
INVALID_POINT = 6                                                 # P252_ERR_INVALID_POINT


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


def done(engine, async_):
    if async_:
        engine.sync()


def mont(pt):
    return je.rows([pt])[0]


def dhke(s, pt):
    """jo.dhke with the memoized product"""
    return je.mul(s, pt) if 0 <= s < je.R_J and jo.on_curve(pt) else None


def expect(secrets, points):
    want = [dhke(s, p) for s, p in zip(secrets, points)]
    ok = np.array([w is not None for w in want], dtype=np.uint8)
    rows = je.rows([w if w is not None else (0, 0) for w in want])
    rows[ok == 0] = 0
    return rows, ok


def receiver_rows(n):
    a, A, B = je.receiver()
    return a, je.rows([A] * n), je.rows([B] * n)


# 1 ---- dhke_batch: public keys at every edge class, results placed at every edge class ---------------------------------
@pytest.mark.parametrize("mem,async_", MEMS_ASYNC)
def test_dhke_public_at_edges(engine, mem, async_):
    pts = [e.pt for e in je.all_edges()]
    secs = [SECRETS[i % len(SECRETS)] for i in range(len(pts))]
    want, wok = expect(secs, pts)
    assert wok.all()
    out, ok = engine.dhke_batch(to_mem(jubjub_limbs(secs), mem), to_mem(je.rows(pts), mem), async_=async_)
    done(engine, async_)
    assert np.array_equal(host(ok), wok) and np.array_equal(host(out), want) and engine.last_dhke_invalid() == 0
    # the (1, n) shape: one secret selecting tab[15] in 62 windows against every edge point
    s = int("f" * 62, 16)
    want, _ = expect([s] * len(pts), pts)
    out, ok = engine.dhke_batch(to_mem(jubjub_limbs([s]), mem), to_mem(je.rows(pts), mem), async_=async_)
    done(engine, async_)
    assert host(ok).all() and np.array_equal(host(out), want)


@pytest.mark.parametrize("mem,async_", MEMS_ASYNC)
def test_dhke_results_placed_at_edges(engine, mem, async_):
    pl = je.output_placements()
    secs, pubs, Q = [s for _, s, _ in pl], [p for _, _, p in pl], [e.pt for e, _, _ in pl]
    want, wok = expect(secs, pubs)
    assert np.array_equal(want, je.rows(Q)) and wok.all()
    out, ok = engine.dhke_batch(to_mem(jubjub_limbs(secs), mem), to_mem(je.rows(pubs), mem), async_=async_)
    done(engine, async_)
    assert host(ok).all() and np.array_equal(host(out), want)
    # (1, n): the placements made with s = 3
    idx = [i for i, s in enumerate(secs) if s == 3]
    out, ok = engine.dhke_batch(to_mem(jubjub_limbs([3]), mem), to_mem(je.rows([pubs[i] for i in idx]), mem),
                                async_=async_)
    done(engine, async_)
    assert host(ok).all() and np.array_equal(host(out), want[idx])


@pytest.mark.parametrize("mem", ["host", "device"])
def test_fused_dhke_at_edges_equal_separate_calls(engine, mem):
    rng = np.random.default_rng(1)
    pl = je.output_placements()[::9]
    edge = [e.pt for e in je.edges("sum") + je.edges("kt")][:6]
    secs = [s for _, s, _ in pl] + SECRETS[5:5 + len(edge)]
    pubs = [p for _, _, p in pl] + edge
    shared, _ = expect(secs, pubs)
    n, L = len(secs), 2
    msgs, nonce = random_scalars(rng, (n, L)), random_scalars(rng, n)
    sl, pr = to_mem(jubjub_limbs(secs), mem), to_mem(je.rows(pubs), mem)
    cip, ok = engine.encrypt_batch_dhke(to_mem(msgs, mem), sl, pr, to_mem(nonce, mem))
    assert host(ok).all() and engine.last_dhke_invalid() == 0
    assert np.array_equal(host(cip), engine.encrypt_batch(msgs, shared, nonce))
    msg, ok = engine.decrypt_batch_dhke(cip, sl, pr, to_mem(nonce, mem))
    assert host(ok).all() and np.array_equal(host(msg), msgs) and engine.last_decrypt_failures() == 0
    m2, ok2 = engine.decrypt_batch(host(cip), shared, nonce)
    assert np.array_equal(m2, msgs) and ok2.all()


# 2 ---- fixed_base_batch / encrypt_batch_ephemeral ------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def edge_bases():
    """the first point of every named target of every class"""
    seen, out = set(), []
    for e in je.all_edges():
        if (e.kind, e.name) not in seen:
            seen.add((e.kind, e.name))
            out.append(e)
    return tuple(out)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_fixed_base_bases_at_edges(engine, mem):
    for i, e in enumerate(edge_bases()):
        secs = [SECRETS[i % len(SECRETS)], SECRETS[(i + 7) % len(SECRETS)]]
        want, wok = expect(secs, [e.pt] * 2)
        out, ok = engine.fixed_base_batch(to_mem(jubjub_limbs(secs), mem), mont(e.pt))
        assert np.array_equal(host(ok), wok) and np.array_equal(host(out), want), e.label


@pytest.mark.parametrize("mem", ["host", "device"])
def test_fixed_base_table_entries_at_edges(engine, mem):
    """Entry (w, j) of the table is the edge point; each secret selects it with one of the signs the recoding allows
    there, so the swap and the negation of the third Niels coordinate run on the edge.  encrypt_batch_ephemeral reads
    the same table: its R rows equal the fixed-base result, its ciphers encrypt_batch_dhke's."""
    rng = np.random.default_rng(2)
    _, A, _ = je.receiver()
    for t in je.table_placements():
        secs = [s for _, s in t.secrets]
        want, _ = expect(secs, [t.base] * len(secs))
        sl = to_mem(jubjub_limbs(secs), mem)
        out, ok = engine.fixed_base_batch(sl, mont(t.base))
        assert host(ok).all() and np.array_equal(host(out), want), (t.w, t.j, t.edge.label)
        n = len(secs)
        msgs, nonce = to_mem(random_scalars(rng, (n, 1)), mem), to_mem(random_scalars(rng, n), mem)
        Ar = to_mem(je.rows([A]), mem)
        cip, R, ok = engine.encrypt_batch_ephemeral(msgs, sl, mont(t.base), Ar, nonce)
        c2, ok2 = engine.encrypt_batch_dhke(msgs, sl, Ar, nonce)
        assert host(ok).all() and host(ok2).all() and np.array_equal(host(R), want)
        assert np.array_equal(host(cip), host(c2))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_fixed_base_results_placed_at_edges(engine, mem):
    for e, s, pub in je.output_placements():
        want, _ = expect([s], [pub])
        out, ok = engine.fixed_base_batch(to_mem(jubjub_limbs([s]), mem), mont(pub))
        assert host(ok).all() and np.array_equal(host(out), want) and np.array_equal(want[0], mont(e.pt)), e.label


def test_fixed_base_cache_hit_and_rebuild_at_an_edge_base(engine):
    e = je.edges("u")[[x.name for x in je.edges("u")].index("p-1")]
    secs = SECRETS[:6]
    want, _ = expect(secs, [e.pt] * len(secs))
    s = jubjub_limbs(secs)
    out, _ = engine.fixed_base_batch(s, mont(e.pt))
    before = engine.launch_count
    out2, ok = engine.fixed_base_batch(s, mont(e.pt))              # the cached table
    assert engine.launch_count == before + 1 and np.array_equal(out2, want) and np.array_equal(out, want)
    engine.fixed_base_batch(s, mont(G))
    before = engine.launch_count
    out3, ok = engine.fixed_base_batch(s, mont(e.pt))              # rebuilt
    assert engine.launch_count == before + 2 and np.array_equal(out3, want) and ok.all()


# 3 ---- stealth_address_batch ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", MEMS_ASYNC)
def test_stealth_B_per_item_at_edges_and_note_pk_placed(engine, mem, async_):
    """B at every edge point (the device on_curve and to_niels on it), then B placed so that note_pk is each output
    edge; one r and one A for all items."""
    r = je.STEALTH_R
    hG = je.sender_hG()
    placed = [e.pt for e in je.output_edges()]
    Bs = [e.pt for e in je.all_edges()] + [je.note_pk_placement(q) for q in placed]
    n = len(Bs)
    _, Ar, _ = receiver_rows(n)
    R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs([r] * n), mem), mont(G), to_mem(Ar, mem),
                                             to_mem(je.rows(Bs), mem), async_=async_)
    done(engine, async_)
    assert host(ok).all() and engine.last_stealth_invalid() == 0
    assert np.array_equal(host(R), je.rows([je.mul(r, G)] * n))
    want = je.rows([jo.add(hG, B) for B in Bs])
    assert np.array_equal(host(pk), want)
    assert np.array_equal(host(pk)[n - len(placed):], je.rows(placed))


@functools.lru_cache(maxsize=None)
def R_placed_edges():
    """every top-limb coordinate result and the first result of every class"""
    outs = je.output_edges()
    firsts = [next(e for e in outs if e.kind == k) for k in je.KINDS]
    return tuple(firsts + [e for e in outs if e.name in je.TOP_LIMB_NAMES and e not in firsts])


@pytest.mark.parametrize("mem", ["host", "device"])
def test_stealth_R_placed_at_edges(engine, mem):
    _, A, _ = je.receiver()
    for e in R_placed_edges():
        Gq, Bq, pk_want = je.R_placement(e.pt)
        R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs([je.STEALTH_R]), mem), mont(Gq),
                                                 to_mem(je.rows([A]), mem), to_mem(je.rows([Bq]), mem))
        assert host(ok).all(), e.label
        assert np.array_equal(host(R)[0], mont(e.pt)) and np.array_equal(host(pk)[0], mont(pk_want)), e.label


# 4 ---- stealth_owns_batch -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,async_", MEMS_ASYNC)
def test_scan_note_pk_placed_at_edges_and_near_misses(engine, mem, async_):
    """note_pk = Q through spend_B = Q - [h] G: owned; -Q, Q + (0, -1), swapped coordinates and v +- 1 are not owned
    and not invalid."""
    a, _, _ = je.receiver()
    Rn, _ = je.scan_note()
    al = to_mem(jubjub_limbs([a]), mem)
    for e in je.output_edges():
        notes = [e.pt] + [q for _, q in je.near_misses(e.pt)]
        n = len(notes)
        owned = engine.stealth_owns_batch(al, mont(je.spend_B_placement(e.pt)), mont(G), to_mem(je.rows([Rn] * n), mem),
                                          to_mem(je.rows(notes), mem), async_=async_)
        done(engine, async_)
        assert list(host(owned)) == [1] + [0] * (n - 1), e.label
        assert engine.last_stealth_owned() == 1 and engine.last_stealth_invalid() == 0


@pytest.mark.parametrize("mem", ["host", "device"])
def test_scan_spend_B_at_host_niels_edges(engine, mem):
    """spend_B at the sum / difference / product edges: the host's jubjub_niels adds, subtracts and multiplies at them."""
    a, _, _ = je.receiver()
    Rn, hG = je.scan_note()
    al = to_mem(jubjub_limbs([a]), mem)
    for e in je.edges("sum") + je.edges("diff") + je.edges("uv") + je.edges("kt"):
        pk = jo.add(hG, e.pt)
        notes = [pk, (pk[0], (pk[1] + 1) % je.P)]
        owned = engine.stealth_owns_batch(al, mont(e.pt), mont(G), to_mem(je.rows([Rn] * 2), mem),
                                          to_mem(je.rows(notes), mem))
        assert list(host(owned)) == [1, 0] and engine.last_stealth_invalid() == 0, e.label


# 5 ---- exact-boundary coordinates: only the canonical check tells them from their twins --------------------------------
def interleaved():
    """[twin_0, raw_0, twin_1, raw_1, ...] as raw Montgomery pairs, the twins' points, and valid flags"""
    bs = je.boundaries()
    pairs = [x for b in bs for x in (b.twin, b.raw)]
    valid = np.array([1, 0] * len(bs), dtype=np.uint8)
    return bs, pairs, valid


@pytest.mark.parametrize("mem", ["host", "device"])
def test_boundary_dhke_public(engine, mem):
    bs, pairs, valid = interleaved()
    n = len(pairs)
    secs = [SECRETS[5 + i % 8] for i in range(n)]
    want = je.rows([dhke(secs[i], bs[i // 2].pt) if valid[i] else (0, 0) for i in range(n)])
    want[valid == 0] = 0
    big = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    sl, pr = to_mem(jubjub_limbs(secs), mem), to_mem(je.raw_rows(pairs), mem)
    _, ok = engine.dhke_batch(sl, pr, out=big[1:n + 1])
    big = host(big)
    assert np.array_equal(host(ok), valid) and np.array_equal(big[1:n + 1], want)
    assert (big[0] == CANARY).all() and (big[n + 1] == CANARY).all()
    assert engine.last_dhke_invalid() == int((valid == 0).sum())
    # the fused calls: zeroed rows and exact counts, the twins encrypt with the oracle's shared secret
    rng = np.random.default_rng(3)
    L = 2
    msgs, nonce = random_scalars(rng, (n, L)), random_scalars(rng, n)
    cbig = to_mem(np.full((n + 2, L + 1, 4), CANARY, dtype=np.uint64), mem)
    _, ok = engine.encrypt_batch_dhke(to_mem(msgs, mem), sl, pr, to_mem(nonce, mem), out=cbig[1:n + 1])
    cb = host(cbig)
    assert np.array_equal(host(ok), valid) and engine.last_dhke_invalid() == int((valid == 0).sum())
    assert not cb[1:n + 1][valid == 0].any() and (cb[0] == CANARY).all() and (cb[n + 1] == CANARY).all()
    good = valid == 1
    assert np.array_equal(cb[1:n + 1][good], engine.encrypt_batch(msgs, want, nonce)[good])
    cip = cb[1:n + 1].copy()
    cip[~good] = engine.encrypt_batch(msgs, want, nonce)[~good]       # a well-formed cipher: only the key is invalid
    msg, ok = engine.decrypt_batch_dhke(to_mem(cip, mem), sl, pr, to_mem(nonce, mem))
    assert np.array_equal(host(ok), valid) and engine.last_decrypt_failures() == int((valid == 0).sum())
    assert np.array_equal(host(msg)[good], msgs[good]) and not host(msg)[~good].any()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("which", ["A", "B"])
def test_boundary_stealth_A_and_B(engine, mem, which):
    bs, pairs, valid = interleaved()
    n = len(pairs)
    _, A, B = je.receiver()
    r = je.STEALTH_R
    other = je.rows([B if which == "A" else A] * n)
    edge = je.raw_rows(pairs)
    Ar, Br = (edge, other) if which == "A" else (other, edge)
    bR = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    bP = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    _, _, ok = engine.stealth_address_batch(to_mem(jubjub_limbs([r] * n), mem), mont(G), to_mem(Ar, mem), to_mem(Br, mem),
                                            R_out=bR[1:n + 1], out=bP[1:n + 1])
    assert np.array_equal(host(ok), valid) and engine.last_stealth_invalid() == int((valid == 0).sum())
    bR, bP = host(bR), host(bP)
    for big in (bR, bP):
        assert not big[1:n + 1][valid == 0].any() and (big[0] == CANARY).all() and (big[n + 1] == CANARY).all()
    for i in range(0, n, 2):
        Ai, Bi = (bs[i // 2].pt, B) if which == "A" else (A, bs[i // 2].pt)
        hG = je.mul(je.hash_point(je.mul(r, Ai)), G)
        assert np.array_equal(bR[1 + i], mont(je.mul(r, G))) and np.array_equal(bP[1 + i], mont(jo.add(hG, Bi)))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_boundary_scan_R(engine, mem):
    bs, pairs, valid = interleaved()
    n = len(pairs)
    a, _, B = je.receiver()
    notes = [jo.add(je.mul(je.hash_point(je.mul(a, bs[i // 2].pt)), G), B) for i in range(n)]
    big = to_mem(np.full(n + 2, 0xA5, dtype=np.uint8), mem)
    owned = engine.stealth_owns_batch(to_mem(jubjub_limbs([a]), mem), mont(B), mont(G), to_mem(je.raw_rows(pairs), mem),
                                      to_mem(je.rows(notes), mem), out=big[1:n + 1])
    bigh = host(big)
    assert np.array_equal(host(owned), valid) and bigh[0] == 0xA5 and bigh[n + 1] == 0xA5
    assert engine.last_stealth_owned() == int(valid.sum()) and engine.last_stealth_invalid() == int((valid == 0).sum())


@pytest.mark.parametrize("mem", ["host", "device"])
def test_boundary_scan_note_pk(engine, mem):
    """spend_B placed so that the twin is the note key: the twin is owned, the raw coordinate is invalid"""
    a, _, _ = je.receiver()
    Rn, _ = je.scan_note()
    al = to_mem(jubjub_limbs([a]), mem)
    for b in je.boundaries():
        owned = engine.stealth_owns_batch(al, mont(je.spend_B_placement(b.pt)), mont(G), to_mem(je.rows([Rn] * 2), mem),
                                          to_mem(je.raw_rows([b.twin, b.raw]), mem))
        assert list(host(owned)) == [1, 0], b.name
        assert engine.last_stealth_owned() == 1 and engine.last_stealth_invalid() == 1, b.name


@pytest.mark.parametrize("mem", ["host", "device"])
def test_boundary_host_read_points_refused(engine, mem):
    """base (fixed_base_batch, encrypt_batch_ephemeral, stealth_address_batch, the scan's G) and spend_B are read and
    checked on the host: a raw coordinate is refused with nothing written and no launch, its twin is accepted."""
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    a, A, B = je.receiver()
    Rn, _ = je.scan_note()
    n, L = 3, 1
    rng = np.random.default_rng(4)
    secs = [3, SECRETS[7], SECRETS[11]]
    s, al = to_mem(jubjub_limbs(secs), mem), to_mem(jubjub_limbs([a]), mem)
    msg, non = to_mem(random_scalars(rng, (n, L)), mem), to_mem(random_scalars(rng, n), mem)
    Am, Bm, Rm = to_mem(je.rows([A]), mem), to_mem(je.rows([B]), mem), to_mem(je.rows([Rn] * n), mem)
    gm, bm = mont(G), mont(B)

    def calls(pt):
        """rc of every host-read site with pt there, and the buffers they could write"""
        out = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        out2 = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
        cip = to_mem(np.full((n, L + 1, 4), CANARY, dtype=np.uint64), mem)
        ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)
        c1, c2 = ctypes.c_size_t(CANARY), ctypes.c_size_t(CANARY)
        p = pt.ctypes.data
        rcs = [lib.p252_fixed_base_batch(ctx, p, P_(s), n, P_(out), P_(ok), ctypes.byref(c1), flags),
               lib.p252_encrypt_batch_ephemeral(ctx, P_(msg), n, L, P_(s), p, P_(Am), 1, P_(non), P_(cip), P_(out2),
                                                P_(ok), ctypes.byref(c1), flags),
               lib.p252_stealth_address_batch(ctx, P_(s), n, p, P_(Am), P_(Bm), 1, P_(out), P_(out2), P_(ok),
                                              ctypes.byref(c1), flags),
               lib.p252_stealth_owns_batch(ctx, P_(al), bm.ctypes.data, p, P_(Rm), P_(out), n, P_(ok), ctypes.byref(c1),
                                           ctypes.byref(c2), flags),
               lib.p252_stealth_owns_batch(ctx, P_(al), p, gm.ctypes.data, P_(Rm), P_(out), n, P_(ok), ctypes.byref(c1),
                                           ctypes.byref(c2), flags)]
        engine.sync()
        return rcs, (out, out2, cip, ok), (c1, c2)

    for b in je.boundaries():
        raw, twin = je.raw_rows([b.raw])[0], je.raw_rows([b.twin])[0]
        before = engine.launch_count
        rcs, bufs, cnts = calls(raw)
        assert rcs == [INVALID_POINT] * 5, b.name
        assert engine.launch_count == before and all(c.value == CANARY for c in cnts), b.name
        assert all((host(x) == (0xA5 if host(x).dtype == np.uint8 else CANARY)).all() for x in bufs), b.name
        with pytest.raises(pb.InvalidPoint):
            engine.fixed_base_batch(s, raw)
        rcs, _, _ = calls(twin)
        assert rcs == [0] * 5, b.name
        out, ok = engine.fixed_base_batch(s, twin)
        want, _ = expect(secs, [b.pt] * n)
        assert host(ok).all() and np.array_equal(host(out), want), b.name
