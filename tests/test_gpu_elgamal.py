"""JubJub ElGamal and the encrypted note sender on the device (p252_elgamal_{encrypt,decrypt}_batch,
p252_note_sender_{encrypt,decrypt}_batch) against the model of elgamal_oracle.py (affine complete addition,
double-and-add), against the existing calls they compose (fixed_base_batch, dhke_batch, note_create_batch,
wallet_scan_batch), and the calls' own plumbing: tampering, invalid items, refused calls, batch sizes, staging wipes,
injected chunk failures, launches per chunk and the table cache."""
import ctypes
import functools

import numpy as np
import pytest

import elgamal_oracle as eo
import jubjub_edges as je
import jubjub_oracle as jo
import nullifier_oracle as nuo
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_gpu_notes import _random_notes, g_prime
from test_gpu_stealth import CANARY, R_EDGES, _sizes, classes, host, mont, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
MEMS = [("host", False), ("device", False), ("device", True)]
SCALARS = [r for r in R_EDGES if r < N] + [N - 2]


@functools.lru_cache(maxsize=None)
def mul(k, pt):
    return jo.mul(k, tuple(pt))


@functools.lru_cache(maxsize=None)
def points():
    """every order class (identity, orders 2, 4 and 8, G, subgroup, full group), the other small-order points and one
    subgroup point of every edge class of jubjub_edges"""
    rng = np.random.default_rng(200)
    out = list(classes()) + [p for p in jo.small_order_points(rng) if p not in classes()]
    return tuple(out + [e.pt for e in je.subgroup_edges()])


def pts(points_, ok=None):
    out = jo.points_mont(list(points_))
    if ok is not None:
        out[np.asarray(ok) == 0] = 0
    return out


def done(engine, async_):
    if async_:
        engine.sync()


@functools.lru_cache(maxsize=None)
def enc_model(PK, M, r):
    """(c1, c2) as the device writes them, with the oracle's mul memoized"""
    if not (0 <= r < N and jo.on_curve(PK) and jo.on_curve(M)):
        return None
    return mul(r, G), jo.add(M, mul(r, PK))


@functools.lru_cache(maxsize=None)
def dec_model(sk, c1, c2):
    if not (0 <= sk < N and jo.on_curve(c1) and jo.on_curve(c2)):
        return None
    return eo.sub(c2, mul(sk, c1))


@functools.lru_cache(maxsize=None)
def wallet(seed):
    rng = np.random.default_rng(seed)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    return a, b, mul(a, G), mul(b, G)


def stealth(r, A, B):
    return mul(r, G), jo.add(mul(so.hash_point(mul(r, A)), G), B)


def enc_rows(encs):
    """[(c1_A, c2_A), (c1_B, c2_B)] per note -> (n, 4, 2, 4); None (an invalid item) -> zeros"""
    flat = [p for e in encs for pair in (e or [((0, 0), (0, 0))] * 2) for p in pair]
    return pts(flat).reshape(len(encs), 4, 2, 4)


# 1 ---- parity against the model: edge scalars x points of every class, broadcasts 1 and n ----------------------------
@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("bcast", ["one", "n"])
def test_encrypt_decrypt_against_model(engine, mem, async_, bcast):
    ps = points()
    items = [(ps[i % len(ps)] if bcast == "n" else ps[4], ps[(3 * i + 1) % len(ps)], r)
             for i, r in enumerate(SCALARS * 3)]
    PK, M, r = zip(*items)
    want = [enc_model(*x) for x in items]
    k = 1 if bcast == "one" else len(items)
    c1, c2, ok = engine.elgamal_encrypt_batch(to_mem(pts(PK[:k]), mem), to_mem(pts(M), mem), to_mem(jubjub_limbs(r), mem),
                                              mont(G), async_=async_)
    done(engine, async_)
    assert host(ok).all() and engine.last_elgamal_invalid() == 0
    assert np.array_equal(host(c1), pts([w[0] for w in want])) and np.array_equal(host(c2), pts([w[1] for w in want]))
    # decryption of edge ciphertexts: any two curve points under edge keys
    dec = [(SCALARS[i % len(SCALARS)] if bcast == "n" else SCALARS[5], ps[i % len(ps)], ps[(5 * i + 2) % len(ps)])
           for i in range(len(items))]
    sk, d1, d2 = zip(*dec)
    ks = 1 if bcast == "one" else len(dec)
    msg, ok = engine.elgamal_decrypt_batch(to_mem(jubjub_limbs(sk[:ks]), mem), to_mem(pts(d1), mem), to_mem(pts(d2), mem),
                                           async_=async_)
    done(engine, async_)
    assert host(ok).all() and engine.last_elgamal_invalid() == 0
    assert np.array_equal(host(msg), pts([dec_model(*x) for x in dec]))
    i = 7
    one = pb.elgamal_encrypt(mont(PK[i]), mont(M[i]), r[i], mont(G), engine=engine)
    assert np.array_equal(one[0], host(c1)[i]) and np.array_equal(one[1], host(c2)[i])
    assert np.array_equal(pb.elgamal_decrypt(sk[i] if bcast == "n" else sk[0], mont(d1[i]), mont(d2[i]), engine=engine),
                          host(msg)[i])


@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("bcast", ["one", "n"])
def test_sender_against_model(engine, mem, async_, bcast):
    ps = points()
    a, b, A, B = wallet(210)
    n = 24
    rs = [SCALARS[i % len(SCALARS)] for i in range(n)]
    notes = [stealth(jo.random_secret(np.random.default_rng(211 + i)), A, B) for i in range(n)]
    SA = [ps[i % len(ps)] if bcast == "n" else ps[5] for i in range(n)]
    SB = [ps[(2 * i + 3) % len(ps)] if bcast == "n" else ps[3] for i in range(n)]
    bl = [(rs[i], SCALARS[(i + 4) % len(SCALARS)]) for i in range(n)]
    want = [[enc_model(notes[i][1], SA[i], bl[i][0]), enc_model(notes[i][1], SB[i], bl[i][1])] for i in range(n)]
    k = 1 if bcast == "one" else n
    enc, ok = engine.note_sender_encrypt_batch(to_mem(pts([x[1] for x in notes]), mem), to_mem(pts(SA[:k]), mem),
                                               to_mem(pts(SB[:k]), mem),
                                               to_mem(jubjub_limbs([x for p in bl for x in p]).reshape(n, 2, 4), mem),
                                               mont(G), async_=async_)
    done(engine, async_)
    assert host(ok).all() and engine.last_elgamal_invalid() == 0
    assert np.array_equal(host(enc), enc_rows(want))
    # the owner recovers every sender; every other note is decrypted under a key that does not own it
    a2, b2, _, _ = wallet(212)
    keys = [(a, b) if i % 3 else (a2, b2) for i in range(n)]
    ka, kb = zip(*keys)
    ks = n if bcast == "n" else 1
    if bcast == "one":
        ka, kb = (a,) * n, (b,) * n
    gotA, gotB, ok = engine.note_sender_decrypt_batch(to_mem(jubjub_limbs(ka[:ks]), mem), to_mem(jubjub_limbs(kb[:ks]), mem),
                                                      to_mem(pts([x[0] for x in notes]), mem),
                                                      to_mem(pts([x[1] for x in notes]), mem), enc, mont(G), async_=async_)
    done(engine, async_)
    owned = np.array([int(ka[i] == a) for i in range(n)], dtype=np.uint8)
    assert np.array_equal(host(ok), owned) and engine.last_sender_failed() == n - owned.sum()
    assert np.array_equal(host(gotA), pts(SA, owned)) and np.array_equal(host(gotB), pts(SB, owned))
    i = 1
    one = pb.note_sender_decrypt(a, b, mont(notes[i][0]), mont(notes[i][1]), host(enc)[i], mont(G), engine=engine)
    assert np.array_equal(one[0], mont(SA[i])) and np.array_equal(one[1], mont(SB[i]))
    with pytest.raises(pb.DecryptionFailed):
        pb.note_sender_decrypt(a2, b2, mont(notes[i][0]), mont(notes[i][1]), host(enc)[i], mont(G), engine=engine)


def test_sender_decrypt_at_note_sk_zero_and_the_wrap(engine):
    """b = r_J - h gives note_sk = 0 (note_pk the identity), b = r_J - h + 1 wraps to note_sk = 1 (note_pk = G)"""
    rng = np.random.default_rng(220)
    a = jo.random_secret(rng)
    R = mul(jo.random_secret(rng), G)
    h = so.hash_point(mul(a, R))
    SA, SB = points()[5], points()[3]
    pks = [jo.IDENTITY, G]
    bs = [N - h, N - h + 1]
    enc, ok = engine.note_sender_encrypt_batch(pts(pks), pts([SA]), pts([SB]), jubjub_limbs([3, 4, 5, 6]).reshape(2, 2, 4),
                                               mont(G))
    assert ok.all()
    A, B, ok = engine.note_sender_decrypt_batch(jubjub_limbs([a, a]), jubjub_limbs(bs), pts([R, R]), pts(pks), enc, mont(G))
    assert ok.all() and np.array_equal(A, pts([SA, SA])) and np.array_equal(B, pts([SB, SB]))
    assert [nuo.note_sk(a, x, R) for x in bs] == [0, 1]


# 2 ---- against the existing calls ------------------------------------------------------------------------------------
def test_encrypt_equals_fixed_base_and_dhke(engine):
    """c1 = fixed_base_batch(r, G); with M = the identity c2 = dhke_batch(r, PK), and with random M c2 - M (in the model)
    is that dhke row; the sender call equals two encrypt calls under note_pk"""
    import torch
    rng = np.random.default_rng(230)
    n = 4096
    gm = mont(G)
    pool = [jo.random_subgroup_point(rng) for _ in range(16)] + list(points())
    PK = [pool[i] for i in rng.integers(0, len(pool), n)]
    M = [pool[i] for i in rng.integers(0, len(pool), n)]
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(n)])
    d = lambda x: to_mem(x, "device")                                         # noqa: E731
    PKd, Md, rd = d(pts(PK)), d(pts(M)), d(r)
    c1, c2, ok = engine.elgamal_encrypt_batch(PKd, Md, rd, gm)
    f, okf = engine.fixed_base_batch(rd, gm)
    s, oks = engine.dhke_batch(rd, PKd)
    i1, i2, oki = engine.elgamal_encrypt_batch(PKd, d(pts([jo.IDENTITY] * n)), rd, gm)
    torch.cuda.synchronize()
    assert host(ok).all() and host(okf).all() and host(oks).all() and host(oki).all()
    assert torch.equal(c1, f) and torch.equal(i1, f) and torch.equal(i2, s)
    hc2, hs = jo.points_from_mont(host(c2)), jo.points_from_mont(host(s))
    for i in rng.choice(n, 32, replace=False):
        assert eo.sub(hc2[i], M[i]) == hs[i]
    # the sender call = two encrypt calls with PK = note_pk (n_public = n)
    rb = jubjub_limbs([jo.random_secret(rng) for _ in range(2 * n)]).reshape(n, 2, 4)
    SA, SB = pool[3], pool[20]
    enc, oke = engine.note_sender_encrypt_batch(PKd, d(pts([SA])), d(pts([SB])), d(rb), gm)
    a1, a2, oka = engine.elgamal_encrypt_batch(PKd, d(pts([SA] * n)), d(np.ascontiguousarray(rb[:, 0])), gm)
    b1, b2, okb = engine.elgamal_encrypt_batch(PKd, d(pts([SB] * n)), d(np.ascontiguousarray(rb[:, 1])), gm)
    torch.cuda.synchronize()
    assert host(oke).all() and host(oka).all() and host(okb).all()
    assert torch.equal(enc, torch.stack([a1, a2, b1, b2], dim=1))


def test_phoenix_flow_at_2_18(engine):
    """note_create_batch -> note_sender_encrypt_batch on its note_pk -> wallet_scan_batch with two keys ->
    note_sender_decrypt_batch with per-note keys gathered by owner: every sender of the two wallets comes back, the notes
    of a third wallet come back ok = 0"""
    import torch
    rng = np.random.default_rng(240)
    n = 1 << 18
    gm, gpm = mont(G), mont(g_prime())
    W = [wallet(s) for s in (241, 242, 243)]
    who = rng.integers(0, 3, n)
    A = to_mem(pts([W[w][2] for w in range(3)])[who], "device")
    B = to_mem(pts([W[w][3] for w in range(3)])[who], "device")
    r, v, bl, nonce = (to_mem(x, "device") for x in _random_notes(rng, n, None, None))
    R, note_pk, C, cipher, ok = engine.note_create_batch(r, v, bl, nonce, gm, gpm, A, B)
    senders = [jo.random_subgroup_point(rng) for _ in range(8)]
    pick = rng.integers(0, 8, (n, 2))
    SA, SB = to_mem(pts(senders)[pick[:, 0]], "device"), to_mem(pts(senders)[pick[:, 1]], "device")
    blind = to_mem(jubjub_limbs([jo.random_secret(rng) for _ in range(64)])[rng.integers(0, 64, 2 * n)].reshape(n, 2, 4),
                   "device")
    enc, oke = engine.note_sender_encrypt_batch(note_pk, SA, SB, blind, gm)
    ka, kb = jubjub_limbs([W[0][0], W[1][0]]), jubjub_limbs([W[0][1], W[1][1]])
    pos = torch.arange(n, dtype=torch.int64, device="cuda")
    owner, _, _, _, _, _ = engine.wallet_scan_batch(to_mem(ka, "device"), to_mem(kb, "device"), R, note_pk, pos, nonce,
                                                    cipher, C, gm, gpm)
    own = host(owner)
    assert np.array_equal(own, np.where(who < 2, who, -1).astype(np.int32))
    key = np.maximum(own, 0)
    gotA, gotB, okd = engine.note_sender_decrypt_batch(to_mem(ka[key], "device"), to_mem(kb[key], "device"), R, note_pk,
                                                       enc, gm)
    torch.cuda.synchronize()
    assert host(ok).all() and host(oke).all()
    mine = (own >= 0).astype(np.uint8)
    assert np.array_equal(host(okd), mine) and engine.last_sender_failed() == n - int(mine.sum())
    hA, hB, hSA, hSB = host(gotA), host(gotB), host(SA), host(SB)
    assert np.array_equal(hA[mine == 1], hSA[mine == 1]) and np.array_equal(hB[mine == 1], hSB[mine == 1])
    assert not hA[mine == 0].any() and not hB[mine == 0].any()


# 3 ---- tampering --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_tampered_sender_fields(engine, mem):
    rng = np.random.default_rng(250)
    a, b, A, B = wallet(251)
    notes = [stealth(jo.random_secret(rng), A, B) for _ in range(2)]
    SA, SB = jo.random_subgroup_point(rng), jo.random_point(rng)
    encs = [eo.sender_encrypt(pk, SA, SB, jo.random_secret(rng), jo.random_secret(rng)) for _, pk in notes]
    e0, e1 = encs
    cases = [(notes[0], e0),                                               # genuine
             (notes[0], [e0[1], e0[0]]),                                   # the pairs swapped: (B, A)
             (notes[0], [(e0[0][1], e0[0][0]), e0[1]]),                    # c1 and c2 swapped
             (notes[0], [e1[0], e0[1]]),                                   # a ciphertext from another note
             ((notes[0][0], notes[1][1]), e0),                             # note_pk of another note
             ((notes[1][0], notes[0][1]), e0)]                             # R of another note
    sk = nuo.note_sk(a, b, notes[0][0])
    want = [eo.sender_decrypt(a, b, R, pk, enc) for (R, pk), enc in cases]
    assert want[0] == (SA, SB) and want[1] == (SB, SA) and want[4] is None and want[5] is None
    assert want[2][0] == eo.sub(e0[0][0], mul(sk, e0[0][1])) != SA and want[3][0] != SA
    n = len(cases)
    A_, B_, ok = engine.note_sender_decrypt_batch(to_mem(jubjub_limbs([a]), mem), to_mem(jubjub_limbs([b]), mem),
                                                  to_mem(pts([c[0][0] for c in cases]), mem),
                                                  to_mem(pts([c[0][1] for c in cases]), mem),
                                                  to_mem(enc_rows([c[1] for c in cases]), mem), mont(G))
    okw = np.array([int(w is not None) for w in want], dtype=np.uint8)
    assert np.array_equal(host(ok), okw) and engine.last_sender_failed() == n - okw.sum()
    assert np.array_equal(host(A_), pts([w[0] if w else (0, 0) for w in want], okw))
    assert np.array_equal(host(B_), pts([w[1] if w else (0, 0) for w in want], okw))


# 4 ---- invalid items, with canaries around every output, counted once -----------------------------------------------
def _canary(mem, n, shape, byte=False):
    return to_mem(np.full((n + 2,) + shape, 0xA5 if byte else CANARY, dtype=np.uint8 if byte else np.uint64), mem)


def _inner(buf, n):
    h = host(buf)
    canary = 0xA5 if h.dtype == np.uint8 else CANARY
    assert (h[0] == canary).all() and (h[n + 1] == canary).all()
    return h[1:n + 1]


@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(260)
    lib, P_, ctx = _native.lib(), engine._ptr, engine._ctx
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    gm = mont(G)
    off, big = jo.off_curve_point(rng), (G[0] + P, G[1])
    n = 8
    pool = [jo.random_subgroup_point(rng) for _ in range(4)]
    # encrypt: r >= r_J, PK off the curve, M with u >= p, everything at once
    PK, M = [pool[i % 4] for i in range(n)], [pool[(i + 1) % 4] for i in range(n)]
    r = [jo.random_secret(rng) for _ in range(n)]
    r[1], PK[2], M[3] = N, off, big
    r[4], PK[4], M[4] = (1 << 256) - 1, big, off
    want = [enc_model(PK[i], M[i], r[i]) if i not in (3, 4) else None for i in range(n)]
    okw = np.array([int(w is not None) for w in want], dtype=np.uint8)
    c1, c2, ok = _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    ins = [to_mem(pts_raw(PK), mem), to_mem(pts_raw(M), mem), to_mem(jubjub_limbs(r), mem)]
    assert lib.p252_elgamal_encrypt_batch(ctx, P_(ins[0]), n, P_(ins[1]), P_(ins[2]), n, gm.ctypes.data, P_(c1) + 64,
                                          P_(c2) + 64, P_(ok) + 1, ctypes.byref(cnt), flags) == 0
    assert np.array_equal(_inner(ok, n), okw) and cnt.value == n - okw.sum() == 4
    assert np.array_equal(_inner(c1, n), pts([w[0] if w else (0, 0) for w in want], okw))
    assert np.array_equal(_inner(c2, n), pts([w[1] if w else (0, 0) for w in want], okw))
    # decrypt: sk >= r_J, c1 off the curve, c2 with v >= p
    sk = [jo.random_secret(rng) for _ in range(n)]
    d1, d2 = list(M), list(PK)
    d1[3], d2[4] = pool[0], pool[1]
    d1[2], d2[2] = pool[2], pool[3]
    sk[5], d1[6], d2[7] = N + 3, off, (G[0], G[1] + P)
    want = [dec_model(sk[i], d1[i], d2[i]) if jo.on_curve(d1[i]) and jo.on_curve(d2[i]) and
            all(0 <= c < P for c in d1[i] + d2[i]) else None for i in range(n)]
    okw = np.array([int(w is not None) for w in want], dtype=np.uint8)
    assert okw.sum() == n - 4                                              # items 4 (c1 off the curve), 5, 6 and 7
    msg, ok = _canary(mem, n, (2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    ins = [to_mem(jubjub_limbs(sk), mem), to_mem(pts_raw(d1), mem), to_mem(pts_raw(d2), mem)]
    assert lib.p252_elgamal_decrypt_batch(ctx, P_(ins[0]), n, P_(ins[1]), P_(ins[2]), n, P_(msg) + 64, P_(ok) + 1,
                                          ctypes.byref(cnt), flags) == 0
    assert np.array_equal(_inner(ok, n), okw) and cnt.value == n - okw.sum()
    assert np.array_equal(_inner(msg, n), pts([w if w else (0, 0) for w in want], okw))
    # sender encrypt: a blinder >= r_J, note_pk, A or B invalid
    a, b, A, B = wallet(261)
    notes = [stealth(jo.random_secret(rng), A, B) for _ in range(n)]
    npk = [x[1] for x in notes]
    SA, SB = [pool[0]] * n, [pool[1]] * n
    bl = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(n)]
    bl[1] = (bl[1][0], N)
    npk[2], SA[3], SB[4] = off, big, off
    npk[5], SA[5], bl[5] = big, off, (N, N + 1)
    good = [i for i in range(n) if i not in (1, 2, 3, 4, 5)]
    want = [eo.sender_encrypt(npk[i], SA[i], SB[i], *bl[i]) if i in good else None for i in range(n)]
    okw = np.array([int(w is not None) for w in want], dtype=np.uint8)
    enc, ok = _canary(mem, n, (4, 2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    ins = [to_mem(pts_raw(npk), mem), to_mem(pts_raw(SA), mem), to_mem(pts_raw(SB), mem),
           to_mem(jubjub_limbs([x for p in bl for x in p]).reshape(n, 2, 4), mem)]
    assert lib.p252_note_sender_encrypt_batch(ctx, P_(ins[0]), P_(ins[1]), P_(ins[2]), n, P_(ins[3]), n, gm.ctypes.data,
                                              P_(enc) + 256, P_(ok) + 1, ctypes.byref(cnt), flags) == 0
    assert np.array_equal(_inner(ok, n), okw) and cnt.value == 5
    assert np.array_equal(_inner(enc, n), enc_rows(want))
    # sender decrypt: a or b >= r_J, R off the curve, a ciphertext point off the curve, note_pk off the curve or >= p,
    # a note of another wallet: each counted once in n_failed
    encs = [eo.sender_encrypt(x[1], pool[0], pool[1], 5, 6) for x in notes]
    Rs, pks = [x[0] for x in notes], [x[1] for x in notes]
    a_s, b_s = [a] * n, [b] * n
    a_s[0] = N
    b_s[1] = N + 7
    Rs[2] = off
    encs[3] = [encs[3][0], (encs[3][1][0], off)]
    pks[4], pks[5] = off, (pks[5][0] + P, pks[5][1])
    a_s[6], b_s[6] = a_s[6] + 1, b_s[6]
    rows = enc_rows(encs)
    A_, B_, ok = _canary(mem, n, (2, 4)), _canary(mem, n, (2, 4)), _canary(mem, n, (), True)
    cnt = ctypes.c_size_t(CANARY)
    ins = [to_mem(jubjub_limbs(a_s), mem), to_mem(jubjub_limbs(b_s), mem), to_mem(pts_raw(Rs), mem),
           to_mem(pts_raw(pks), mem), to_mem(rows, mem)]
    assert lib.p252_note_sender_decrypt_batch(ctx, P_(ins[0]), P_(ins[1]), n, P_(ins[2]), P_(ins[3]), P_(ins[4]), n,
                                              gm.ctypes.data, P_(A_) + 64, P_(B_) + 64, P_(ok) + 1, ctypes.byref(cnt),
                                              flags) == 0
    okw = np.array([0, 0, 0, 0, 0, 0, 0, 1], dtype=np.uint8)
    assert np.array_equal(_inner(ok, n), okw) and cnt.value == n - 1
    assert np.array_equal(_inner(A_, n), pts([pool[0]] * n, okw)) and np.array_equal(_inner(B_, n), pts([pool[1]] * n, okw))
    with pytest.raises(pb.InvalidPoint):
        pb.elgamal_encrypt(gm, gm, N, gm, engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.elgamal_decrypt(N, gm, gm, engine=engine)


def pts_raw(points_):
    """(u, v) rows in Montgomery form, coordinates >= p passed through raw (the device must see them)"""
    from test_gpu_schnorr import fr_rows
    return fr_rows([c for p in points_ for c in p]).reshape(len(points_), 2, 4)


# 5 ---- refused calls ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing_and_launch_nothing(engine, mem):
    rng = np.random.default_rng(270)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 4
    gm = mont(G)
    sc = to_mem(jubjub_limbs([3] * (2 * n)), mem)
    pt = to_mem(pts([G] * n), mem)
    e4 = to_mem(pts([G] * (4 * n)).reshape(n, 4, 2, 4), mem)
    oa, ob, oe = (to_mem(np.full(s, CANARY, dtype=np.uint64), mem) for s in ((n, 2, 4), (n, 2, 4), (n, 4, 2, 4)))
    ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)

    def p(x):
        return P_(x) if x is not None else None

    def enc_(g, nn=n, npub=n, pk=pt, m=pt, r=sc, c1=oa, c2=ob, cnt=None):
        return lib.p252_elgamal_encrypt_batch(ctx, p(pk), npub, p(m), p(r), nn, g, p(c1), p(c2), P_(ok), cnt, flags)

    def dec_(nn=n, ns=n, sk=sc, c1=pt, c2=pt, m=oa, cnt=None):
        return lib.p252_elgamal_decrypt_batch(ctx, p(sk), ns, p(c1), p(c2), nn, p(m), P_(ok), cnt, flags)

    def senc(g, nn=n, ns=n, pk=pt, A=pt, bl=sc, out=oe, cnt=None):
        return lib.p252_note_sender_encrypt_batch(ctx, p(pk), p(A), P_(pt), ns, p(bl), nn, g, p(out), P_(ok), cnt, flags)

    def sdec(g, nn=n, ns=n, a=sc, R=pt, e=e4, A=oa, cnt=None):
        return lib.p252_note_sender_decrypt_batch(ctx, p(a), P_(sc), ns, p(R), P_(pt), p(e), nn, g, p(A), P_(ob), P_(ok),
                                                  cnt, flags)

    def unchanged():
        assert all((host(x) == CANARY).all() for x in (oa, ob, oe)) and (host(ok) == 0xA5).all()

    before = engine.launch_count
    for bad in [mont(jo.off_curve_point(rng)), pts_raw([(G[0] + P, G[1])])[0], pts_raw([(G[0], G[1] + P)])[0]]:
        c = ctypes.c_size_t(CANARY)
        for nn in (n, 0):
            assert enc_(bad.ctypes.data, nn=nn, npub=1, cnt=ctypes.byref(c)) == 6
            assert senc(bad.ctypes.data, nn=nn, ns=1, cnt=ctypes.byref(c)) == 6
            assert sdec(bad.ctypes.data, nn=nn, ns=1, cnt=ctypes.byref(c)) == 6
        assert c.value == CANARY
        with pytest.raises(pb.InvalidPoint):
            engine.elgamal_encrypt_batch(pt, pt, sc[:n], bad)
    g = gm.ctypes.data
    assert enc_(None) == -1 and senc(None) == -1 and sdec(None) == -1
    for kw in ("pk", "m", "r", "c1", "c2"):
        assert enc_(g, **{kw: None}) == -1, kw
    for kw in ("sk", "c1", "c2", "m"):
        assert dec_(**{kw: None}) == -1, kw
    for kw in ("pk", "A", "bl", "out"):
        assert senc(g, **{kw: None}) == -1, kw
    for kw in ("a", "R", "e", "A"):
        assert sdec(g, **{kw: None}) == -1, kw
    for k in (0, 2):
        assert enc_(g, npub=k) == -1 and dec_(ns=k) == -1 and senc(g, ns=k) == -1 and sdec(g, ns=k) == -1
    if mem == "device":                                                    # misaligned DEVICE rows
        assert lib.p252_elgamal_encrypt_batch(ctx, P_(pt), n, P_(pt) + 8, P_(sc), 1, g, P_(oa), P_(ob), P_(ok), None,
                                              flags) == -1
        assert lib.p252_elgamal_decrypt_batch(ctx, P_(sc), 1, P_(pt), P_(pt), 1, P_(oa) + 8, P_(ok), None, flags) == -1
        assert lib.p252_note_sender_encrypt_batch(ctx, P_(pt), P_(pt), P_(pt), 1, P_(sc) + 8, 1, g, P_(oe), P_(ok), None,
                                                  flags) == -1
        assert lib.p252_note_sender_decrypt_batch(ctx, P_(sc), P_(sc), 1, P_(pt), P_(pt), P_(e4) + 8, 1, g, P_(oa), P_(ob),
                                                  P_(ok), None, flags) == -1
    # n == 0 writes and counts nothing
    c = ctypes.c_size_t(CANARY)
    assert enc_(g, nn=0, npub=1, cnt=ctypes.byref(c)) == 0 and c.value == 0
    assert dec_(nn=0, ns=1, cnt=ctypes.byref(c)) == 0 and sdec(g, nn=0, ns=1, cnt=ctypes.byref(c)) == 0 and c.value == 0
    assert engine.launch_count == before
    unchanged()


# 6 ---- plumbing: batch sizes, staging, injected failures, launches per chunk, the table cache ------------------------
def test_batch_sizes_round_trip(engine):
    """encrypt -> decrypt and sender encrypt -> decrypt at every size, 2^18 included; sampled rows against the model"""
    import torch
    rng = np.random.default_rng(280)
    a, b, A, B = wallet(281)
    gm = mont(G)
    sk = jo.random_secret(rng)
    PK = mul(sk, G)
    pool = pts([jo.random_subgroup_point(rng) for _ in range(16)])
    rpool = jubjub_limbs([jo.random_secret(rng) for _ in range(64)])
    notes = [stealth(jo.random_secret(rng), A, B) for _ in range(16)]
    Rn, pkn = pts([x[0] for x in notes]), pts([x[1] for x in notes])
    for n in _sizes():
        d = lambda x: to_mem(np.ascontiguousarray(x), "device")           # noqa: E731
        M = d(pool[rng.integers(0, 16, n)])
        r = d(rpool[rng.integers(0, 64, n)])
        c1, c2, ok = engine.elgamal_encrypt_batch(d(pts([PK])), M, r, gm)
        m, okd = engine.elgamal_decrypt_batch(d(jubjub_limbs([sk])), c1, c2)
        which = rng.integers(0, 16, n)
        enc, oke = engine.note_sender_encrypt_batch(d(pkn[which]), M, M, d(rpool[rng.integers(0, 64, 2 * n)].reshape(n, 2, 4)),
                                                    gm)
        sa, sb, oks = engine.note_sender_decrypt_batch(d(jubjub_limbs([a])), d(jubjub_limbs([b])), d(Rn[which]),
                                                       d(pkn[which]), enc, gm)
        torch.cuda.synchronize()
        assert host(ok).all() and host(okd).all() and host(oke).all() and host(oks).all()
        assert torch.equal(m, M) and torch.equal(sa, M) and torch.equal(sb, M)
        for i in rng.choice(n, min(n, 2), replace=False):
            ri = sum(int(host(r)[i][k]) << (64 * k) for k in range(4))
            w = enc_model(PK, jo.points_from_mont(host(M)[i:i + 1])[0], ri)
            assert np.array_equal(host(c1)[i], mont(w[0])) and np.array_equal(host(c2)[i], mont(w[1]))


@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_every_call(engine, mem):
    rng = np.random.default_rng(290)
    a, b, A, B = wallet(291)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    gm = mont(G)
    notes = [stealth(jo.random_secret(rng), A, B) for _ in range(8)]
    M = to_mem(pts([jo.random_subgroup_point(rng) for _ in range(8)]), mem)
    r = to_mem(jubjub_limbs([jo.random_secret(rng) for _ in range(16)]), mem)
    calls = [lambda: engine.elgamal_encrypt_batch(to_mem(pts([A]), mem), M, r[:8], gm),
             lambda: engine.elgamal_decrypt_batch(to_mem(jubjub_limbs([a]), mem), M, M),
             lambda: engine.note_sender_encrypt_batch(to_mem(pts([x[1] for x in notes]), mem), M, M, r.reshape(8, 2, 4), gm)]
    for call in calls:
        assert host(call()[-1]).all()
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    enc, _ = calls[2]()
    sa, sb, ok = engine.note_sender_decrypt_batch(to_mem(jubjub_limbs([a]), mem), to_mem(jubjub_limbs([b]), mem),
                                                  to_mem(pts([x[0] for x in notes]), mem),
                                                  to_mem(pts([x[1] for x in notes]), mem), enc, gm)
    assert host(ok).all() and np.array_equal(host(sa), host(M))
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(300)
    n = 600000                                                    # several staged chunks for every call
    a, b, A, B = wallet(301)
    gm = mont(G)
    pool = pts([jo.random_subgroup_point(rng) for _ in range(16)])
    notes = [stealth(jo.random_secret(rng), A, B) for _ in range(16)]
    which = rng.integers(0, 16, n)
    Rn, pkn = pts([x[0] for x in notes])[which], pts([x[1] for x in notes])[which]
    M = pool[rng.integers(0, 16, n)]
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(64)])[rng.integers(0, 64, 2 * n)]
    c1, c2, ok = engine.elgamal_encrypt_batch(pts([A]), M, r[:n], gm)
    enc, oke = engine.note_sender_encrypt_batch(pkn, M, M, r.reshape(n, 2, 4), gm)
    assert ok.all() and oke.all()
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    al, bl = jubjub_limbs([a]), jubjub_limbs([b])
    calls = {"encrypt": (lambda: engine.elgamal_encrypt_batch(pts([A]), M, r[:n], gm), 1, (c1, c2)),
             "decrypt": (lambda: engine.elgamal_decrypt_batch(al, c1, c2), 1, (M,)),
             "sender encrypt": (lambda: engine.note_sender_encrypt_batch(pkn, M, M, r.reshape(n, 2, 4), gm), 1, (enc,)),
             "sender decrypt": (lambda: engine.note_sender_decrypt_batch(al, bl, Rn, pkn, enc, gm), 3, (M, M))}
    for name, (call, per_chunk, want) in calls.items():
        for fail_at in (1, 2):
            assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
            with pytest.raises(pb.EngineError):
                call()
            assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
        before = engine.launch_count
        res = call()                                              # the retry is correct
        launches = engine.launch_count - before
        assert launches % per_chunk == 0 and launches > per_chunk, (name, launches)
        assert res[-1].all(), name
        for g, w in zip(res, want):
            assert np.array_equal(g, w), name
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_table_cache_by_launch_count(engine):
    """after note_create_batch with the same G the sender calls build no table, and they evict neither G' nor the
    single-base slot"""
    rng = np.random.default_rng(310)
    a, b, A, B = wallet(311)
    gm, gpm = mont(G), mont(g_prime())
    third = mont(mul(12345, G))
    r, v, bl, nonce = _random_notes(rng, 8, A, B)
    engine.fixed_base_batch(r, third)                                        # the single-base slot: a third base

    def launches(call):
        before = engine.launch_count
        res = call()
        assert res[-1].all()
        return engine.launch_count - before, res

    k, (R, pk, C, cipher, _) = launches(lambda: engine.note_create_batch(r, v, bl, nonce, gm, gpm, pts([A]), pts([B])))
    M = pts([jo.random_subgroup_point(rng) for _ in range(8)])
    k, (enc, _) = launches(lambda: engine.note_sender_encrypt_batch(pk, M, M, jubjub_limbs([3] * 16).reshape(8, 2, 4), gm))
    assert k == 1
    assert launches(lambda: engine.note_sender_decrypt_batch(jubjub_limbs([a]), jubjub_limbs([b]), R, pk, enc, gm))[0] == 3
    assert launches(lambda: engine.elgamal_encrypt_batch(pts([A]), M, r, gm))[0] == 1
    assert launches(lambda: engine.elgamal_decrypt_batch(jubjub_limbs([a]), M, M))[0] == 1
    assert launches(lambda: engine.note_open_batch(jubjub_limbs([a]), R, nonce, cipher, C, gm, gpm))[0] == 3   # G' kept
    assert launches(lambda: engine.fixed_base_batch(r, third))[0] == 1          # the single-base slot is still the third
    # a new G builds its table once, in the first slot
    G2 = mont(mul(7, G))
    assert launches(lambda: engine.elgamal_encrypt_batch(pts([A]), M, r, G2))[0] == 2
    assert launches(lambda: engine.elgamal_encrypt_batch(pts([A]), M, r, G2))[0] == 1


# 7 ---- the C and C++ consumers on the GPU ---------------------------------------------------------------------------
def test_c_elgamal_smoke_gpu():
    from test_elgamal_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "ELGAMAL_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_elgamal_mirror_gpu():
    from test_elgamal_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "elgamal mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
