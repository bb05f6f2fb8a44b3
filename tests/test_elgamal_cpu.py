"""JubJub ElGamal and the encrypted note sender without a GPU: the model of elgamal_oracle.py (round trips at edge
scalars and points, the additive homomorphism, wrong keys, the sender round trip for stealth notes, ownership, note_sk = 0
and its wrap, invalid items), a model of each kernel's schedule in extended coordinates that counts its field products
and reproduces the model's results, and the bindings of the four calls -- the header, the library, the ctypes signature
table and the Rust block in elgamal.rs agree, the plain-C program calls exactly the new block, the C and C++ programs
compile with -Wall -Werror, and the calls fail loudly without a GPU.  The same C and C++ programs run on the device in
test_gpu_elgamal.py."""
import ctypes
import os
import re

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
from test_notes_cpu import _compile
from test_stealth_cpu import RUST, ROOT, _blocks, _header

WANT = {"p252_elgamal_encrypt_batch": 12, "p252_elgamal_decrypt_batch": 10, "p252_note_sender_encrypt_batch": 12,
        "p252_note_sender_decrypt_batch": 14}
N, P, G = jo.R_J, jo.P, jo.GENERATOR
EDGE_SCALARS = (0, 1, 2, 15, 16, (1 << 251) + 1, N - 2, N - 1)


def _wallet(rng):
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    return a, b, A, B


def _sender_note(rng, A, B):
    """a stealth note to (A, B): (R, note_pk)"""
    return so.stealth_address(jo.random_secret(rng), A, B)


# ---- the model ------------------------------------------------------------------------------------------------------
def test_round_trips_at_edge_scalars_and_points():
    rng = np.random.default_rng(1)
    points = [jo.IDENTITY, G, jo.random_subgroup_point(rng), jo.random_point(rng)] + list(jo.small_order_points(rng))
    for sk in EDGE_SCALARS:
        PK = jo.mul(sk, G)
        for r in EDGE_SCALARS[::3] + (jo.random_secret(rng),):
            for M in points:
                c1, c2 = eo.encrypt(PK, M, r)
                assert c1 == jo.mul(r, G) and eo.decrypt(sk, c1, c2) == M
    for PK in jo.small_order_points(rng):                          # a small-order key: [r] PK cycles with r mod its order
        for M in points[:3]:
            c1, c2 = eo.encrypt(PK, M, 5)
            assert eo.sub(c2, M) == jo.mul(5, PK) == jo.mul(5 % 8, PK)
    assert eo.encrypt(G, G, 0) == (jo.IDENTITY, G)                # r = 0: (identity, M)
    assert eo.decrypt(0, G, jo.IDENTITY) == jo.IDENTITY           # sk = 0: c2


def test_additive_homomorphism():
    rng = np.random.default_rng(2)
    sk = jo.random_secret(rng)
    PK = jo.mul(sk, G)
    M1, M2 = jo.random_subgroup_point(rng), jo.random_point(rng)
    r1, r2 = jo.random_secret(rng), jo.random_secret(rng)
    (a1, b1), (a2, b2) = eo.encrypt(PK, M1, r1), eo.encrypt(PK, M2, r2)
    c1, c2 = jo.add(a1, a2), jo.add(b1, b2)
    assert (c1, c2) == eo.encrypt(PK, jo.add(M1, M2), (r1 + r2) % N)
    assert eo.decrypt(sk, c1, c2) == jo.add(M1, M2)
    # the same r twice under one key reveals M1 - M2
    (a1, b1), (a2, b2) = eo.encrypt(PK, M1, r1), eo.encrypt(PK, M2, r1)
    assert a1 == a2 and eo.sub(b1, b2) == eo.sub(M1, M2)


def test_a_wrong_key_yields_another_point():
    rng = np.random.default_rng(3)
    sk = jo.random_secret(rng)
    M = jo.random_subgroup_point(rng)
    c1, c2 = eo.encrypt(jo.mul(sk, G), M, jo.random_secret(rng))
    for wrong in (sk + 1, (sk + N // 2) % N, 0, jo.random_secret(rng)):
        got = eo.decrypt(wrong, c1, c2)
        assert got is not None and jo.on_curve(got) and got != M


def test_sender_round_trip_for_stealth_notes():
    rng = np.random.default_rng(4)
    a, b, A, B = _wallet(rng)
    sa, sb, SA, SB = _wallet(rng)                                 # the sender's public key (SA, SB)
    for _ in range(3):
        R, pk = _sender_note(rng, A, B)
        assert jo.mul(nuo.note_sk(a, b, R), G) == pk
        enc = eo.sender_encrypt(pk, SA, SB, jo.random_secret(rng), jo.random_secret(rng))
        assert len(enc) == 2 and all(len(pair) == 2 for pair in enc)
        assert eo.sender_decrypt(a, b, R, pk, enc) == (SA, SB)
        assert eo.decrypt(nuo.note_sk(a, b, R), *enc[0]) == SA


def test_another_wallet_does_not_own_the_note():
    rng = np.random.default_rng(5)
    a, b, A, B = _wallet(rng)
    a2, b2, _, _ = _wallet(rng)
    R, pk = _sender_note(rng, A, B)
    R2, pk2 = _sender_note(rng, A, B)
    enc = eo.sender_encrypt(pk, G, G, 3, 4)
    assert eo.sender_decrypt(a, b, R, pk, enc) == (G, G)
    assert eo.sender_decrypt(a2, b2, R, pk, enc) is None          # another key
    assert eo.sender_decrypt(a, b, R, pk2, enc) is None           # another note's note_pk
    assert eo.sender_decrypt(a, b, R2, pk, enc) is None           # another note's R
    assert eo.sender_decrypt(a, b, R, jo.off_curve_point(rng), enc) is None
    assert eo.sender_decrypt(a, b, R, (pk[0] + P, pk[1]), enc) is None


def test_note_sk_zero_and_its_wrap():
    rng = np.random.default_rng(6)
    a = jo.random_secret(rng)
    R = jo.mul(jo.random_secret(rng), G)
    h = so.hash_point(jo.mul(a, R))
    enc = eo.sender_encrypt(jo.IDENTITY, G, jo.IDENTITY, 9, 10)
    assert nuo.note_sk(a, N - h, R) == 0                           # note_pk = [0] G = the identity: owned
    assert eo.sender_decrypt(a, N - h, R, jo.IDENTITY, enc) == (G, jo.IDENTITY)
    assert nuo.note_sk(a, N - h + 1, R) == 1                       # the sum wraps past r_J
    enc = eo.sender_encrypt(G, jo.IDENTITY, G, 9, 10)
    assert eo.sender_decrypt(a, N - h + 1, R, G, enc) == (jo.IDENTITY, G)
    assert nuo.note_sk(a, N - 1, R) == h - 1


def test_invalid_items_of_the_model():
    rng = np.random.default_rng(7)
    off = jo.off_curve_point(rng)
    big = (G[0] + P, G[1])
    assert eo.encrypt(G, G, N) is None and eo.encrypt(off, G, 1) is None and eo.encrypt(G, big, 1) is None
    assert eo.decrypt(N, G, G) is None and eo.decrypt(1, off, G) is None and eo.decrypt(1, G, big) is None
    assert eo.sender_encrypt(G, G, G, 1, N) is None and eo.sender_encrypt(G, off, G, 1, 1) is None
    a, b, A, B = _wallet(rng)
    R, pk = _sender_note(rng, A, B)
    enc = eo.sender_encrypt(pk, G, G, 1, 2)
    assert eo.sender_decrypt(N, b, R, pk, enc) is None and eo.sender_decrypt(a, N, R, pk, enc) is None
    assert eo.sender_decrypt(a, b, off, pk, enc) is None
    assert eo.sender_decrypt(a, b, R, pk, [enc[0], (enc[1][0], off)]) is None


# ---- a model of the kernels' schedules, counting field products -------------------------------------------------------
class Field:
    """Arithmetic mod p that counts products (montmul / montsqr on the device); additions are free"""

    def __init__(self):
        self.n = 0

    def mul(self, a, b):
        self.n += 1
        return a * b % P

    def inv(self, z):
        """Fermat over the bits of p - 2, left to right: (bits - 1) squarings and (ones - 1) products"""
        e = P - 2
        self.n += e.bit_length() - 1 + bin(e).count("1") - 1
        return pow(z, e, P)


TWO_D = 2 * jo.D % P


def _add(f, p, q, want_t):          # p extended, q cached (Y - X, Y + X, 2d T, 2 Z): 8 products, 7 without T
    X1, Y1, Z1, T1 = p
    A, B = f.mul((Y1 - X1) % P, q[0]), f.mul((Y1 + X1) % P, q[1])
    C, D = f.mul(T1, q[2]), f.mul(Z1, q[3])
    E, F, G_, H = (B - A) % P, (D - C) % P, (D + C) % P, (B + A) % P
    return (f.mul(E, F), f.mul(G_, H), f.mul(F, G_), f.mul(E, H) if want_t else None)


def _madd(f, p, q, want_t):         # q Niels (v - u, v + u, 2d u v): D = 2 Z1 without a product
    X1, Y1, Z1, T1 = p
    A, B, C = f.mul((Y1 - X1) % P, q[0]), f.mul((Y1 + X1) % P, q[1]), f.mul(T1, q[2])
    D = 2 * Z1 % P
    E, F, G_, H = (B - A) % P, (D - C) % P, (D + C) % P, (B + A) % P
    return (f.mul(E, F), f.mul(G_, H), f.mul(F, G_), f.mul(E, H) if want_t else None)


def _dbl(f, p, want_t):             # a = -1: 4 squarings + 4 products, 3 without T
    X1, Y1, Z1, _ = p
    A, B, C = f.mul(X1, X1), f.mul(Y1, Y1), 2 * f.mul(Z1, Z1) % P
    E = (f.mul((X1 + Y1) % P, (X1 + Y1) % P) - A - B) % P
    G_ = (B - A) % P
    F, H = (G_ - C) % P, (-(A + B)) % P
    return (f.mul(E, F), f.mul(G_, H), f.mul(F, G_), f.mul(E, H) if want_t else None)


def _cached(f, p):
    X, Y, Z, T = p
    return ((Y - X) % P, (Y + X) % P, f.mul(T, TWO_D), 2 * Z % P)


def _niels(f, pt):
    u, v = pt
    return ((v - u) % P, (v + u) % P, f.mul(f.mul(u, v), TWO_D))


def _on_curve(f, pt):
    u, v = pt
    uu, vv = f.mul(u, u), f.mul(v, v)
    return (vv - uu) % P == (1 + f.mul(f.mul(uu, vv), jo.D)) % P


IDENT_EXT = (0, 1, 1, 0)


def _var_table(f, pt):
    """var_table: the 16-entry cached table of pt, 2 + 14 x 9 products"""
    u, v = pt
    acc = (u, v, 1, f.mul(u, v))
    pc = _cached(f, acc)
    tab = [(1, 1, 0, 2), pc]
    for _ in range(2, 16):
        acc = _add(f, acc, pc, True)
        tab.append(_cached(f, acc))
    return tab


def _var_walk(f, tab, s, last_t):
    """var_walk: 63 windows of 4 doublings and one addition from the table, most significant first"""
    acc = IDENT_EXT
    for w in range(62, -1, -1):
        for k in range(4):
            acc = _dbl(f, acc, k == 3)
        acc = _add(f, acc, tab[(s >> (4 * w)) & 15], last_t and w == 0)
    return acc


def _fb_walk(f, s, base=G):
    """the fixed-base walk over the affine Niels table of base (built once per base, not counted), signed digits"""
    acc = IDENT_EXT
    digits = je.recode(s)
    for w, e in enumerate(digits):
        q = jo.mul(abs(e) << (4 * w), base)
        if e < 0:
            q = jo.neg(q)
        ni = ((q[1] - q[0]) % P, (q[1] + q[0]) % P, TWO_D * q[0] * q[1] % P)
        acc = _madd(f, acc, ni, w < len(digits) - 1)
    return acc


def _batch_affine(f, pts):
    pre = [pts[0][2]]
    for p in pts[1:]:
        pre.append(f.mul(pre[-1], p[2]))
    inv = f.inv(pre[-1])
    out = [None] * len(pts)
    for k in range(len(pts) - 1, -1, -1):
        if k:
            zi, inv = f.mul(inv, pre[k - 1]), f.mul(inv, pts[k][2])
        else:
            zi = inv
        out[k] = (f.mul(pts[k][0], zi), f.mul(pts[k][1], zi))
    return out


def model_enc(PK, msgs, rs):
    """k_elgamal_enc<len(msgs)>: PK's table once, per pair [r] PK + M and [r] G, one shared inversion"""
    f = Field()
    for pt in [PK] + list(msgs):
        _on_curve(f, pt)
    tab = _var_table(f, PK)
    out = []
    for M, r in zip(msgs, rs):
        c2 = _madd(f, _var_walk(f, tab, r, True), _niels(f, M), False)
        out += [_fb_walk(f, r), c2]
    res = _batch_affine(f, out)
    return [(res[2 * j], res[2 * j + 1]) for j in range(len(msgs))], f.n


def model_dec(sk, pairs, note_pk=None):
    """k_elgamal_dec: per pair c2 + [sk] (-c1), one shared inversion; the note form adds the ownership walk"""
    f = Field()
    for c1, c2 in pairs:
        _on_curve(f, c1)
        _on_curve(f, c2)
    owned = True
    out = []
    for c1, c2 in pairs:
        walk = _var_walk(f, _var_table(f, (-c1[0] % P, c1[1])), sk, True)
        out.append(_madd(f, walk, _niels(f, c2), False))
    if note_pk is not None:
        X, Y, Z, _ = _fb_walk(f, sk)
        owned = f.mul(note_pk[0], Z) == X and f.mul(note_pk[1], Z) == Y
    return _batch_affine(f, out), owned, f.n


def test_schedules_reproduce_the_model_with_the_pinned_product_counts():
    rng = np.random.default_rng(8)
    sk = jo.random_secret(rng)
    PK = jo.mul(sk, G)
    M1, M2 = jo.random_subgroup_point(rng), jo.small_order_points(rng)[3]
    r1, r2 = N - 1, jo.random_secret(rng)
    got, n = model_enc(PK, [M1], [r1])
    assert got == [eo.encrypt(PK, M1, r1)] and n == 3284
    got, n = model_enc(PK, [M1, M2], [r1, r2])
    assert got == [eo.encrypt(PK, M1, r1), eo.encrypt(PK, M2, r2)] and n == 6022
    c = eo.encrypt(PK, M1, r1)
    got, _, n = model_dec(sk, [c])
    assert got == [M1] and n == 2832
    a, b, A, B = _wallet(rng)
    R, pk = _sender_note(rng, A, B)
    enc = eo.sender_encrypt(pk, M1, M2, r1, r2)
    note_sk = nuo.note_sk(a, b, R)
    got, owned, n = model_dec(note_sk, enc, pk)
    assert owned and tuple(got) == eo.sender_decrypt(a, b, R, pk, enc) and n == 5699
    assert not model_dec((note_sk + 1) % N, enc, pk)[1]


def test_product_counts_are_pinned_in_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    for pin in ("kProductsPerElGamalEnc == 3284", "kProductsPerSenderEnc == 6022", "kProductsPerElGamalDec == 2832",
                "kProductsPerSenderDec == 5699", "kProductsPerDhke == 2819", "kProductsPerFixedBase == 866"):
        assert pin in src, pin
    # the chains the calls replace: fixed base + dhke per pair, dhke per decryption
    assert 866 + 2819 > 3284 and 2 * (866 + 2819) > 6022 and 2832 - 2819 == 13


# ---- bindings ------------------------------------------------------------------------------------------------------
def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "elgamal_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "elgamal_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "elgamal_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "elgamal_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "elgamal.rs")) == [WANT]             # one block, exactly the four functions
    assert "mod elgamal;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)


def test_existing_rust_modules_keep_their_blocks():
    assert [set(b) for b in _blocks(os.path.join(RUST, "notes.rs"))] == [
        {"p252_value_commit_batch", "p252_note_create_batch", "p252_note_open_batch"}]
    assert _blocks(os.path.join(RUST, "nullifier.rs")) == [{"p252_nullifier_batch": 12}]


def test_c_smoke_calls_exactly_the_elgamal_block():
    block = _blocks(os.path.join(RUST, "elgamal.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "elgamal_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("elgamal_encrypt", "elgamal_encrypt_batch", "elgamal_decrypt", "elgamal_decrypt_batch",
                 "note_sender_encrypt_batch", "note_sender_decrypt", "note_sender_decrypt_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("elgamal_encrypt_batch", "elgamal_decrypt_batch", "note_sender_encrypt_batch", "note_sender_decrypt_batch",
                 "last_elgamal_invalid", "last_sender_failed"):
        assert callable(getattr(pb.Engine, name))


def test_c_elgamal_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "ELGAMAL_SMOKE_NO_DEVICE" in res.stdout or "ELGAMAL_SMOKE_OK" in res.stdout


def test_cpp_elgamal_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "elgamal mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([G])[0]
    with pytest.raises(pb.EngineError):
        pb.elgamal_encrypt(g, g, 3, g)
    with pytest.raises(pb.EngineError):
        pb.elgamal_decrypt(3, g, g)
    with pytest.raises(pb.EngineError):
        pb.note_sender_decrypt_batch(jubjub_limbs([3]), jubjub_limbs([4]), g[None], g[None], np.zeros((1, 4, 2, 4), np.uint64),
                                     g)
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "ELGAMAL_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
