"""Point compression on the device (p252_points_from_bytes / p252_points_to_bytes) against the model of points_oracle.py
(Tonelli-Shanks on big integers), for HOST and DEVICE buffers: the edges of the encoding, random strings, invalid points,
round trips both ways, batch arguments, asynchronous counts, canary rows, and the composition with the stealth-address
scan and Schnorr verification, all on the device."""
import ctypes
import functools

import numpy as np
import pytest

import jubjub_oracle as jo
import points_oracle as po
import poseidon252_b200 as pb
import schnorr_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs

pytestmark = pytest.mark.gpu

CANARY = 0xA5A5A5A5A5A5A5A5
P = jo.P
G = jo.GENERATOR
MEMS = ["host", "device"]


def enc(v, s=0):
    return (v | s << 255).to_bytes(32, "little")


def to_mem(a, mem):
    if mem == "host":
        return a
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a if a.dtype == np.uint8 else a.view(np.int64)).cuda()


def bytes_mem(rows, mem):
    """(n, 32) uint8 -> host as is, device as an (n, 4) 64-bit tensor of the same bytes"""
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    return rows if mem == "host" else to_mem(rows.view(np.uint64).reshape(-1, 4), mem)


def host(x):
    if isinstance(x, np.ndarray):
        return x
    a = x.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def host_bytes(x):
    return np.ascontiguousarray(host(x)).view(np.uint8).reshape(-1, 32)


@functools.lru_cache(maxsize=None)
def decoded(b):
    return po.decode(b)


def expect_from(encodings):
    """(points (n, 2, 4) as the device writes them, ok (n,))"""
    pts = [decoded(bytes(b)) for b in encodings]
    ok = np.array([p is not None for p in pts], dtype=np.uint8)
    return jo.points_mont([p if p is not None else (0, 0) for p in pts]), ok


def expect_to(points):
    """(bytes (n, 32), ok (n,)) for points of ints (a coordinate may be >= p)"""
    encs = [po.encode(p) for p in points]
    ok = np.array([e is not None for e in encs], dtype=np.uint8)
    return po.bytes_rows([e if e is not None else po.FF for e in encs]), ok


@functools.lru_cache(maxsize=None)
def edge_encodings():
    rng = np.random.default_rng(1)
    pts = [jo.random_point(rng) for _ in range(12)] + [jo.random_subgroup_point(rng) for _ in range(3)] + \
        jo.small_order_points(rng) + [G, jo.neg(G)]
    encs = [po.encode(p) for p in pts]
    ns = next(v for v in range(2, 100) if po.decode(enc(v)) is None)
    encs += [enc(0), enc(0, 1),                             # v = 0, both signs: the order-4 points
             enc(1), enc(1, 1), enc(P - 1), enc(P - 1, 1),  # u = 0 with the sign bit clear and set: accepted
             enc(P), enc(P, 1), po.FF, enc((1 << 255) - 1),  # v >= p: rejected
             enc(ns), enc(ns, 1)]                            # u^2 a non-square: rejected
    return tuple(encs)


# 1 ---- from_bytes against the model -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_from_bytes_edges_against_model(engine, mem):
    encs = edge_encodings()
    want, wok = expect_from(encs)
    assert wok.sum() == len(encs) - 6
    pts, ok = engine.points_from_bytes(bytes_mem(po.bytes_rows(list(encs)), mem))
    assert np.array_equal(host(ok), wok) and np.array_equal(host(pts), want)
    assert engine.last_points_invalid() == 6
    assert jo.points_from_mont(host(pts)[-12:-10]) == [(jo.SQRT_M1 if jo.SQRT_M1 & 1 == 0 else P - jo.SQRT_M1, 0),
                                                       (jo.SQRT_M1 if jo.SQRT_M1 & 1 else P - jo.SQRT_M1, 0)]
    assert jo.points_from_mont(host(pts)[-10:-6]) == [(0, 1), (0, 1), (0, P - 1), (0, P - 1)]


@pytest.mark.parametrize("mem", MEMS)
def test_from_bytes_random_strings(engine, mem):
    rng = np.random.default_rng(2)
    rows = rng.integers(0, 256, (10000, 32), dtype=np.uint8)
    want, wok = expect_from(rows)
    assert 4000 < int(wok.sum()) < 6000                       # about half of all strings decode
    pts, ok = engine.points_from_bytes(bytes_mem(rows, mem))
    assert np.array_equal(host(ok), wok) and np.array_equal(host(pts), want)
    assert engine.last_points_invalid() == int((wok == 0).sum())


# 2 ---- to_bytes against the model, invalid rows included --------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_to_bytes_against_model(engine, mem):
    rng = np.random.default_rng(3)
    pts = [jo.random_point(rng) for _ in range(10)] + jo.small_order_points(rng) + [G]
    pts += [(G[0] + P, G[1]), (G[0], G[1] + P), ((1 << 256) - 1, 1), jo.off_curve_point(rng), (0, 0), (G[1], G[0])]
    want, wok = expect_to(pts)
    assert int((wok == 0).sum()) == 6
    b, ok = engine.points_to_bytes(to_mem(jo.points_mont(pts), mem))
    assert np.array_equal(host(ok), wok) and np.array_equal(host_bytes(b), want)
    assert engine.last_points_invalid() == 6
    assert (host_bytes(b)[wok == 0] == 0xff).all()


# 3 ---- round trips on the device ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", MEMS)
def test_round_trips(engine, mem):
    rng = np.random.default_rng(4)
    base = [jo.random_point(rng) for _ in range(16)] + jo.small_order_points(rng) + [G]
    n = 5000
    idx = rng.integers(0, len(base), n)
    pts = jo.points_mont(base)[idx]
    b, ok = engine.points_to_bytes(to_mem(pts, mem))
    assert host(ok).all() and engine.last_points_invalid() == 0
    back, ok2 = engine.points_from_bytes(b)
    assert host(ok2).all() and np.array_equal(host(back), pts)
    # bytes -> points -> bytes on random strings: every decodable string encodes back to itself
    rows = rng.integers(0, 256, (3000, 32), dtype=np.uint8)
    pts2, ok3 = engine.points_from_bytes(bytes_mem(rows, mem))
    good = host(ok3).astype(bool)
    b2, ok4 = engine.points_to_bytes(pts2)
    assert np.array_equal(host(ok4), host(ok3))
    b2h = host_bytes(b2)
    ident = rows[good].copy()
    u0 = np.all(host(pts2)[good][:, 0] == 0, axis=1)           # u = 0: a set sign bit does not survive
    ident[u0, 31] &= 0x7f
    assert np.array_equal(b2h[good], ident) and (b2h[~good] == 0xff).all()


def test_single_item_front_ends(engine):
    g = jo.points_mont([G])[0]
    b = pb.point_to_bytes(g, engine=engine)
    assert b == po.encode(G)
    assert np.array_equal(pb.point_from_bytes(b, engine=engine), g)
    with pytest.raises(pb.InvalidPoint):
        pb.point_from_bytes(po.FF, engine=engine)
    with pytest.raises(pb.InvalidPoint):
        pb.point_to_bytes(jo.points_mont([(G[1], G[0])])[0], engine=engine)
    pts, ok = pb.points_from_bytes_batch(po.bytes_rows([b, po.FF]), engine=engine)
    assert list(ok) == [1, 0]
    out, ok = pb.points_to_bytes_batch(pts, engine=engine)
    assert list(ok) == [1, 0] and out[0].tobytes() == b


# 4 ---- HOST and DEVICE plumbing -------------------------------------------------------------------------------------------
def test_host_batch_of_several_chunks(engine):
    rng = np.random.default_rng(5)
    encs = edge_encodings()
    want, wok = expect_from(encs)
    n = 300000                                                   # more than one 2^17-item staging chunk
    idx = rng.integers(0, len(encs), n)
    rows = po.bytes_rows(list(encs))[idx]
    before = engine.launch_count
    pts, ok = engine.points_from_bytes(rows)
    assert engine.launch_count - before > 1
    assert np.array_equal(ok, wok[idx]) and np.array_equal(pts, want[idx])
    assert engine.last_points_invalid() == int((wok[idx] == 0).sum())
    b, ok2 = engine.points_to_bytes(pts)
    assert np.array_equal(ok2, wok[idx]) and engine.last_points_invalid() == int((wok[idx] == 0).sum())
    wb = rows.copy()
    wb[wok[idx] == 0] = 0xff
    wb[(wok[idx] == 1) & np.all(pts[:, 0] == 0, axis=1), 31] &= 0x7f
    assert np.array_equal(b, wb)


@pytest.mark.parametrize("mem", MEMS)
def test_empty_batch(engine, mem):
    lib, ctx = _native.lib(), engine._ctx
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    c = ctypes.c_size_t(CANARY)
    before = engine.launch_count
    assert lib.p252_points_from_bytes(ctx, None, 0, None, None, ctypes.byref(c), flags) == 0 and c.value == 0
    c.value = CANARY
    assert lib.p252_points_to_bytes(ctx, None, 0, None, None, ctypes.byref(c), flags) == 0 and c.value == 0
    assert engine.launch_count == before
    pts, ok = engine.points_from_bytes(bytes_mem(np.zeros((0, 32), np.uint8), mem))
    assert tuple(pts.shape) == (0, 2, 4) and tuple(ok.shape) == (0,)


@pytest.mark.parametrize("mem", MEMS)
def test_batch_argument_errors(engine, mem):
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 4
    rows = po.bytes_rows([po.encode(G)] * n)
    b = bytes_mem(rows, mem)
    pts = to_mem(np.full((n, 2, 4), CANARY, dtype=np.uint64), mem)
    out = bytes_mem(np.full((n, 32), 0xA5, dtype=np.uint8), mem)
    ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)
    c = ctypes.c_size_t(CANARY)
    before = engine.launch_count
    for args in ((None, n, P_(pts), P_(ok)), (P_(b), n, None, P_(ok)), (P_(b), n, P_(pts), None)):
        assert lib.p252_points_from_bytes(ctx, *args, ctypes.byref(c), flags) == -1
    for args in ((None, n, P_(out), P_(ok)), (P_(pts), n, None, P_(ok)), (P_(pts), n, P_(out), None)):
        assert lib.p252_points_to_bytes(ctx, *args, ctypes.byref(c), flags) == -1
    if mem == "device":
        assert lib.p252_points_from_bytes(ctx, P_(b) + 8, 1, P_(pts), P_(ok), ctypes.byref(c), flags) == -1
        assert lib.p252_points_from_bytes(ctx, P_(b), 1, P_(pts) + 8, P_(ok), ctypes.byref(c), flags) == -1
        assert lib.p252_points_to_bytes(ctx, P_(pts) + 8, 1, P_(out), P_(ok), ctypes.byref(c), flags) == -1
        assert lib.p252_points_to_bytes(ctx, P_(pts), 1, P_(out) + 8, P_(ok), ctypes.byref(c), flags) == -1
        # ok needs no alignment
        assert lib.p252_points_from_bytes(ctx, P_(b), 1, P_(pts), P_(ok) + 1, None, flags) == 0
        before += 1
    assert engine.launch_count == before and c.value == CANARY
    assert (host(ok)[[0, 2, 3]] == 0xA5).all() and (host(out).view(np.uint8) == 0xA5).all()
    assert (host(pts)[1:] == CANARY).all()
    with pytest.raises(pb.EngineError):
        engine.points_from_bytes(np.zeros((2, 31), np.uint8))
    with pytest.raises(pb.EngineError):
        engine.points_to_bytes(to_mem(np.zeros((2, 4), np.uint64), mem))


@pytest.mark.parametrize("direction", ["from", "to"])
def test_async_counts_after_sync(engine, direction):
    rng = np.random.default_rng(6)
    rows = rng.integers(0, 256, (4000, 32), dtype=np.uint8)
    want, wok = expect_from(rows)
    if direction == "from":
        pts, ok = engine.points_from_bytes(bytes_mem(rows, "device"), async_=True)
    else:
        pts = to_mem(want, "device")                           # invalid rows are (0, 0): off the curve
        b, ok = engine.points_to_bytes(pts, async_=True)
    engine.sync()
    assert engine.last_points_invalid() == int((wok == 0).sum())
    assert np.array_equal(host(ok), wok)


@pytest.mark.parametrize("mem", MEMS)
def test_guard_rows_around_every_buffer(engine, mem):
    rng = np.random.default_rng(7)
    encs = list(edge_encodings())
    n = len(encs)
    want, wok = expect_from(encs)
    bp = to_mem(np.full((n + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    pts, ok = engine.points_from_bytes(bytes_mem(po.bytes_rows(encs), mem), out=bp[1:n + 1])
    bph = host(bp)
    assert np.array_equal(bph[1:n + 1], want) and (bph[0] == CANARY).all() and (bph[n + 1] == CANARY).all()
    assert np.array_equal(host(ok), wok)
    # raw calls with guard rows around the output and ok buffers of both directions
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    src_pts = [jo.random_point(rng) for _ in range(5)] + [jo.off_curve_point(rng), (G[0] + P, G[1])]
    m = len(src_pts)
    wb, wok2 = expect_to(src_pts)
    pin = to_mem(jo.points_mont(src_pts), mem)
    bb = bytes_mem(np.full((m + 2, 32), 0xA5, dtype=np.uint8), mem)
    okb = to_mem(np.full(m + 2, 0xA5, dtype=np.uint8), mem)
    c = ctypes.c_size_t(CANARY)
    assert lib.p252_points_to_bytes(ctx, P_(pin), m, P_(bb) + 32, P_(okb) + 1, ctypes.byref(c), flags) == 0
    bbh, okh = host_bytes(bb), host(okb)
    assert np.array_equal(bbh[1:m + 1], wb) and (bbh[0] == 0xA5).all() and (bbh[m + 1] == 0xA5).all()
    assert np.array_equal(okh[1:m + 1], wok2) and okh[0] == 0xA5 and okh[m + 1] == 0xA5 and c.value == 2
    pb2 = to_mem(np.full((m + 2, 2, 4), CANARY, dtype=np.uint64), mem)
    okb2 = to_mem(np.full(m + 2, 0xA5, dtype=np.uint8), mem)
    assert lib.p252_points_from_bytes(ctx, P_(bb) + 32, m, P_(pb2) + 64, P_(okb2) + 1, ctypes.byref(c), flags) == 0
    pbh, okh2 = host(pb2), host(okb2)
    wp, _ = expect_from(wb)
    assert np.array_equal(pbh[1:m + 1], wp) and (pbh[0] == CANARY).all() and (pbh[m + 1] == CANARY).all()
    assert np.array_equal(okh2[1:m + 1], wok2) and okh2[0] == 0xA5 and okh2[m + 1] == 0xA5 and c.value == 2


# 5 ---- composition on the device ---------------------------------------------------------------------------------------
def test_scan_from_wire_bytes(engine):
    rng = np.random.default_rng(8)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = jo.mul(a, G), jo.mul(b, G)
    n = 64
    gm = jo.points_mont([G])[0]
    r = [jo.random_secret(rng) for _ in range(n)]
    R, pk, ok = engine.stealth_address_batch(to_mem(jubjub_limbs(r), "device"), gm, to_mem(jo.points_mont([A]), "device"),
                                             to_mem(jo.points_mont([B]), "device"))
    pkh = host(pk).copy()
    pkh[::4, 1, 0] ^= np.uint64(1)                               # tampered notes: not ours (or not even on the curve)
    Rb, okR = engine.points_to_bytes(R)
    Pb, okP = engine.points_to_bytes(to_mem(pkh, "device"))
    al = to_mem(jubjub_limbs([a]), "device")
    want = host(engine.stealth_owns_batch(al, jo.points_mont([B])[0], gm, R, to_mem(pkh, "device")))
    # the wire form of the notes, decoded on the device, straight into the scan
    R2, okR2 = engine.points_from_bytes(Rb)
    P2, okP2 = engine.points_from_bytes(Pb)
    owned = engine.stealth_owns_batch(al, jo.points_mont([B])[0], gm, R2, P2)
    assert host(okR).all() and host(okR2).all()
    assert np.array_equal(host(owned), want) and want.sum() == n - n // 4 and not want[::4].any()


def test_signatures_verify_after_R_goes_through_bytes(engine):
    import torch
    rng = np.random.default_rng(9)
    n = 40
    sk = jo.random_secret(rng)
    PK = so.public_key(sk)
    gm = jo.points_mont([G])[0]
    r = [jo.random_secret(rng) for _ in range(n)]
    msg = to_mem(rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64), "device")
    u, R, ok = engine.schnorr_sign_batch(to_mem(jubjub_limbs([sk]), "device"), to_mem(jubjub_limbs(r), "device"), msg, gm)
    Rb, okb = engine.points_to_bytes(R)
    R2, ok2 = engine.points_from_bytes(Rb)
    torch.cuda.synchronize()
    assert host(ok).all() and host(okb).all() and host(ok2).all() and torch.equal(R, R2)
    pk = to_mem(jo.points_mont([PK]), "device")
    verified = engine.schnorr_verify_batch(pk, u, R2, msg, gm)
    assert host(verified).all() and engine.last_schnorr_verified() == n
    # a flipped sign bit is -R: no signature verifies
    Rbh = host(Rb).copy().view(np.uint8).reshape(n, 32)
    Rbh[:, 31] ^= 0x80
    R3, ok3 = engine.points_from_bytes(bytes_mem(Rbh, "device"))
    assert host(ok3).all()
    assert not host(engine.schnorr_verify_batch(pk, u, R3, msg, gm)).any()


# 6 ---- the C and C++ consumers on the GPU ------------------------------------------------------------------------------
def test_c_points_smoke_gpu():
    from test_points_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "POINTS_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_points_mirror_gpu():
    from test_points_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "points mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
