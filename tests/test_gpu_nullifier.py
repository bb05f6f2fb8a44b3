"""Note nullifiers on the device (p252_nullifier_batch) against the model of nullifier_oracle.py (affine complete addition,
double-and-add, the Python Hades), against the existing calls they are built from (stealth_address_batch + hash_batch
with G' = G; dhke_batch -> hash_batch_truncated -> a host add -> fixed_base_batch -> hash_batch with G' != G), and the
call's own plumbing: invalid items, refused calls, batch sizes, staging wipes, injected chunk failures and launches."""
import ctypes
import functools

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_edges as je
import jubjub_oracle as jo
import nullifier_oracle as no
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs, to_mont
from test_gpu_schnorr import fr_rows
from test_gpu_stealth import CANARY, _sizes, host, mont, s_int, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
POS = [0, 1, 1 << 32, (1 << 64) - 1]
A_EDGES = [1, 2, N - 1, int("f" * 62, 16)] + list(je.OUTPUT_SECRETS)
B_EDGES = [0, 1, N - 1, (1 << 250) + 3, 0x0b3f6a5c1d2e3f405162738495a6b7c8d9eafb0c1d2e3f4051627384950a1b2c]


@functools.lru_cache(maxsize=None)
def g_prime():
    """a random point of the prime-order subgroup as G' (GENERATOR_NUMS is not pinned here)"""
    return jo.random_subgroup_point(np.random.default_rng(700))


@functools.lru_cache(maxsize=None)
def model(a, b, R, pos, Gp):
    """(nullifier, ok) as the device writes them: 0 for an invalid item"""
    v = no.nullifier(a, b, R, pos, Gp)
    return (0, 0) if v is None else (v, 1)


def expect(a_s, b_s, Rs, pos, Gp):
    rows = [model(a, b, R, p, Gp) for a, b, R, p in zip(a_s, b_s, Rs, pos)]
    out = fr_rows([r[0] for r in rows])
    ok = np.array([r[1] for r in rows], dtype=np.uint8)
    out[ok == 0] = 0
    return out, ok


def pos_rows(pos, mem):
    return to_mem(np.array(pos, dtype=np.uint64), mem)


def h_of(a, R):
    return so.hash_point(je.mul(a, R))


@functools.lru_cache(maxsize=None)
def edge_R():
    """R at the field's edges: one prime-subgroup point of every class, the first point of every class (any order), G,
    and the small-order points"""
    rng = np.random.default_rng(701)
    pts = [e.pt for e in je.subgroup_edges()] + [je.edges(k)[0].pt for k in je.KINDS] + [G]
    return tuple(dict.fromkeys(pts + jo.small_order_points(rng)))


# 1 ---- parity with the model: edge R, secrets and positions, both G', every memory space and n_secret ---------------------
@pytest.mark.parametrize("mem,async_", [("host", False), ("device", False), ("device", True)])
@pytest.mark.parametrize("n_secret", ["one", "n"])
@pytest.mark.parametrize("gp", ["random", "G"])
def test_parity_with_model(engine, mem, async_, n_secret, gp):
    Gp = g_prime() if gp == "random" else G
    Rs = list(edge_R())
    n = len(Rs)
    pos = [POS[i % len(POS)] for i in range(n)]
    if n_secret == "n":
        a_s = [A_EDGES[i % len(A_EDGES)] for i in range(n)]
        b_s = [B_EDGES[(3 * i) % len(B_EDGES)] for i in range(n)]
        b_s[0] = N - h_of(a_s[0], Rs[0])                          # note_sk = 0
        b_s[1] = N - h_of(a_s[1], Rs[1]) + 5                      # h + b = r_J + 5: wraps to 5
        calls, zero = [(a_s, b_s)], (0, 0)
    else:                                                         # b = r_J - 1 wraps for every h > 0; note_sk = 0 at item 2
        calls = [([A_EDGES[0]] * n, [B_EDGES[3]] * n), ([A_EDGES[5]] * n, [N - 1] * n),
                 ([A_EDGES[6]] * n, [N - h_of(A_EDGES[6], Rs[2])] * n)]
        zero = (2, 2)
    za, zb = calls[zero[0]][0][zero[1]], calls[zero[0]][1][zero[1]]
    assert no.note_sk(za, zb, Rs[zero[1]]) == 0                   # pk' = (0, 1)
    assert model(za, zb, Rs[zero[1]], pos[zero[1]], Gp)[0] == ho.Hash.digest(ho.Domain.Other, [0, 1, pos[zero[1]]])[0]
    for a_s, b_s in calls:
        want, wok = expect(a_s, b_s, Rs, pos, Gp)
        assert wok.all()
        k = 1 if n_secret == "one" else n
        out, ok = engine.nullifier_batch(to_mem(jubjub_limbs(a_s[:k]), mem), to_mem(jubjub_limbs(b_s[:k]), mem), mont(Gp),
                                         to_mem(jo.points_mont(Rs), mem), pos_rows(pos, mem), async_=async_)
        if async_:
            engine.sync()
        assert np.array_equal(host(ok), wok) and np.array_equal(host(out), want)
        assert engine.last_nullifier_invalid() == 0
    one = pb.nullifier(a_s[3], b_s[3], mont(Gp), mont(Rs[3]), pos[3], engine=engine)
    assert np.array_equal(one, expect([a_s[3]], [b_s[3]], [Rs[3]], [pos[3]], Gp)[0][0])


# 2 ---- against the existing calls, 2^18 notes ------------------------------------------------------------------------------
def _random_r(rng, n):
    r = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    r[:, 3] %= np.uint64(N >> 192)
    return r


def test_equals_stealth_note_keys_with_G(engine):
    """[note_sk] G is the note's key: with G' = G the nullifier is hash_batch(Other, [note_pk.u, note_pk.v, pos])"""
    import torch
    rng = np.random.default_rng(20)
    n = 1 << 18
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    gm = mont(G)
    pool = np.array(POS + [int(x) for x in rng.integers(0, 1 << 63, 60, dtype=np.uint64)], dtype=np.uint64)
    sel = rng.integers(0, len(pool), n)
    pos, pm = pool[sel], to_mont([int(x) for x in pool])[sel]
    R, pk, ok = engine.stealth_address_batch(to_mem(_random_r(rng, n), "device"), gm, to_mem(jo.points_mont([A]), "device"),
                                             to_mem(jo.points_mont([B]), "device"))
    nul, okn = engine.nullifier_batch(to_mem(jubjub_limbs([a]), "device"), to_mem(jubjub_limbs([b]), "device"), gm, R,
                                      to_mem(pos, "device"))
    rows = torch.cat([pk.reshape(n, 2, 4), to_mem(pm, "device").reshape(n, 1, 4)], dim=1).contiguous()
    want = engine.hash_batch(pb.Domain.Other, rows)
    torch.cuda.synchronize()
    assert host(ok).all() and host(okn).all() and engine.last_nullifier_invalid() == 0
    assert torch.equal(nul.reshape(n, 4), want.reshape(n, 4))
    for i in rng.choice(n, 3, replace=False):
        Ri = jo.points_from_mont(host(R)[i:i + 1])[0]
        assert np.array_equal(host(nul)[i], expect([a], [b], [Ri], [int(pos[i])], G)[0][0])


def test_equals_the_five_call_chain(engine):
    """with G' != G: dhke_batch -> hash_batch_truncated -> (h + b) mod r_J on the host -> fixed_base_batch(G') -> host
    pack [u, v, pos] -> hash_batch"""
    import torch
    rng = np.random.default_rng(21)
    n = 1 << 18
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    Gp = g_prime()
    gpm = mont(Gp)
    R, _ = engine.fixed_base_batch(to_mem(_random_r(rng, n), "device"), mont(G))
    pool = np.array(POS + [int(x) for x in rng.integers(0, 1 << 63, 60, dtype=np.uint64)], dtype=np.uint64)
    sel = rng.integers(0, len(pool), n)
    pos, pm = pool[sel], to_mont([int(x) for x in pool])[sel]
    al, bl = to_mem(jubjub_limbs([a]), "device"), to_mem(jubjub_limbs([b]), "device")
    nul, ok = engine.nullifier_batch(al, bl, gpm, R, to_mem(pos, "device"))
    shared, oks = engine.dhke_batch(al, R)
    h = host(engine.hash_batch_truncated(pb.Domain.Other, shared)).reshape(n, 4)
    sk = np.frombuffer(b"".join(((int.from_bytes(row.tobytes(), "little") + b) % N).to_bytes(32, "little") for row in h),
                       dtype=np.uint64).reshape(n, 4).copy()
    pkp, okp = engine.fixed_base_batch(to_mem(sk, "device"), gpm)
    rows = np.concatenate([host(pkp).reshape(n, 2, 4), pm.reshape(n, 1, 4)], axis=1)
    want = host(engine.hash_batch(pb.Domain.Other, to_mem(rows, "device")))
    torch.cuda.synchronize()
    assert host(ok).all() and host(oks).all() and host(okp).all() and engine.last_nullifier_invalid() == 0
    assert np.array_equal(host(nul).reshape(n, 4), want.reshape(n, 4))
    for i in rng.choice(n, 2, replace=False):
        Ri = jo.points_from_mont(host(R)[i:i + 1])[0]
        assert np.array_equal(host(nul)[i], expect([a], [b], [Ri], [int(pos[i])], Gp)[0][0])


# 3 ---- invalid items, with canaries around every output -----------------------------------------------------------------
def _raw_call(engine, mem, a_l, b_l, ns, Gm, Rm, pos, n):
    """the C call with canary rows before and after the nullifier and ok buffers -> (nullifier, ok, whole buffers, count)"""
    lib, P_ = _native.lib(), engine._ptr
    big = to_mem(np.full((n + 2, 4), CANARY, dtype=np.uint64), mem)
    okb = to_mem(np.full(n + 2, 0xA5, dtype=np.uint8), mem)
    cnt = ctypes.c_size_t(CANARY)
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    assert lib.p252_nullifier_batch(engine._ctx, P_(a_l), P_(b_l), ns, Gm.ctypes.data, P_(Rm), P_(pos), n, P_(big) + 32,
                                    P_(okb) + 1, ctypes.byref(cnt), flags) == 0
    bh, oh = host(big), host(okb)
    assert (bh[0] == CANARY).all() and (bh[n + 1] == CANARY).all() and oh[0] == 0xA5 and oh[n + 1] == 0xA5
    return bh[1:n + 1], oh[1:n + 1], cnt.value


@pytest.mark.parametrize("mem", ["host", "device"])
def test_invalid_items_zeroed_and_counted_once(engine, mem):
    rng = np.random.default_rng(30)
    n = 12
    Gp = g_prime()
    a_s = [jo.random_secret(rng) for _ in range(n)]
    b_s = [jo.random_secret(rng) for _ in range(n)]
    Rs = [je.mul(jo.random_secret(rng), G) for _ in range(n)]
    pos = [int(x) for x in rng.integers(0, 1 << 63, n, dtype=np.uint64)]
    a_s[1] = N                                                    # a >= r_J
    b_s[2] = N                                                    # b >= r_J
    Rs[3] = (Rs[3][0] + P, Rs[3][1])                              # an R coordinate >= p
    Rs[4] = jo.off_curve_point(rng)                               # R off the curve
    b_s[5] = (1 << 256) - 1                                       # b far out of range
    a_s[6], b_s[6], Rs[6] = N + 5, N + 1, (0, 0)                  # all three
    bad = np.zeros(n, dtype=bool)
    bad[1:7] = True
    want, wok = expect(a_s, b_s, Rs, pos, Gp)
    assert np.array_equal(wok, (~bad).astype(np.uint8))
    Rm = to_mem(jo.points_mont(Rs), mem)
    out, ok, cnt = _raw_call(engine, mem, to_mem(jubjub_limbs(a_s), mem), to_mem(jubjub_limbs(b_s), mem), n, mont(Gp), Rm,
                             pos_rows(pos, mem), n)
    assert np.array_equal(ok, wok) and np.array_equal(out, want) and cnt == 6
    # a >= r_J for the whole batch (n_secret = 1): every item invalid
    out, ok, cnt = _raw_call(engine, mem, to_mem(jubjub_limbs([N]), mem), to_mem(jubjub_limbs([3]), mem), 1, mont(Gp), Rm,
                             pos_rows(pos, mem), n)
    assert not ok.any() and not out.any() and cnt == n
    with pytest.raises(pb.InvalidPoint):
        pb.nullifier(1, N, mont(Gp), mont(G), 0, engine=engine)
    res, okp = engine.nullifier_batch(to_mem(jubjub_limbs([N]), mem), to_mem(jubjub_limbs([3]), mem), mont(Gp), Rm,
                                      pos_rows(pos, mem))
    assert not host(okp).any() and engine.last_nullifier_invalid() == n


# 4 ---- refused calls ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing(engine, mem):
    rng = np.random.default_rng(40)
    lib, ctx, P_ = _native.lib(), engine._ctx, engine._ptr
    flags = 0 if mem == "host" else _native.MEM_DEVICE
    n = 5
    al, bl = to_mem(jubjub_limbs([3] * n), mem), to_mem(jubjub_limbs([4] * n), mem)
    Rm = to_mem(jo.points_mont([G] * n), mem)
    pm = pos_rows(list(range(n)), mem)
    gm = mont(G)
    for bp in [mont(jo.off_curve_point(rng)), mont((G[0] + P, G[1])), mont((G[0], G[1] + P))]:
        out = to_mem(np.full((n, 4), CANARY, dtype=np.uint64), mem)
        ok = to_mem(np.full(n, 0xA5, dtype=np.uint8), mem)
        c = ctypes.c_size_t(CANARY)
        before = engine.launch_count
        for nn in (n, 0):
            assert lib.p252_nullifier_batch(ctx, P_(al), P_(bl), 1, bp.ctypes.data, P_(Rm), P_(pm), nn, P_(out), P_(ok),
                                            ctypes.byref(c), flags) == 6
        assert engine.launch_count == before and c.value == CANARY
        assert (host(out) == CANARY).all() and (host(ok) == 0xA5).all()
        with pytest.raises(pb.InvalidPoint):
            engine.nullifier_batch(al, bl, bp, Rm, pm)
    out = to_mem(np.zeros((n, 4), dtype=np.uint64), mem)
    ok = to_mem(np.zeros(n, dtype=np.uint8), mem)
    args = [P_(al), P_(bl), P_(Rm), P_(pm), P_(out), P_(ok)]

    def call(a_, b_, ns, g_, R_, p_, o_, k_, nn=n):
        return lib.p252_nullifier_batch(ctx, a_, b_, ns, g_, R_, p_, nn, o_, k_, None, flags)

    assert call(args[0], args[1], n, None, *args[2:]) == -1
    for k in range(6):                                            # each buffer NULL in turn
        x = list(args)
        x[k] = None
        assert call(x[0], x[1], n, gm.ctypes.data, *x[2:]) == -1
    assert call(args[0], args[1], 2, gm.ctypes.data, *args[2:]) == -1
    assert call(args[0], args[1], 0, gm.ctypes.data, *args[2:]) == -1
    if mem == "device":
        for k, off in ((0, 8), (1, 8), (2, 8), (4, 8), (3, 4)):   # a, b, R, nullifier by 8; pos by 4
            x = list(args)
            x[k] += off
            assert call(x[0], x[1], 1, gm.ctypes.data, *x[2:], nn=1) == -1
    assert (host(out) == 0).all()


# 5 ---- plumbing: batch sizes, staging, injected failures, launches per chunk ---------------------------------------------
@functools.lru_cache(maxsize=None)
def pool(seed, k=8):
    """k notes R (subgroup points), four positions, one wallet key, G' and the model's nullifiers of every (R, pos)"""
    rng = np.random.default_rng(seed)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    Rs = [je.mul(jo.random_secret(rng), G) for _ in range(k)]
    Gp = g_prime()
    table = np.stack([expect([a] * len(POS), [b] * len(POS), [R] * len(POS), POS, Gp)[0] for R in Rs])
    return a, b, Rs, Gp, table


def test_batch_sizes(engine):
    rng = np.random.default_rng(50)
    a, b, Rs, Gp, table = pool(51)
    Rm = jo.points_mont(Rs)
    al, bl = to_mem(jubjub_limbs([a]), "device"), to_mem(jubjub_limbs([b]), "device")
    for n in _sizes():
        ri, pi = rng.integers(0, len(Rs), n), rng.integers(0, len(POS), n)
        out, ok = engine.nullifier_batch(al, bl, mont(Gp), to_mem(Rm[ri], "device"),
                                         to_mem(np.array(POS, dtype=np.uint64)[pi], "device"))
        rows = rng.choice(n, min(n, 32), replace=False)
        assert host(ok).all() and engine.last_nullifier_invalid() == 0
        assert np.array_equal(host(out)[rows], table[ri[rows], pi[rows]])


@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_calls(engine, mem):
    a, b, Rs, Gp, table = pool(52)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    out, ok = engine.nullifier_batch(to_mem(jubjub_limbs([a]), mem), to_mem(jubjub_limbs([b]), mem), mont(Gp),
                                     to_mem(jo.points_mont(Rs), mem), pos_rows([POS[1]] * len(Rs), mem))
    assert host(ok).all() and np.array_equal(host(out), table[:, 1])
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def test_host_multi_chunk_fault_retry_and_launches(engine):
    rng = np.random.default_rng(53)
    n = 200000                                                    # several staged chunks
    a, b, Rs, Gp, table = pool(54)
    ri, pi = rng.integers(0, len(Rs), n), rng.integers(0, len(POS), n)
    Rm, pos = jo.points_mont(Rs)[ri], np.array(POS, dtype=np.uint64)[pi]
    al, bl, gpm = jubjub_limbs([a]), jubjub_limbs([b]), mont(Gp)
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    for fail_at in (1, 2):
        assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
        with pytest.raises(pb.EngineError):
            engine.nullifier_batch(al, bl, gpm, Rm, pos)
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    engine.fixed_base_batch(al, gpm)                              # the table of G' is built
    before = engine.launch_count
    out, ok = engine.nullifier_batch(al, bl, gpm, Rm, pos)        # the retry is correct
    launches = engine.launch_count - before
    assert ok.all() and np.array_equal(out, table[ri, pi]) and engine.last_nullifier_invalid() == 0
    # no table rebuild for the repeated G': 5 launches per chunk, over several chunks
    assert launches % 5 == 0 and launches > 5
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


# 6 ---- the C and C++ consumers on the GPU ---------------------------------------------------------------------------------
def test_c_nullifier_smoke_gpu():
    from test_nullifier_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "NULLIFIER_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_nullifier_mirror_gpu():
    from test_nullifier_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "nullifier mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
