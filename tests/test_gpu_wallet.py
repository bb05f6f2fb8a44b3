"""Wallet scans on the device (p252_wallet_scan_batch) against the model of wallet_oracle.py, against the chain of
existing calls they replace (stealth_owns_batch per key, nullifier_batch and note_open_batch on the owned rows), and the
call's own plumbing: owned notes that do not open, 128-bit totals, invalid notes and bad keys, refused calls, batch sizes,
staging wipes, injected chunk failures and the two-generator table cache.  Fixtures live here."""
import ctypes
import functools

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import poseidon252_b200 as pb
import stealth_oracle as so
import wallet_oracle as wo
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_gpu_notes import ciphers, g_prime, pts
from test_gpu_schnorr import fr_rows
from test_gpu_stealth import CANARY, classes, host, mont, to_mem

pytestmark = pytest.mark.gpu

N, P, G = jo.R_J, jo.P, jo.GENERATOR
MEMS = [("host", False), ("device", False), ("device", True)]
RINV = pow(ho.R, -1, P)


@functools.lru_cache(maxsize=None)
def keyring(seed, k):
    """k good keys (a, b) and their public keys (A, B)"""
    rng = np.random.default_rng(seed)
    keys = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(k)]
    return keys, [so.keys(a, b) for a, b in keys]


def make_notes(engine, rng, publics, values):
    """HOST inputs of notes created on the device for the receivers publics[i] = (A, B) with values[i]: dict of R,
    note_pk, pos, nonce, cipher, C, and the blinders"""
    n = len(values)
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(n)])
    bl = jubjub_limbs([jo.random_secret(rng) for _ in range(n)])
    nonce = rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64)
    nonce[:, 3] = 0
    v = np.array([int(x) for x in values], dtype=np.uint64)
    A, B = pts([p[0] for p in publics]), pts([p[1] for p in publics])
    R, pk, C, cipher, ok = engine.note_create_batch(r, v, bl, nonce, mont(G), mont(g_prime()), A, B)
    assert ok.all()
    pos = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    return {"R": R, "note_pk": pk, "pos": pos, "nonce": nonce, "cipher": cipher, "C": C, "blinder": bl, "value": v}


def scan(engine, keys, notes, mem="host", async_=False, base_p=None):
    a = to_mem(jubjub_limbs([k[0] for k in keys]), mem)
    b = to_mem(jubjub_limbs([k[1] for k in keys]), mem)
    args = [to_mem(notes[x], mem) for x in ("R", "note_pk", "pos", "nonce", "cipher", "C")]
    out = engine.wallet_scan_batch(a, b, *args, mont(G), mont(g_prime() if base_p is None else base_p), async_=async_)
    if async_:
        engine.sync()
    return [host(x) for x in out]


def fr_int(row):
    """Montgomery limbs -> the canonical int; a value >= p is passed through raw, so that the model sees it (as fr_rows)"""
    x = sum(int(row[k]) << (64 * k) for k in range(4))
    return x if x >= P else x * RINV % P


def pt_int(rows):
    return (fr_int(rows[0]), fr_int(rows[1]))


def model_notes(notes):
    return [(pt_int(notes["R"][i]), pt_int(notes["note_pk"][i]), int(notes["pos"][i]), fr_int(notes["nonce"][i]),
             [fr_int(c) for c in notes["cipher"][i]], pt_int(notes["C"][i])) for i in range(len(notes["pos"]))]


def check_against_model(engine, keys, notes, out):
    """every output of the call against wallet_oracle.scan; the counts of the engine"""
    owner, nul, value, blinder, opened, totals = out
    want = wo.scan(keys, model_notes(notes), g_prime())
    assert owner.tolist() == want["owner"]
    assert np.array_equal(nul, fr_rows([0 if x is None else x for x in want["nullifier"]]))
    assert value.tolist() == want["value"] and opened.tolist() == want["opened"]
    assert np.array_equal(blinder, jubjub_limbs(want["blinder"]))
    assert totals.tolist() == want["totals"]
    assert engine.last_wallet_invalid() == want["n_invalid"] and engine.last_wallet_bad_keys() == want["n_bad_keys"]


def chain(engine, keys, notes):
    """the chain of existing calls: per key the ownership scan, then nullifier_batch and note_open_batch on its rows"""
    n = len(notes["pos"])
    owner = np.full(n, -1, np.int32)
    nul, value = np.zeros((n, 4), np.uint64), np.zeros(n, np.uint64)
    blinder, opened = np.zeros((n, 4), np.uint64), np.zeros(n, np.uint8)
    totals = np.zeros((len(keys), 4), np.uint64)
    gm, gpm = mont(G), mont(g_prime())
    for j, (a, b) in enumerate(keys):
        B = pts([jo.mul(b, G)])[0]
        owned = engine.stealth_owns_batch(jubjub_limbs([a]), B, gm, notes["R"], notes["note_pk"])
        rows = np.flatnonzero((owned != 0) & (owner < 0))
        if not len(rows):
            continue
        owner[rows] = j
        nul[rows], _ = engine.nullifier_batch(jubjub_limbs([a]), jubjub_limbs([b]), gpm, notes["R"][rows], notes["pos"][rows])
        value[rows], blinder[rows], opened[rows] = engine.note_open_batch(
            jubjub_limbs([a]), notes["R"][rows], notes["nonce"][rows], notes["cipher"][rows], notes["C"][rows], gm, gpm)
        s = sum(int(x) for x in value[rows])
        totals[j] = [s & ((1 << 64) - 1), s >> 64, len(rows), int(opened[rows].sum())]
    return owner, nul, value, blinder, opened, totals


def concat(*parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


# 1 ---- against the model: owned, foreign, invalid and edge notes, bad and duplicate keys ------------------------------
@pytest.mark.parametrize("mem,async_", MEMS)
@pytest.mark.parametrize("k", [1, 3, 8])
def test_against_model(engine, mem, async_, k):
    rng = np.random.default_rng(100 + k)
    keys, pubs = keyring(10 + k, k)
    keys = list(keys)
    if k >= 3:
        keys[1] = (keys[1][0] + N, keys[1][1])                     # bad keys: a >= r_J, b >= r_J
        keys[2] = (keys[2][0], keys[2][1] + N)
    if k == 8:
        keys[7] = keys[4]                                         # a duplicate: the smaller index owns
    stranger = so.keys(jo.random_secret(rng), jo.random_secret(rng))
    publics = [pubs[j % k] for j in range(2 * k)] + [stranger] * 2
    vals = [int(x) for x in rng.integers(0, 1 << 62, len(publics))]
    notes = make_notes(engine, rng, publics, vals)
    n0 = len(vals)
    # invalid notes: R off the curve, R with u >= p, note_pk with v >= p; a foreign note_pk off the curve (canonical)
    bad = {key: notes[key][:4].copy() for key in notes}
    bad["R"][0] = pts([jo.off_curve_point(rng)])[0]
    bad["R"][1, 0] = fr_rows([P])[0]
    bad["note_pk"][2, 1] = fr_rows([P + 5])[0]
    bad["note_pk"][3] = pts([jo.off_curve_point(rng)])[0]
    # edge R: every order class, each with the note key key 0 derives from it (owned by key 0; the cipher does not open)
    edge = {key: notes[key][:len(classes())].copy() for key in notes} if n0 >= len(classes()) else None
    parts = [notes, bad]
    if edge is not None:
        a0, b0 = keys[0]
        edge["R"] = pts(list(classes()))
        edge["note_pk"] = pts([so.note_key(a0, jo.mul(b0, G), R) for R in classes()])
        parts.append(edge)
    allnotes = concat(*parts)
    out = scan(engine, keys, allnotes, mem, async_)
    check_against_model(engine, keys, allnotes, out)
    assert (out[0][:2 * k] >= 0).sum() >= 1 and (out[0][n0:n0 + 4] == -1).all()


# 2 ---- against the chain of existing calls, k = 5 and a few thousand notes ------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_equals_existing_calls(engine, mem):
    rng = np.random.default_rng(200)
    keys, pubs = keyring(20, 5)
    strangers = [so.keys(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(3)]
    n = 3000
    pick = rng.integers(0, 20, n)                                 # a quarter owned, spread over the keys
    publics = [pubs[p] if p < 5 else strangers[p % 3] for p in pick]
    notes = make_notes(engine, rng, publics, rng.integers(0, 1 << 63, n, dtype=np.uint64) * 2 + 1)
    out = scan(engine, keys, notes, mem)
    want = chain(engine, keys, notes)
    for got, w in zip(out, want):
        assert np.array_equal(got, w)
    assert (out[0] >= 0).sum() == (pick < 5).sum() and out[4][out[0] >= 0].all()


# 3 ---- owned notes that do not open ---------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_owned_notes_that_do_not_open(engine, mem):
    rng = np.random.default_rng(300)
    keys, pubs = keyring(30, 2)
    notes = make_notes(engine, rng, [pubs[1]] * 4, [5, 6, 7, 8])
    notes["cipher"][0, 1, 0] ^= 1                                 # tampered cipher
    notes["C"][1] = notes["C"][2]                                 # another note's commitment
    a, b = keys[1]                                                # an out-of-range plaintext with its own commitment
    R = pt_int(notes["R"][3])
    m0, m1 = (1 << 64) + 3, 11
    notes["cipher"][3] = ciphers([ho.encrypt([m0, m1], list(jo.mul(a, R)), fr_int(notes["nonce"][3]))])[0]
    notes["C"][3] = pts([jo.add(jo.mul(m0, G), jo.mul(m1, g_prime()))])[0]
    out = scan(engine, keys, notes, mem)
    owner, nul, value, blinder, opened, totals = out
    assert owner.tolist() == [1] * 4 and opened.tolist() == [0, 0, 1, 0]
    assert value.tolist() == [0, 0, 7, 0] and not blinder[[0, 1, 3]].any() and nul.all(axis=1).all()
    assert totals.tolist() == [[0, 0, 0, 0], [7, 0, 4, 1]]
    check_against_model(engine, keys, notes, out)


# 4 ---- totals carry into value_hi ------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_totals_carry_into_value_hi(engine, mem):
    rng = np.random.default_rng(400)
    keys, pubs = keyring(40, 2)
    top = (1 << 64) - 1
    notes = make_notes(engine, rng, [pubs[0]] * 3 + [pubs[1]] * 2, [top, top, top, top, 1])
    totals = scan(engine, keys, notes, mem)[5]
    assert totals.tolist() == [[(3 * top) & top, 2, 3, 3], [0, 1, 2, 2]]


# 5 ---- refused calls: nothing written, nothing launched --------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "device"])
def test_refused_calls_write_nothing_and_launch_nothing(engine, mem):
    rng = np.random.default_rng(500)
    keys, pubs = keyring(50, 2)
    notes = {k: to_mem(v, mem) for k, v in make_notes(engine, rng, [pubs[0]] * 4, [1, 2, 3, 4]).items()}
    lib, ctx = _native.lib(), engine._ctx
    flags = _native.MEM_DEVICE if mem == "device" else _native.MEM_HOST
    ab = to_mem(jubjub_limbs([k[0] for k in keys]), mem)
    g, gp = mont(G), mont(g_prime())
    off = g.copy()
    off[1, 0] ^= 1
    outs = [to_mem(np.full(s, CANARY, np.uint64), mem) for s in ((2,), (4, 4), (4,), (4, 4), (1,), (2, 4))]
    owner, nul, value, blinder, opened, totals = outs            # owner and opened are 8 canary bytes
    ptr = lambda x: x.data_ptr() if mem == "device" else x.ctypes.data   # noqa: E731
    inval, bad = ctypes.c_size_t(9), ctypes.c_size_t(9)

    def call(nk=2, n=4, G_=g, Gp_=gp, R=None, own=None, pos=None):
        return lib.p252_wallet_scan_batch(ctx, ptr(ab), ptr(ab), nk, ptr(notes["R"]) if R is None else R,
                                          ptr(notes["note_pk"]), ptr(notes["pos"]) if pos is None else pos,
                                          ptr(notes["nonce"]), ptr(notes["cipher"]), ptr(notes["C"]), n, G_.ctypes.data,
                                          Gp_.ctypes.data, ptr(owner) if own is None else own, ptr(nul), ptr(value),
                                          ptr(blinder), ptr(opened), ptr(totals), ctypes.byref(inval), ctypes.byref(bad),
                                          flags)

    before = engine.launch_count
    refusals = [call(nk=0), call(nk=257), call(R=0), call(own=0)]        # INVALID_ARGUMENT (-1)
    if mem == "device":
        refusals += [call(R=ptr(notes["R"]) + 8), call(pos=ptr(notes["pos"]) + 4), call(own=ptr(owner) + 2)]
    assert refusals == [-1] * len(refusals), refusals
    assert call(Gp_=off) == call(G_=off, n=0) == 6                        # INVALID_POINT, also for n == 0
    assert engine.launch_count == before
    for o in outs:
        assert (host(o) == CANARY).all()
    assert inval.value == 9 and bad.value == 9


# 6 ---- plumbing: batch sizes, staging, injected failures, the table cache ----------------------------------------------
def test_batch_sizes(engine):
    rng = np.random.default_rng(600)
    keys, pubs = keyring(60, 3)
    stranger = so.keys(jo.random_secret(rng), jo.random_secret(rng))
    big = 70000                                                  # several staged chunks in both memory spaces
    pick = rng.integers(0, 12, big)
    notes = make_notes(engine, rng, [pubs[p] if p < 3 else stranger for p in pick],
                       rng.integers(0, 1 << 63, big, dtype=np.uint64))
    import torch
    coop = 24 * torch.cuda.get_device_properties(0).multi_processor_count
    for n in (0, 1, 31, 32, 33, 1023, 1024, 1025, coop // 3, coop // 3 + 1, big):
        part = {k: v[:n] for k, v in notes.items()}
        want = chain(engine, keys, part) if n else None
        for mem in ("host", "device"):
            out = scan(engine, keys, part, mem)
            if n == 0:
                assert all(x.shape[0] == 0 for x in out[:5]) and not out[5].any()
                continue
            for got, w in zip(out, want):
                assert np.array_equal(got, w), (n, mem)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_staging_zero_after_every_call(engine, mem):
    rng = np.random.default_rng(700)
    keys, pubs = keyring(70, 2)
    notes = make_notes(engine, rng, [pubs[0], pubs[1]] * 4, list(range(8)))
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    out = scan(engine, keys, notes, mem)
    assert out[4].all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


def chunks(n, k, mem):
    """the chunk sizes p252_wallet_scan_batch stages n notes in: pipeline_chunk's size from the bytes per note of its
    staged buffers (a DEVICE call stages only its arena rows), then the ramp-up of the first chunks"""
    r16 = lambda x: (x + 15) // 16 * 16                           # noqa: E731
    arena = [64 * k, k, 32 * k, k, 8, 64, 32, 32, 8, 32, 96, 64, 1, 96, 32, 64, 1, 8, 32]
    io = [64, 64, 8, 32, 96, 64, 4, 32, 8, 32, 1] if mem == "host" else []
    per = sum(r16(x) for x in arena + io)
    chunk = max(1024, min(1 << 17, (24 << 20) // per))
    chunk = min((chunk + 127) // 128 * 128, n)
    cur, out, off = (max(1024, chunk // 8 // 128 * 128) if n > 2 * chunk else chunk), [], 0
    while off < n:
        out.append(min(cur, n - off))
        off += out[-1]
        cur = min(chunk, cur * 2)
    return out


@pytest.mark.parametrize("mem", ["host", "device"])
def test_multi_chunk_fault_retry_and_launches(engine, mem):
    rng = np.random.default_rng(800)
    keys, pubs = keyring(80, 2)
    n = 60000
    notes = make_notes(engine, rng, [pubs[i % 2] for i in range(n)], rng.integers(0, 1 << 40, n, dtype=np.uint64))
    sizes = chunks(n, 2, mem)
    assert len(sizes) >= 4, sizes
    lib, ctx, nz = _native.lib(), engine._ctx, ctypes.c_size_t(1)
    want = chain(engine, keys, notes)
    # a chunk's second phase is enqueued after the next chunk's first: a failure at chunk 1 leaves chunk 0's first phase
    # (5 launches), one at chunk 2 the first phases of chunks 0 and 1 and the second phase of chunk 0 (15)
    for fail_at, launched in ((1, 5), (2, 15)):
        assert lib.p252_debug_fail_chunk(ctx, fail_at) == 0
        before = engine.launch_count
        with pytest.raises(pb.EngineError):
            scan(engine, keys, notes, mem)
        assert engine.launch_count - before == launched
        assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0
    before = engine.launch_count
    out = scan(engine, keys, notes, mem)                          # the retry is correct
    assert engine.launch_count - before == 10 * len(sizes)        # 5 + 5 per chunk: every chunk has owned notes
    for got, w in zip(out, want):
        assert np.array_equal(got, w)
    assert (out[0] >= 0).all() and out[4].all()
    assert lib.p252_debug_staging_nonzero(ctx, ctypes.byref(nz)) == 0 and nz.value == 0


@pytest.mark.parametrize("mem", ["host", "device"])
def test_empty_batch_writes_and_counts_nothing(engine, mem):
    """n == 0 runs nothing: with a bad key both counts are 0 and the totals are left as they were"""
    keys, _ = keyring(85, 2)
    bad = [keys[0], (keys[1][0] + N, keys[1][1])]
    empty = {"R": np.zeros((0, 2, 4), np.uint64), "note_pk": np.zeros((0, 2, 4), np.uint64), "pos": np.zeros(0, np.uint64),
             "nonce": np.zeros((0, 4), np.uint64), "cipher": np.zeros((0, 3, 4), np.uint64),
             "C": np.zeros((0, 2, 4), np.uint64)}
    before = engine.launch_count
    out = scan(engine, bad, empty, mem)
    assert engine.launch_count == before and not out[5].any()
    assert engine.last_wallet_invalid() == 0 and engine.last_wallet_bad_keys() == 0


def test_table_cache_by_launch_count(engine):
    """after a double-key call the scan builds no table, alternating with the note calls rebuilds none, and the
    single-base slot is left alone"""
    rng = np.random.default_rng(900)
    keys, pubs = keyring(90, 2)
    gm, gpm = mont(G), mont(g_prime())
    third = mont(jo.mul(12345, G))
    notes = make_notes(engine, rng, [pubs[0], pubs[1]] * 4, list(range(8)))   # (the note calls' tables are built here)
    r = jubjub_limbs([jo.random_secret(rng) for _ in range(8)])
    engine.fixed_base_batch(r, third)

    def launches(call):
        before = engine.launch_count
        call()
        return engine.launch_count - before

    al = jubjub_limbs([keys[0][0]])
    for _ in range(2):
        assert launches(lambda: scan(engine, keys, notes)) == 10
        assert launches(lambda: engine.note_open_batch(al, notes["R"], notes["nonce"], notes["cipher"], notes["C"], gm,
                                                       gpm)) == 3
        assert launches(lambda: engine.schnorr_sign_double_batch(r[:1], r, fr_rows([1] * 8), gm, gpm)) == 5
    assert launches(lambda: engine.fixed_base_batch(r, third)) == 1


# 7 ---- the C and C++ consumers on the GPU ---------------------------------------------------------------------------
def test_c_wallet_smoke_gpu():
    from test_wallet_cpu import c_smoke
    res = c_smoke()
    assert res.returncode == 0 and "WALLET_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


def test_cpp_wallet_mirror_gpu():
    from test_wallet_cpu import cpp_mirror
    res = cpp_mirror()
    assert res.returncode == 0 and "wallet mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
