"""Note values without a GPU: the model of note_oracle.py (create -> open round trips, the commitment's homomorphism,
notes that must not open), a model of the kernels' 17-window recoding of a u64, the product counts the kernels pin, and
the bindings of p252_value_commit_batch / p252_note_create_batch / p252_note_open_batch -- the header, the library, the
ctypes signature table and the Rust block in notes.rs agree, the plain-C program calls exactly the new block, the C and
C++ programs compile, and the calls fail loudly without a GPU.  The same C and C++ programs run on the device in
test_gpu_notes.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import note_oracle as nto
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_stealth_cpu import LIBDIR, ROOT, RUST, _blocks, _header

WANT = {"p252_value_commit_batch": 10, "p252_note_create_batch": 18, "p252_note_open_batch": 15}
N, P, G = jo.R_J, jo.P, jo.GENERATOR
V_EDGES = [0, 1, 7, 8, 9, 15, 16, int("7" * 16, 16), int("8" * 16, 16), 1 << 63, (1 << 64) - 1]


def _wallet(seed):
    rng = np.random.default_rng(seed)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    return rng, a, A, B, jo.random_subgroup_point(rng)


def _note(rng, A, B, Gp, v=None, blinder=None):
    v = int(rng.integers(0, 1 << 63)) * 2 + 1 if v is None else v
    blinder = jo.random_secret(rng) if blinder is None else blinder
    nonce = int(rng.integers(0, 1 << 62))
    R, pk, C, cipher = nto.create(jo.random_secret(rng), v, blinder, nonce, A, B, Gp)
    return v, blinder, nonce, R, pk, C, cipher


# ---- the model ------------------------------------------------------------------------------------------------------
def test_create_open_round_trips():
    rng, a, A, B, Gp = _wallet(1)
    for v, bl in ((0, 0), (1, 1), ((1 << 64) - 1, N - 1), (int("8" * 16, 16), 12345)):
        v_, b_, nonce, R, pk, C, cipher = _note(rng, A, B, Gp, v, bl)
        assert len(cipher) == 3 and C == nto.commit(v, bl, Gp)
        assert nto.open_note(a, R, nonce, cipher, C, Gp) == (v, bl)
        assert so.owns(a, B, R, pk) == 1
    _, _, nonce, R, _, C, cipher = _note(rng, A, B, G, 5, 9)     # G' = G: C = [v + blinder] G
    assert C == jo.mul(14, G) and nto.open_note(a, R, nonce, cipher, C, G) == (5, 9)


def test_commitment_is_homomorphic():
    rng, _, _, _, Gp = _wallet(2)
    for _ in range(3):
        v1, v2 = int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 62))
        b1, b2 = jo.random_secret(rng), jo.random_secret(rng)
        assert jo.add(nto.commit(v1, b1, Gp), nto.commit(v2, b2, Gp)) == nto.commit(v1 + v2, (b1 + b2) % N, Gp)


def test_tampered_notes_do_not_open():
    rng, a, A, B, Gp = _wallet(3)
    v, bl, nonce, R, pk, C, cipher = _note(rng, A, B, Gp)
    v2, bl2, nonce2, R2, pk2, C2, cipher2 = _note(rng, A, B, Gp)
    assert nto.open_note(a, R, nonce, cipher, C, Gp) == (v, bl)
    assert nto.open_note(jo.random_secret(rng), R, nonce, cipher, C, Gp) is None          # another view key
    assert nto.open_note(a, R, nonce, cipher, nto.commit(v + 1, bl, Gp), Gp) is None       # C of v + 1
    assert nto.open_note(a, R, nonce, cipher, C2, Gp) is None                             # another note's C
    swapped = ho.encrypt([bl, v], list(jo.mul(a, R)), nonce)                             # m0 and m1 swapped
    assert nto.open_note(a, R, nonce, swapped, C, Gp) is None
    for k in range(3):                                                                    # a cipher element + 1
        bad = list(cipher)
        bad[k] = (bad[k] + 1) % P
        assert nto.open_note(a, R, nonce, bad, C, Gp) is None
    assert nto.open_note(a, R, nonce + 1, cipher, C, Gp) is None                         # nonce + 1
    assert nto.open_note(a, R2, nonce, cipher, C, Gp) is None                            # another note's R


def test_out_of_range_openings_do_not_open_even_when_the_commitment_matches():
    rng, a, A, B, Gp = _wallet(4)
    R = jo.mul(jo.random_secret(rng), G)
    S = list(jo.mul(a, R))
    for m0, m1 in (((1 << 64), 3), (5, N), ((1 << 64) + 7, N + 1)):
        C = jo.add(jo.mul(m0, G), jo.mul(m1, Gp))                       # the commitment of the crafted opening
        cipher = ho.encrypt([m0, m1], S, 11)
        assert nto.decrypt_rows(a, R, 11, cipher) == (m0, m1)
        assert nto.open_note(a, R, 11, cipher, C, Gp) is None
    # [r_J] G' is the identity: (5, r_J) has the commitment of the in-range opening (5, 0), which opens -- the range
    # rule, not the commitment, rejects the crafted one
    C = nto.commit(5, 0, Gp)
    assert jo.add(jo.mul(5, G), jo.mul(N, Gp)) == C
    assert nto.open_note(a, R, 11, ho.encrypt([5, N], S, 11), C, Gp) is None
    assert nto.open_note(a, R, 11, ho.encrypt([5, 0], S, 11), C, Gp) == (5, 0)


def test_invalid_inputs_of_the_model():
    rng, a, A, B, Gp = _wallet(5)
    assert nto.commit(3, N, Gp) is None
    assert nto.create(N, 1, 1, 0, A, B, Gp) is None and nto.create(1, 1, N, 0, A, B, Gp) is None
    assert nto.create(1, 1, 1, 0, jo.off_curve_point(rng), B, Gp) is None
    assert nto.create(1, 1, 1, 0, A, (B[0] + P, B[1]), Gp) is None
    v, bl, nonce, R, pk, C, cipher = _note(rng, A, B, Gp)
    assert nto.open_note(N + a, R, nonce, cipher, C, Gp) is None
    assert nto.open_note(a, jo.off_curve_point(rng), nonce, cipher, C, Gp) is None
    assert not nto.valid_opening(N, R) and not nto.valid_opening(a, (R[0] + P, R[1])) and nto.valid_opening(a, R)


# ---- the 17-window recoding of a u64 ---------------------------------------------------------------------------------
def test_recoding_reconstructs_every_u64():
    rng = np.random.default_rng(6)
    for v in V_EDGES + [int(x) for x in rng.integers(0, 1 << 63, 50, dtype=np.uint64)] + \
            [int(x) | 1 << 63 for x in rng.integers(0, 1 << 63, 50, dtype=np.uint64)]:
        d = nto.recode_u64(v)
        assert len(d) == 17 and all(-8 <= e < 8 for e in d[:16]) and d[16] in (0, 1)
        assert sum(e * 16 ** w for w, e in enumerate(d)) == v
    assert nto.recode_u64((1 << 64) - 1)[16] == 1 and nto.recode_u64(int("7" * 16, 16))[16] == 0
    assert nto.recode_u64(int("8" * 16, 16)) == [-8] + [-7] * 15 + [1]


def test_recoded_walk_equals_double_and_add():
    rng, _, _, _, Gp = _wallet(7)
    for v in (0, 1, 8, 15, int("8" * 16, 16), (1 << 64) - 1, int(rng.integers(0, 1 << 63))):
        assert nto.walk_u64(v, G) == jo.mul(v, G)
    bl = jo.random_secret(rng)
    assert nto.walk_u64(77, G, acc=jo.mul(bl, Gp)) == nto.commit(77, bl, Gp)


def test_product_counts_match_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    for pin in ("kProductsPerValueCommit == 985", "kProductsPerNoteCreateValue == 987", "kProductsPerNoteOpenValue == 568",
                "kValueWindows = 17", "kProductsPerFixedBase == 866"):
        assert pin in src, pin
    assert 64 * 7 + 16 * 7 + 6 + 254 + 163 + 2 == 985 and 64 * 7 + 16 * 7 + 6 + 2 == 568
    assert 2 * 866 > 985                                       # against two fixed-base walks and an addition


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "notes_smoke.c"), os.path.join(ROOT, "tests", "c", "notes_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "notes_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "notes_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "notes.rs")) == [WANT]               # one block, exactly the three functions
    assert "mod notes;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)


def test_c_smoke_calls_exactly_the_notes_block():
    block = _blocks(os.path.join(RUST, "notes.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "notes_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("value_commit", "value_commit_batch", "note_create", "note_create_batch", "note_open", "note_open_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("value_commit_batch", "note_create_batch", "note_open_batch", "last_note_invalid", "last_note_failed"):
        assert callable(getattr(pb.Engine, name))


def test_c_notes_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "NOTES_SMOKE_NO_DEVICE" in res.stdout or "NOTES_SMOKE_OK" in res.stdout


def test_cpp_notes_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "notes mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([G])[0]
    z = np.zeros(4, np.uint64)
    with pytest.raises(pb.EngineError):
        pb.value_commit(3, 5, g, g)
    with pytest.raises(pb.EngineError):
        pb.note_create(3, 5, 7, z, g, g, g, g)
    with pytest.raises(pb.EngineError):
        pb.note_open_batch(jubjub_limbs([3]), g[None], z[None], np.zeros((1, 3, 4), np.uint64), g[None], g, g)
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "NOTES_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
