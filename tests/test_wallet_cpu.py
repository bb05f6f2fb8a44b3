"""Wallet scans without a GPU: the model of wallet_oracle.py (notes created for several keys are found by their key,
duplicate keys resolve to the smallest index, bad keys and invalid notes), the product counts the kernels pin, and the
bindings of p252_wallet_scan_batch -- the header, the library, the ctypes signature table and the Rust block in wallet.rs
agree, the plain-C program calls exactly the new block, the C and C++ programs compile, and the call fails loudly
without a GPU.  The same C and C++ programs run on the device in test_gpu_wallet.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import jubjub_oracle as jo
import note_oracle as nto
import nullifier_oracle as nuo
import poseidon252_b200 as pb
import stealth_oracle as so
import wallet_oracle as wo
from poseidon252_b200 import _native
from test_stealth_cpu import LIBDIR, ROOT, RUST, _blocks, _header

WANT = {"p252_wallet_scan_batch": 22}
N, P, G = jo.R_J, jo.P, jo.GENERATOR


def _note(rng, a, b, Gp, v, pos):
    A, B = so.keys(a, b)
    bl, nonce = jo.random_secret(rng), int(rng.integers(0, 1 << 62))
    R, pk, C, cipher = nto.create(jo.random_secret(rng), v, bl, nonce, A, B, Gp)
    return (R, pk, pos, nonce, cipher, C), bl


# ---- the model ------------------------------------------------------------------------------------------------------
def test_notes_of_several_keys_round_trip():
    rng = np.random.default_rng(1)
    Gp = jo.random_subgroup_point(rng)
    keys = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(3)]
    notes, want = [], []
    for i, (j, v) in enumerate(((0, 5), (2, 7), (1, 1 << 63), (2, (1 << 64) - 1), (2, (1 << 64) - 1))):
        note, bl = _note(rng, *keys[j], Gp, v, 100 + i)
        notes.append(note)
        want.append((j, v, bl))
    stranger, _ = _note(rng, jo.random_secret(rng), jo.random_secret(rng), Gp, 9, 7)
    notes.append(stranger)
    out = wo.scan(keys, notes, Gp)
    assert out["owner"] == [w[0] for w in want] + [-1]
    for i, (j, v, bl) in enumerate(want):
        assert out["opened"][i] == 1 and out["value"][i] == v and out["blinder"][i] == bl
        assert out["nullifier"][i] == nuo.nullifier(*keys[j], notes[i][0], notes[i][2], Gp)
    assert out["opened"][-1] == 0 and out["nullifier"][-1] is None and out["value"][-1] == 0
    s2 = 7 + 2 * ((1 << 64) - 1)
    assert out["totals"] == [[5, 0, 1, 1], [1 << 63, 0, 1, 1], [s2 & ((1 << 64) - 1), s2 >> 64, 3, 3]]
    assert out["n_invalid"] == 0 and out["n_bad_keys"] == 0


def test_duplicate_keys_resolve_to_the_smallest_index():
    rng = np.random.default_rng(2)
    Gp = jo.random_subgroup_point(rng)
    k = (jo.random_secret(rng), jo.random_secret(rng))
    other = (jo.random_secret(rng), jo.random_secret(rng))
    note, _ = _note(rng, *k, Gp, 3, 0)
    assert wo.scan([other, k, k], [note], Gp)["owner"] == [1]
    # the same spend key with another view key does not own the note
    assert wo.scan([(other[0], k[1]), k], [note], Gp)["owner"] == [1]


def test_bad_keys_and_invalid_notes():
    rng = np.random.default_rng(3)
    Gp = jo.random_subgroup_point(rng)
    k = (jo.random_secret(rng), jo.random_secret(rng))
    note, _ = _note(rng, *k, Gp, 3, 0)
    out = wo.scan([(k[0] + N, k[1]), (k[0], k[1] + N), k], [note], Gp)
    assert out["owner"] == [2] and out["n_bad_keys"] == 2
    R, pk, pos, nonce, cipher, C = note
    for bad in ((jo.off_curve_point(rng), pk), ((R[0] + P, R[1]), pk), (R, (pk[0], pk[1] + P))):
        out = wo.scan([k], [(bad[0], bad[1], pos, nonce, cipher, C)], Gp)
        assert out["owner"] == [-1] and out["n_invalid"] == 1 and out["totals"] == [[0, 0, 0, 0]]
    out = wo.scan([k], [(R, jo.off_curve_point(rng), pos, nonce, cipher, C)], Gp)     # canonical, off the curve
    assert out["owner"] == [-1] and out["n_invalid"] == 0


def test_owned_notes_that_do_not_open_keep_owner_and_nullifier():
    rng = np.random.default_rng(4)
    Gp = jo.random_subgroup_point(rng)
    k = (jo.random_secret(rng), jo.random_secret(rng))
    (R, pk, pos, nonce, cipher, C), _ = _note(rng, *k, Gp, 3, 5)
    tampered = [cipher[0], (cipher[1] + 1) % P, cipher[2]]
    out = wo.scan([k], [(R, pk, pos, nonce, tampered, C), (R, pk, pos, nonce, cipher, nto.commit(4, 1, Gp))], Gp)
    assert out["owner"] == [0, 0] and out["opened"] == [0, 0] and out["value"] == [0, 0]
    assert out["nullifier"] == [nuo.nullifier(*k, R, pos, Gp)] * 2
    assert out["totals"] == [[0, 0, 2, 0]]


def test_product_counts_match_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    for pin in ("kProductsPerWalletKey == 868", "kProductsPerWalletPair == 3275", "kProductsPerWalletOwned == 1435",
                "kProductsPerWalletSelect = 4", "kProductsPerDhke == 2819", "kProductsPerStealthOwns == 456",
                "kProductsPerNullifierKey == 867", "kProductsPerNoteOpenValue == 568"):
        assert pin in src, pin
    perm = 365                                                     # Montgomery products per Hades permutation
    assert 2819 + perm + 456 == 3640                               # a pair, with the hash of [a_j] R_i
    assert 867 + perm + 2 * perm + 568 == 2530                     # an owned note: nullifier digest, decryption at L = 2


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "wallet_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "wallet_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "wallet_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "wallet_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "wallet.rs")) == [WANT]
    assert "mod wallet;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    assert "#define P252_WALLET_MAX_KEYS 256" in src and pb.Engine.WALLET_MAX_KEYS == 256
    assert "pub const WALLET_MAX_KEYS: usize = 256;" in open(os.path.join(RUST, "wallet.rs")).read()


def test_c_smoke_calls_exactly_the_wallet_block():
    block = _blocks(os.path.join(RUST, "wallet.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "wallet_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    assert "wallet_scan_batch" in pb.__all__ and callable(pb.wallet_scan_batch)
    for name in ("wallet_scan_batch", "last_wallet_invalid", "last_wallet_bad_keys"):
        assert callable(getattr(pb.Engine, name))


def test_c_wallet_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "WALLET_SMOKE_NO_DEVICE" in res.stdout or "WALLET_SMOKE_OK" in res.stdout


def test_cpp_wallet_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "wallet mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([G])[0]
    z = np.zeros((1, 4), np.uint64)
    with pytest.raises(pb.EngineError):
        pb.wallet_scan_batch(z + 1, z + 1, g[None], g[None], np.zeros(1, np.uint64), z, np.zeros((1, 3, 4), np.uint64),
                             g[None], g, g)
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "WALLET_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
