"""Double-key Schnorr signatures without a GPU: the model of schnorr_double_oracle.py (round trips, forgeries that must
fail, the note key against the stealth model), the product counts the kernels pin, and the bindings of
p252_schnorr_sign_double_batch / p252_schnorr_verify_double_batch / p252_note_sign_double_batch -- the header, the library,
the ctypes signature table and the Rust block in schnorr_double.rs agree, the plain-C program calls exactly the new block,
the C and C++ programs compile, and the calls fail loudly without a GPU.  The same C and C++ programs run on the device
in test_gpu_schnorr_double.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import jubjub_oracle as jo
import nullifier_oracle as no
import poseidon252_b200 as pb
import schnorr_double_oracle as sdo
import schnorr_oracle as so1
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_stealth_cpu import LIBDIR, ROOT, RUST, _blocks, _header

WANT = {"p252_schnorr_sign_double_batch": 14, "p252_schnorr_verify_double_batch": 15, "p252_note_sign_double_batch": 17}
N, P, G = jo.R_J, jo.P, jo.GENERATOR


def _setup(seed):
    rng = np.random.default_rng(seed)
    Gp = jo.random_subgroup_point(rng)
    sk = jo.random_secret(rng)
    return rng, Gp, sk, sdo.key_pair(sk, Gp)


# ---- the model ------------------------------------------------------------------------------------------------------
def test_round_trips():
    rng, Gp, sk, (pk, pkp) = _setup(1)
    for m in (0, 1, P - 1, int(rng.integers(0, 1 << 62))):
        u, R, Rp = sdo.sign_double(sk, jo.random_secret(rng), m, Gp)
        assert sdo.verify_double(pk, pkp, u, R, Rp, m, Gp) == 1
    for sk2, r in ((0, 5), (1, 0), (N - 1, N - 1)):               # edge keys and nonces
        pk2, pkp2 = sdo.key_pair(sk2, Gp)
        u, R, Rp = sdo.sign_double(sk2, r, 7, Gp)
        assert sdo.verify_double(pk2, pkp2, u, R, Rp, 7, Gp) == 1
    u, R, Rp = sdo.sign_double(sk, 9, 3, G)                       # G' = G: R == R', and the two checks are the same
    assert R == Rp and sdo.verify_double(pk, pk, u, R, Rp, 3, G) == 1


def test_forgeries_fail():
    rng, Gp, sk, (pk, pkp) = _setup(2)
    m, r = 12345, jo.random_secret(rng)
    u, R, Rp = sdo.sign_double(sk, r, m, Gp)
    v = lambda *a: sdo.verify_double(*a, Gp)                     # noqa: E731
    assert v(pk, pkp, u, R, Rp, m) == 1
    # one-sided: a valid single-key (u, R) with a wrong R' -- and the single-key check alone would pass
    R2 = jo.mul(r + 1, Gp)
    assert v(pk, pkp, u, R, R2, m) == 0
    # PK' of another key, [sk + 1] G'
    assert v(pk, jo.mul(sk + 1, Gp), u, R, Rp, m) == 0
    assert v(pk, pkp, u, Rp, R, m) == 0                          # swapped R / R'
    assert v(pk, pkp, (u + 1) % N, R, Rp, m) == 0                # u +- 1
    assert v(pk, pkp, (u - 1) % N, R, Rp, m) == 0
    assert v(pk, pkp, u, R, Rp, m + 1) == 0                      # m + 1
    assert v(pk, pk, u, R, Rp, m) == 0                           # PK' replaced by PK
    assert v(pkp, pkp, u, R, Rp, m) == 0
    # a signature with the same r over (R, R') is not one over G alone: the challenges differ
    u1, R1 = so1.sign(sk, r, m)
    assert R1 == R and u1 != u and v(pk, pkp, u1, R, Rp, m) == 0


def test_challenge_covers_every_row_element():
    rng, Gp, sk, _ = _setup(3)
    R, Rp = jo.mul(5, G), jo.mul(5, Gp)
    c = sdo.challenge2(R, Rp, 9)
    assert 0 <= c < 1 << 250
    assert len({c, sdo.challenge2(Rp, R, 9), sdo.challenge2(R, R, 9), sdo.challenge2(R, Rp, 10),
                so1.challenge(R, 9)}) == 5


def test_invalid_inputs_of_the_model():
    rng, Gp, sk, (pk, pkp) = _setup(4)
    assert sdo.sign_double(N, 1, 0, Gp) is None and sdo.sign_double(1, N, 0, Gp) is None
    assert sdo.sign_double(1, 1, P, Gp) is None
    u, R, Rp = sdo.sign_double(sk, 3, 4, Gp)
    assert sdo.verify_double(pk, pkp, N + u, R, Rp, 4, Gp) is None
    assert sdo.verify_double(pk, pkp, u, R, Rp, P, Gp) is None
    assert sdo.verify_double(pk, pkp, u, (R[0] + P, R[1]), Rp, 4, Gp) is None
    assert sdo.verify_double(pk, pkp, u, R, (Rp[0], Rp[1] + P), 4, Gp) is None
    assert sdo.verify_double(jo.off_curve_point(rng), pkp, u, R, Rp, 4, Gp) is None
    assert sdo.verify_double(pk, jo.off_curve_point(rng), u, R, Rp, 4, Gp) is None
    R_note = jo.random_subgroup_point(rng)
    assert sdo.note_sign_double(N, 1, R_note, 1, 0, Gp) is None
    assert sdo.note_sign_double(1, N, R_note, 1, 0, Gp) is None
    assert sdo.note_sign_double(1, 1, jo.off_curve_point(rng), 1, 0, Gp) is None
    assert sdo.note_sign_double(1, 1, R_note, N, 0, Gp) is None
    assert sdo.note_sign_double(1, 1, R_note, 1, P, Gp) is None


def test_torsion_in_pk_prime_is_not_checked_away():
    """no subgroup check: PK' shifted by a small-order point T is on the curve, so the item is valid and does not verify"""
    rng, Gp, sk, (pk, pkp) = _setup(5)
    u, R, Rp = sdo.sign_double(sk, 11, 2, Gp)
    T = jo.order8_point(rng)
    shifted = jo.add(pkp, T)
    assert jo.on_curve(shifted) and sdo.verify_double(pk, shifted, u, R, Rp, 2, Gp) == 0


def test_note_key_signs_for_the_stealth_note_key():
    """[note_sk] G is stealth_address's note_pk, and [note_sk] G' is the point the nullifier hashes"""
    rng = np.random.default_rng(6)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    Gp = jo.random_subgroup_point(rng)
    for _ in range(2):
        R_note, note_pk = so.stealth_address(jo.random_secret(rng), A, B)
        (u, R, Rp), pkp = sdo.note_sign_double(a, b, R_note, jo.random_secret(rng), 77, Gp)
        assert jo.mul(no.note_sk(a, b, R_note), G) == note_pk
        assert pkp == jo.mul(no.note_sk(a, b, R_note), Gp)
        assert sdo.verify_double(note_pk, pkp, u, R, Rp, 77, Gp) == 1
        import hades_oracle as ho
        assert no.nullifier(a, b, R_note, 3, Gp) == ho.Hash.digest(ho.Domain.Other, [pkp[0], pkp[1], 3])[0]
        a2 = jo.random_secret(rng)                               # another wallet's key signs for another key
        (u2, R2, Rp2), pkp2 = sdo.note_sign_double(a2, b, R_note, 5, 77, Gp)
        assert sdo.verify_double(note_pk, pkp, u2, R2, Rp2, 77, Gp) == 0


def test_product_counts_match_the_kernels():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    for pin in ("kProductsPerSchnorrSignDouble == 1732", "kProductsPerNoteSignDouble == 5417",
                "kProductsPerSchnorrVerifyDouble == 5700", "kProductsPerSchnorrVerify == 2850",
                "kProductsPerFixedBase == 866", "kProductsPerDhke == 2819", "kOrderProductsPerSchnorrSign == 2"):
        assert pin in src, pin
    assert 2 * 866 == 1732 and 1732 + 2819 + 866 == 5417 and 2 * 2850 == 5700


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "schnorr_double_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "schnorr_double_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "schnorr_double_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "schnorr_double_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "schnorr_double.rs")) == [WANT]    # one block, exactly the three functions
    assert "mod schnorr_double;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "schnorr.rs")) for n in b)


def test_c_smoke_calls_exactly_the_schnorr_double_block():
    block = _blocks(os.path.join(RUST, "schnorr_double.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "schnorr_double_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("schnorr_sign_double", "schnorr_sign_double_batch", "schnorr_verify_double", "schnorr_verify_double_batch",
                 "note_sign_double_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("schnorr_sign_double_batch", "schnorr_verify_double_batch", "note_sign_double_batch",
                 "last_schnorr_double_verified", "last_schnorr_double_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_c_schnorr_double_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "SCHNORR_DOUBLE_SMOKE_NO_DEVICE" in res.stdout or "SCHNORR_DOUBLE_SMOKE_OK" in res.stdout


def test_cpp_schnorr_double_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "schnorr double mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([G])[0]
    m = np.zeros(4, np.uint64)
    with pytest.raises(pb.EngineError):
        pb.schnorr_sign_double(3, 5, m, g, g)
    with pytest.raises(pb.EngineError):
        pb.schnorr_verify_double(g, g, 3, g, g, m, g, g)
    with pytest.raises(pb.EngineError):
        pb.note_sign_double_batch(jubjub_limbs([3]), jubjub_limbs([5]), g[None], jubjub_limbs([7]), m[None], g, g)
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "SCHNORR_DOUBLE_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
