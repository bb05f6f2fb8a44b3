"""JubJub key exchange without a GPU: the curve facts the oracle (jubjub_oracle.py) and the kernel rely on, the oracle's
own consistency, and the bindings of p252_dhke_batch / p252_encrypt_batch_dhke / p252_decrypt_batch_dhke -- the header,
the library, the ctypes signature table and the Rust block in dhke.rs agree, lib.rs keeps its three blocks, the plain-C
program calls exactly the new block, the C and C++ programs compile, and the calls fail loudly without a GPU.
GPU part (-m gpu): the same binaries on the device."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
RUST = os.path.join(ROOT, "bindings", "rust", "src")
FN = r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;"
WANT = {"p252_dhke_batch": 10, "p252_encrypt_batch_dhke": 13, "p252_decrypt_batch_dhke": 13}


# ---- curve facts ---------------------------------------------------------------------------------------------------
def test_constants_match_their_definitions():
    assert jo.D == jo.D_HEX == (-10240 * pow(10241, -1, jo.P)) % jo.P
    assert pow(jo.D, (jo.P - 1) // 2, jo.P) == jo.P - 1                  # d is a non-square: the addition is complete
    assert pow(jo.P - 1, (jo.P - 1) // 2, jo.P) == 1                     # -1 is a square
    assert jo.R_J.bit_length() == 252
    assert all(jo.R_J % q for q in range(2, 20000))                      # no small factor, and Fermat-probable prime:
    assert pow(3, jo.R_J - 1, jo.R_J) == 1 and pow(7, jo.R_J - 1, jo.R_J) == 1
    assert jo.SQRT_M1 * jo.SQRT_M1 % jo.P == jo.P - 1


def test_generator_on_curve_with_prime_order():
    assert jo.on_curve(jo.GENERATOR)
    assert jo.mul(jo.R_J, jo.GENERATOR) == jo.IDENTITY
    assert jo.mul(1, jo.GENERATOR) == jo.GENERATOR and jo.mul(jo.R_J - 1, jo.GENERATOR) == jo.neg(jo.GENERATOR)


def test_cofactor_times_order_kills_random_points():
    rng = np.random.default_rng(1)
    for _ in range(4):
        p = jo.random_point(rng)
        assert jo.on_curve(p) and jo.mul(jo.COFACTOR * jo.R_J, p) == jo.IDENTITY


def test_point_classes():
    rng = np.random.default_rng(2)
    ident, o2, o4a, o4b, o8 = jo.small_order_points(rng)
    assert all(jo.on_curve(p) for p in (ident, o2, o4a, o4b, o8))
    assert jo.add(o2, o2) == ident and o2 != ident
    assert jo.mul(2, o4a) == o2 and jo.mul(4, o4b) == ident
    assert jo.mul(4, o8) != ident and jo.mul(8, o8) == ident
    assert not jo.on_curve(jo.off_curve_point(rng))
    assert not jo.on_curve((jo.GENERATOR[0] + jo.P, jo.GENERATOR[1]))    # u >= p is not a point even if u mod p is


def test_addition_law_matches_definitions():
    rng = np.random.default_rng(3)
    p, q = jo.random_point(rng), jo.random_point(rng)
    assert jo.on_curve(jo.add(p, q)) and jo.add(p, q) == jo.add(q, p)
    assert jo.add(p, jo.neg(p)) == jo.IDENTITY and jo.add(p, jo.IDENTITY) == p
    assert jo.mul(5, p) == jo.add(jo.mul(2, p), jo.mul(3, p))


def test_oracle_dhke_symmetric_and_validity():
    rng = np.random.default_rng(4)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = jo.mul(a, jo.GENERATOR), jo.mul(b, jo.GENERATOR)
    assert jo.dhke(a, B) == jo.dhke(b, A)
    assert jo.dhke(jo.R_J, jo.GENERATOR) is None and jo.dhke(1, jo.off_curve_point(rng)) is None
    assert jo.dhke(0, jo.GENERATOR) == jo.IDENTITY


def test_oracle_round_trip():
    rng = np.random.default_rng(5)
    a, r = jo.random_secret(rng), jo.random_secret(rng)
    pk, R = jo.mul(a, jo.GENERATOR), jo.mul(r, jo.GENERATOR)
    msg = [int(x) for x in rng.integers(0, 1 << 62, 5)]
    nonce = 12345
    cipher = jo.encrypt(msg, r, pk, nonce)               # sender: dhke(r, pk)
    assert jo.decrypt(cipher, a, R, nonce) == msg        # receiver: dhke(a, R)
    with pytest.raises(ho.DecryptionFailed):
        jo.decrypt(cipher, (a + 1) % jo.R_J, R, nonce)


def test_jubjub_limbs():
    v = [0, 1, jo.R_J - 1, (1 << 256) - 1]
    rows = jubjub_limbs(v)
    assert rows.dtype == np.uint64 and rows.shape == (4, 4)
    assert [sum(int(r[k]) << (64 * k) for k in range(4)) for r in rows] == v
    assert np.array_equal(rows, jo.jscalar_limbs(v))
    with pytest.raises(ValueError):
        jubjub_limbs([1 << 256])
    with pytest.raises(ValueError):
        jubjub_limbs([-1])


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "dhke_smoke.c"), os.path.join(ROOT, "tests", "c", "dhke_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "dhke_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "dhke_mirror_test"), "-std=c++17")


def _header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read(), flags=re.S)
    return {name: (0 if params.strip() in ("", "void") else len(params.split(",")))
            for name, params in re.findall(r"\b(p252_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S)}


def _blocks(path):
    """every `extern "C"` block of a Rust source file as {name: number of parameters}, in source order"""
    src = open(path).read()
    return [{name: len([p for p in params.split(",") if p.strip()]) for name, params in re.findall(FN, b, flags=re.S)}
            for b in [b.split("\n}\n")[0] for b in src.split('extern "C" {')[1:]]]


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "dhke.rs")) == [WANT]            # one block, exactly the three functions
    assert "mod dhke;" in open(os.path.join(RUST, "lib.rs")).read()
    hsrc = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    assert re.search(r"typedef struct p252_jscalar \{\s*uint64_t l\[4\];\s*\} p252_jscalar;", hsrc)


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_dhke_block():
    block = _blocks(os.path.join(RUST, "dhke.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "dhke_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if "dhke" in n} == set(block)
    assert called - set(block) <= set(first)


def test_c_dhke_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "DHKE_SMOKE_NO_DEVICE" in res.stdout or "DHKE_SMOKE_OK" in res.stdout


def test_cpp_dhke_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "dhke mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])
    with pytest.raises(pb.EngineError):
        pb.dhke(3, g[0])
    with pytest.raises(pb.EngineError):
        pb.decrypt_batch_dhke(np.zeros((1, 3, 4), dtype=np.uint64), jubjub_limbs([3]), g, np.zeros((1, 4), dtype=np.uint64))
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "DHKE_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout


@pytest.mark.gpu
def test_c_dhke_smoke_gpu():
    res = c_smoke()
    assert res.returncode == 0 and "DHKE_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


@pytest.mark.gpu
def test_cpp_dhke_mirror_gpu():
    res = cpp_mirror()
    assert res.returncode == 0 and "dhke mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
