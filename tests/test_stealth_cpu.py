"""Stealth addresses without a GPU: the model of stealth_oracle.py (round trips, the identity note, the hash range), the
product counts the kernel pins, and the bindings of p252_stealth_address_batch / p252_stealth_owns_batch -- the header, the
library, the ctypes signature table and the Rust block in stealth.rs agree, lib.rs keeps its three blocks, the plain-C
program calls exactly the new block, the C and C++ programs compile, and the calls fail loudly without a GPU.
The same C and C++ programs run on the device in test_gpu_stealth.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
RUST = os.path.join(ROOT, "bindings", "rust", "src")
FN = r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;"
WANT = {"p252_stealth_address_batch": 12, "p252_stealth_owns_batch": 11}


# ---- the model ------------------------------------------------------------------------------------------------------
def test_receiver_owns_its_notes_and_no_other_receiver_does():
    rng = np.random.default_rng(1)
    a, b, a2, b2 = (jo.random_secret(rng) for _ in range(4))
    A, B = so.keys(a, b)
    A2, B2 = so.keys(a2, b2)
    for _ in range(3):
        r = jo.random_secret(rng)
        R, pk = so.stealth_address(r, A, B)
        assert jo.mul(r, A) == jo.mul(a, R)                       # the shared point both sides derive
        assert jo.on_curve(pk) and so.owns(a, B, R, pk) == 1
        assert so.owns(a2, B2, R, pk) == 0 and so.owns(a2, B, R, pk) == 0 and so.owns(a, B2, R, pk) == 0
        assert so.owns(a, B, jo.neg(R), pk) == 0
        assert so.owns(a, B, R, (pk[1], pk[0])) == 0


def test_hash_is_a_scalar_below_2_250():
    rng = np.random.default_rng(2)
    for pt in [jo.IDENTITY, (0, 0), jo.GENERATOR, jo.random_point(rng)]:
        h = so.hash_point(pt)
        assert 0 <= h < 1 << 250 < jo.R_J


def test_minus_hG_spend_key_gives_the_identity_note():
    rng = np.random.default_rng(3)
    a, r = jo.random_secret(rng), jo.random_secret(rng)
    A = jo.mul(a, jo.GENERATOR)
    B = jo.neg(jo.mul(so.hash_point(jo.mul(r, A)), jo.GENERATOR))
    R, pk = so.stealth_address(r, A, B)
    assert pk == jo.IDENTITY and so.owns(a, B, R, pk) == 1


def test_invalid_inputs_of_the_model():
    rng = np.random.default_rng(4)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    A, B = so.keys(a, b)
    assert so.stealth_address(jo.R_J, A, B) is None
    assert so.stealth_address(5, jo.off_curve_point(rng), B) is None
    assert so.stealth_address(5, A, (B[0] + jo.P, B[1])) is None
    R, pk = so.stealth_address(5, A, B)
    assert so.owns(jo.R_J, B, R, pk) is None
    assert so.owns(a, B, (R[0], R[1] + jo.P), pk) is None
    assert so.owns(a, B, R, (pk[0] + jo.P, pk[1])) is None
    assert so.owns(a, B, R, jo.off_curve_point(rng)) == 0      # canonical but off the curve: simply not owned


def test_product_counts_match_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    assert "kProductsPerStealthOwns == 456" in src and "kProductsPerStealthDerive == 879" in src
    assert 64 * 7 + 6 + 2 == 456                                   # [h] G with T, + B, projective compare
    assert 4 + 2 + 64 * 7 + 6 + 254 + 163 + 2 == 879               # B check and Niels form, [h] G + B, inversion, affine


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "stealth_smoke.c"), os.path.join(ROOT, "tests", "c", "stealth_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "stealth_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "stealth_mirror_test"), "-std=c++17")


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
    assert _blocks(os.path.join(RUST, "stealth.rs")) == [WANT]         # one block, exactly the two functions
    assert "mod stealth;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_stealth_block():
    block = _blocks(os.path.join(RUST, "stealth.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "stealth_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("stealth_address", "stealth_address_batch", "owns", "stealth_owns_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("stealth_address_batch", "stealth_owns_batch", "last_stealth_owned", "last_stealth_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_c_stealth_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "STEALTH_SMOKE_NO_DEVICE" in res.stdout or "STEALTH_SMOKE_OK" in res.stdout


def test_cpp_stealth_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "stealth mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])[0]
    with pytest.raises(pb.EngineError):
        pb.stealth_address(3, g, g, g)
    with pytest.raises(pb.EngineError):
        pb.owns(3, g, g, g, g)
    with pytest.raises(pb.EngineError):
        pb.stealth_owns_batch(jubjub_limbs([3]), g, g, g[None], g[None])
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "STEALTH_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
