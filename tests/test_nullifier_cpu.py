"""Note nullifiers without a GPU: the model of nullifier_oracle.py against the stealth model (note_sk is the discrete log
of the note's key), its edges (note_sk = 0, the wrap past r_J), the product count the kernel pins, and the bindings of
p252_nullifier_batch -- the header, the library, the ctypes signature table and the Rust block in nullifier.rs agree, the
plain-C program calls exactly the new block, the C and C++ programs compile, and the calls fail loudly without a GPU.
The same C and C++ programs run on the device in test_gpu_nullifier.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import hades_oracle as ho
import jubjub_oracle as jo
import nullifier_oracle as no
import poseidon252_b200 as pb
import stealth_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_stealth_cpu import LIBDIR, ROOT, RUST, _blocks, _header

WANT = {"p252_nullifier_batch": 12}


# ---- the model ------------------------------------------------------------------------------------------------------
def test_note_sk_is_the_discrete_log_of_the_note_key():
    rng = np.random.default_rng(1)
    a, b, a2, b2 = (jo.random_secret(rng) for _ in range(4))
    A, B = so.keys(a, b)
    for _ in range(3):
        R, pk = so.stealth_address(jo.random_secret(rng), A, B)
        assert jo.mul(no.note_sk(a, b, R), jo.GENERATOR) == pk
        assert jo.mul(no.note_sk(a2, b2, R), jo.GENERATOR) != pk        # another receiver's key
        assert jo.mul(no.note_sk(a, b2, R), jo.GENERATOR) != pk


def test_nullifier_is_the_full_digest_of_the_key_and_position():
    rng = np.random.default_rng(2)
    a, b = jo.random_secret(rng), jo.random_secret(rng)
    R, Gp = jo.random_subgroup_point(rng), jo.random_subgroup_point(rng)
    pk = jo.mul(no.note_sk(a, b, R), Gp)
    for pos in (0, 1, 1 << 32, (1 << 64) - 1):
        want = ho.Hash.digest(ho.Domain.Other, [pk[0], pk[1], pos])[0]
        assert no.nullifier(a, b, R, pos, Gp) == want
    assert len({no.nullifier(a, b, R, pos, Gp) for pos in range(4)}) == 4
    assert no.nullifier(a, b, R, 0, Gp) != no.nullifier(a, b, R, 0, jo.GENERATOR)


def test_zero_and_wrapping_note_sk():
    rng = np.random.default_rng(3)
    a, R = jo.random_secret(rng), jo.random_subgroup_point(rng)
    h = so.hash_point(jo.mul(a, R))
    assert 0 <= h < 1 << 250 < jo.R_J
    assert no.note_sk(a, jo.R_J - h, R) == 0                          # pk' = [0] G' = the identity
    want = ho.Hash.digest(ho.Domain.Other, [0, 1, 5])[0]
    assert no.nullifier(a, jo.R_J - h, R, 5, jo.GENERATOR) == want
    assert no.note_sk(a, jo.R_J - 1, R) == h - 1                      # h + b >= r_J wraps
    assert no.note_sk(a, jo.R_J - h + 7, R) == 7


def test_invalid_inputs_of_the_model():
    rng = np.random.default_rng(4)
    a, b, R = jo.random_secret(rng), jo.random_secret(rng), jo.random_subgroup_point(rng)
    G = jo.GENERATOR
    assert no.nullifier(jo.R_J, b, R, 0, G) is None
    assert no.nullifier(a, jo.R_J, R, 0, G) is None
    assert no.nullifier(a, b, jo.off_curve_point(rng), 0, G) is None
    assert no.nullifier(a, b, (R[0] + jo.P, R[1]), 0, G) is None
    assert no.nullifier(a, b, R, 0, G) is not None


def test_product_count_matches_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    assert "kProductsPerNullifierKey == 867" in src and "kProductsPerFixedBase == 866" in src
    assert 63 * 7 + 6 + 254 + 163 + 2 + 1 == 867                     # fixed-base walk, inversion, affine, Montgomery(pos)


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "nullifier_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "nullifier_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "nullifier_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "nullifier_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "nullifier.rs")) == [WANT]       # one block, exactly the one function
    assert "mod nullifier;" in open(os.path.join(RUST, "lib.rs")).read()
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)


def test_c_smoke_calls_exactly_the_nullifier_block():
    import re
    block = _blocks(os.path.join(RUST, "nullifier.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "nullifier_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("nullifier", "nullifier_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("nullifier_batch", "last_nullifier_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_c_nullifier_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "NULLIFIER_SMOKE_NO_DEVICE" in res.stdout or "NULLIFIER_SMOKE_OK" in res.stdout


def test_cpp_nullifier_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "nullifier mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])[0]
    with pytest.raises(pb.EngineError):
        pb.nullifier(3, 5, g, g, 7)
    with pytest.raises(pb.EngineError):
        pb.nullifier_batch(jubjub_limbs([3]), jubjub_limbs([5]), g, g[None], np.zeros(1, np.uint64))
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "NULLIFIER_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
