"""Schnorr signatures without a GPU: the model of schnorr_oracle.py (round trips and forgeries that must fail), the
kernel's limb arithmetic modulo r_J against big integers (edges, both correction paths, random operands, the constants),
the product counts the kernels pin, and the bindings of p252_schnorr_sign_batch / p252_schnorr_verify_batch -- the
header, the library, the ctypes signature table and the Rust block in schnorr.rs agree, lib.rs keeps its three blocks,
the plain-C program calls exactly the new block, the C and C++ programs compile, and the calls fail loudly without a
GPU.  The same C and C++ programs run on the device in test_gpu_schnorr.py."""
import ctypes
import os
import re

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
import schnorr_oracle as so
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs
from test_stealth_cpu import _blocks, _compile, _header

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST = os.path.join(ROOT, "bindings", "rust", "src")
CUH = os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")
WANT = {"p252_schnorr_sign_batch": 12, "p252_schnorr_verify_batch": 12}
N = jo.R_J


# ---- the model ------------------------------------------------------------------------------------------------------
def test_signatures_verify_and_forgeries_do_not():
    rng = np.random.default_rng(1)
    sk, sk2 = jo.random_secret(rng), jo.random_secret(rng)
    PK, PK2 = so.public_key(sk), so.public_key(sk2)
    for _ in range(3):
        r, m = jo.random_secret(rng), int(rng.integers(0, 1 << 62)) << 190 | 12345
        u, R = so.sign(sk, r, m)
        assert R == jo.mul(r, so.G) and 0 <= u < N
        assert so.verify(PK, u, R, m) == 1
        assert so.verify(PK2, u, R, m) == 0                       # another key
        assert so.verify(jo.neg(PK), u, R, m) == 0                # -PK
        assert so.verify(PK, u, R, (m + 1) % jo.P) == 0           # m + 1
        assert so.verify(PK, (u + 1) % N, R, m) == 0              # u + 1
        assert so.verify(PK, (u - 1) % N, R, m) == 0              # u - 1
        assert so.verify(PK, u, jo.neg(R), m) == 0                # -R
        assert so.verify(PK, u, (R[1], R[0]), m) == 0             # swapped R
    # sk = 0: u = r, and the identity key verifies
    u, R = so.sign(0, 99, 5)
    assert u == 99 and so.verify(jo.IDENTITY, u, R, 5) == 1


def test_challenge_is_a_scalar_below_2_250():
    rng = np.random.default_rng(2)
    for R, m in [(jo.IDENTITY, 0), ((0, 0), jo.P - 1), (jo.GENERATOR, 1), (jo.random_point(rng), 7)]:
        assert 0 <= so.challenge(R, m) < 1 << 250 < N


def test_invalid_inputs_of_the_model():
    rng = np.random.default_rng(3)
    sk = jo.random_secret(rng)
    PK = so.public_key(sk)
    assert so.sign(N, 5, 1) is None and so.sign(sk, N, 1) is None and so.sign(sk, 5, jo.P) is None
    u, R = so.sign(sk, 5, 1)
    assert so.verify(PK, N, R, 1) is None
    assert so.verify(PK, u, R, jo.P) is None
    assert so.verify(PK, u, (R[0] + jo.P, R[1]), 1) is None
    assert so.verify(jo.off_curve_point(rng), u, R, 1) is None
    assert so.verify((PK[0], PK[1] + jo.P), u, R, 1) is None
    assert so.verify(PK, u, jo.off_curve_point(rng), 1) == 0      # canonical R off the curve: simply not verified


# ---- arithmetic modulo r_J: the kernel's limb algorithm --------------------------------------------------------------
def _cuh_words(name):
    src = open(CUH).read()
    m = re.search(r"#define %s \{([^}]*)\}" % name, src)
    return sum(int(w.strip().rstrip("u"), 16) << (32 * k) for k, w in enumerate(m.group(1).split(",")))


def test_constants_are_derived_and_match_the_kernel():
    assert (N * so.ORDER_INV) % (1 << 32) == (1 << 32) - 1            # -r_J^-1 mod 2^32
    assert so.ORDER_R2 == pow(2, 512, N)
    assert _cuh_words("P252_JJ_ORDER") == N
    assert _cuh_words("P252_JJ_ORDER_R2") == so.ORDER_R2
    assert re.search(r"kOrderInv = 0x([0-9a-f]+)u;", open(CUH).read()).group(1) == "%08x" % so.ORDER_INV
    assert N.bit_length() == 252 and (1 << 250) < N


EDGES = [0, 1, 2, N - 1, N - 2, (1 << 250) - 1, 1 << 249, (1 << 251) + 1, N // 2, (N + 1) // 2, 0xffffffff,
         1 << 32, (1 << 224) - 1]


def test_mod_rj_edges():
    for a in EDGES:
        for b in EDGES:
            if a < N and b < N:
                assert so.order_mul(a, b) == a * b % N, (a, b)
                assert so.order_sub(a, b) == (a - b) % N, (a, b)
                assert so.order_mont(a, b) == a * b * pow(1 << 256, -1, N) % N
    assert so.order_sub(0, 0) == 0 and so.order_sub(0, 1) == N - 1 and so.order_sub(N - 1, N - 1) == 0
    assert so.order_mul(N - 1, N - 1) == 1 and so.order_mul(0, N - 1) == 0
    c = (1 << 250) - 1                                               # the largest challenge
    assert so.sign_u(N - 1, N - 1, c) == (N - 1 - c * (N - 1)) % N
    assert so.sign_u(0, 0, c) == 0 and so.sign_u(1, c, c) == 0       # result 0
    assert so.sign_u(1, 0, 1) == N - 1                               # result r_J - 1


def test_mod_rj_both_correction_paths():
    rng = np.random.default_rng(4)
    seen_mont, seen_sub = set(), set()
    for _ in range(2000):
        a, b = jo.random_secret(rng), jo.random_secret(rng)
        tm, ts = [], []
        assert so.order_mul(a, b, tm) == a * b % N
        assert so.order_sub(a, b, ts) == (a - b) % N
        seen_mont.update(tm)
        seen_sub.update(ts)
    assert seen_mont == {True, False} and seen_sub == {True, False}


def test_mod_rj_random():
    rng = np.random.default_rng(5)
    for _ in range(10000):
        sk, r = jo.random_secret(rng), jo.random_secret(rng)
        c = int.from_bytes(rng.integers(0, 256, 32, dtype="uint8").tobytes(), "little") >> 6   # < 2^250
        assert so.sign_u(sk, r, c) == (r - c * sk) % N


# ---- product counts -------------------------------------------------------------------------------------------------
def test_product_counts_match_the_kernel():
    src = open(CUH).read()
    assert "kOrderProductsPerSchnorrSign == 2" in src and "kProductsPerSchnorrVerify == 2850" in src
    # PK check, T and 2d T, table 14 x 9, 62 windows x 36, the last with T 37, [u] G from there 63 x 7 + 6, compare 2
    assert 4 + 2 + 14 * 9 + 62 * 36 + 37 + 63 * 7 + 6 + 2 == 2850


# ---- bindings ------------------------------------------------------------------------------------------------------
def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "schnorr_smoke.c"), os.path.join(ROOT, "tests", "c", "schnorr_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "schnorr_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "schnorr_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "schnorr.rs")) == [WANT]         # one block, exactly the two functions
    assert "mod schnorr;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_schnorr_block():
    block = _blocks(os.path.join(RUST, "schnorr.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "schnorr_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("schnorr_sign", "schnorr_sign_batch", "schnorr_verify", "schnorr_verify_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("schnorr_sign_batch", "schnorr_verify_batch", "last_schnorr_verified", "last_schnorr_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_c_schnorr_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "SCHNORR_SMOKE_NO_DEVICE" in res.stdout or "SCHNORR_SMOKE_OK" in res.stdout


def test_cpp_schnorr_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "schnorr mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])[0]
    m = np.zeros(4, dtype=np.uint64)
    with pytest.raises(pb.EngineError):
        pb.schnorr_sign(3, 5, m, g)
    with pytest.raises(pb.EngineError):
        pb.schnorr_verify(g, 3, g, m, g)
    with pytest.raises(pb.EngineError):
        pb.schnorr_verify_batch(g[None], jubjub_limbs([3]), g[None], m[None], g)
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "SCHNORR_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
