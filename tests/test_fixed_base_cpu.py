"""Fixed-base JubJub scalar multiplication without a GPU: a Python model of the kernel's signed 4-bit recoding and of its
table-driven product (jubjub_device.cuh, fixed_base_mul), checked against the double-and-add of jubjub_oracle.py, and the
bindings of p252_fixed_base_batch / p252_encrypt_batch_ephemeral -- the header, the library, the ctypes signature table
and the Rust block in fixed_base.rs agree, lib.rs keeps its three blocks, the plain-C program calls exactly the new block,
the C and C++ programs compile, and the calls fail loudly without a GPU.
GPU part (-m gpu): the same binaries on the device."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.scalar import jubjub_limbs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
RUST = os.path.join(ROOT, "bindings", "rust", "src")
FN = r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;"
WANT = {"p252_fixed_base_batch": 8, "p252_encrypt_batch_ephemeral": 14}
WINDOWS = 64

# scalars whose recoding exercises every digit value, every carry chain and both ends of [0, r_J)
EDGE_SCALARS = ([0, 1, 7, 8, 9, 15, 16, 17, 0x77777777777777777777777777777777777777777777777777777777777777,
                 0x88888888888888888888888888888888888888888888888888888888888888,
                 jo.R_J - 1,
                 (1 << 251) + 1, (1 << 251) + 0x8888, int("8" * 62, 16), int("f" * 62, 16) % jo.R_J,
                 jo.R_J - 8, jo.R_J - 9, jo.R_J >> 1, 1 << 250, (1 << 248) - 1]
                + [(1 << (4 * k)) - 8 for k in range(2, 63, 7)]      # 0xf...f8: a carry through every lower digit
                + [8 << (4 * k) for k in range(0, 63, 9)])


def recode(s):
    """The kernel's recoding (recode_digit): 64 digits in [-8, 8), least significant first."""
    digits, carry = [], 0
    for _ in range(WINDOWS):
        x = (s & 15) + carry
        s >>= 4
        carry = (x + 8) >> 4
        digits.append(x - (carry << 4))
    assert s == 0 and carry == 0
    return digits


def table(base):
    """Entry (w, j) = j 16^w base, j = 1..8, as affine points (the kernel stores them in Niels form)."""
    tab = []
    q = base
    for _ in range(WINDOWS):
        row = [q]
        for _ in range(7):
            row.append(jo.add(row[-1], q))
        tab.append(row)
        q = jo.mul(16, q)
    return tab


def niels(pt):
    u, v = pt
    return ((v - u) % jo.P, (v + u) % jo.P, 2 * jo.D * u * v % jo.P)


def niels_to_affine(n):
    ymx, ypx, _ = n
    inv2 = pow(2, -1, jo.P)
    return ((ypx - ymx) * inv2 % jo.P, (ypx + ymx) * inv2 % jo.P)


def fixed_base_model(s, tab):
    """sum_w sign(e_w) (|e_w| 16^w B): the select (identity for 0), the masked negation (swap the first two Niels
    coordinates, negate the third) and the addition, in the kernel's window order."""
    acc = jo.IDENTITY
    for w, e in enumerate(recode(s)):
        m = abs(e)
        n = (1, 1, 0) if m == 0 else niels(tab[w][m - 1])
        if e < 0:
            n = (n[1], n[0], (-n[2]) % jo.P)
        acc = jo.add(acc, niels_to_affine(n))
    return acc


def test_recoding_reconstructs_the_scalar():
    rng = np.random.default_rng(1)
    scalars = EDGE_SCALARS + [jo.random_secret(rng) for _ in range(200)]
    for s in scalars:
        assert 0 <= s < jo.R_J < 1 << 252
        d = recode(s)
        assert len(d) == WINDOWS and all(-8 <= x < 8 for x in d) and d[-1] in (0, 1)
        assert sum(x << (4 * w) for w, x in enumerate(d)) == s
    # every digit value is reached, and a long carry chain ends in the top window
    assert {x for s in scalars for x in recode(s)} == set(range(-8, 8))
    assert recode(int("8" * 63, 16))[-1] == 1


def test_identity_and_negation_in_niels_form():
    rng = np.random.default_rng(2)
    p = jo.random_point(rng)
    assert niels_to_affine((1, 1, 0)) == jo.IDENTITY
    n = niels(p)
    assert niels_to_affine((n[1], n[0], (-n[2]) % jo.P)) == jo.neg(p) and niels(jo.neg(p))[2] == (-n[2]) % jo.P


@pytest.mark.parametrize("which", ["generator", "subgroup", "full", "order8", "order4", "order2", "identity"])
def test_model_product_matches_oracle(which):
    rng = np.random.default_rng(3)
    ident, o2, o4, _, o8 = jo.small_order_points(rng)
    base = {"generator": jo.GENERATOR, "subgroup": jo.random_subgroup_point(rng), "full": jo.random_point(rng),
            "order8": o8, "order4": o4, "order2": o2, "identity": ident}[which]
    tab = table(base)
    scalars = EDGE_SCALARS if which in ("generator", "full") else EDGE_SCALARS[::3]
    for s in scalars + [jo.random_secret(rng) for _ in range(3)]:
        assert fixed_base_model(s, tab) == jo.mul(s, base), hex(s)


def test_table_size_and_product_count_match_the_kernel():
    src = open(os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")).read()
    assert "kProductsPerFixedBase == 866" in src
    assert (WINDOWS - 1) * 7 + 6 + 254 + 163 + 2 == 866                 # madd 7 / 6, inversion, affine
    assert "kFixedBaseTableBytes = 64 * 8 * 96" in open(os.path.join(ROOT, "poseidon252_b200", "csrc", "kernels.h")).read()


# ---- bindings ------------------------------------------------------------------------------------------------------
def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=300)


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "fixed_base_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "fixed_base_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "fixed_base_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "fixed_base_mirror_test"), "-std=c++17")


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
    assert _blocks(os.path.join(RUST, "fixed_base.rs")) == [WANT]      # one block, exactly the two functions
    assert "mod fixed_base;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_fixed_base_block():
    block = _blocks(os.path.join(RUST, "fixed_base.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "fixed_base_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_c_fixed_base_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "FIXED_BASE_SMOKE_NO_DEVICE" in res.stdout or "FIXED_BASE_SMOKE_OK" in res.stdout


def test_cpp_fixed_base_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "fixed_base mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])[0]
    with pytest.raises(pb.EngineError):
        pb.fixed_base(3, g)
    with pytest.raises(pb.EngineError):
        pb.encrypt_batch_ephemeral(np.zeros((1, 2, 4), dtype=np.uint64), jubjub_limbs([3]), g, g[None],
                                   np.zeros((1, 4), dtype=np.uint64))
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "FIXED_BASE_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout


@pytest.mark.gpu
def test_c_fixed_base_smoke_gpu():
    res = c_smoke()
    assert res.returncode == 0 and "FIXED_BASE_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


@pytest.mark.gpu
def test_cpp_fixed_base_mirror_gpu():
    res = cpp_mirror()
    assert res.returncode == 0 and "fixed_base mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
