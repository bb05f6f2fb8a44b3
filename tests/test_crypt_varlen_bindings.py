"""Variable-length encrypt / decrypt batches (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen) through every front
end: the header, the library, the ctypes signature table and the Rust binding's `extern "C"` block in crypt_varlen.rs
agree; lib.rs keeps its three blocks; a plain-C program calls exactly the new block; the C++ mirror compiles; the Python
output-offset helpers.  CPU part: compile, link, host-only checks, loud failure without a GPU; GPU part (-m gpu): the
same binaries on the device."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import poseidon252_b200 as pb
from poseidon252_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
RUST = os.path.join(ROOT, "bindings", "rust", "src")
FN = r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;"
WANT = {"p252_encrypt_batch_varlen": 11, "p252_decrypt_batch_varlen": 13}


def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=120)


def _c():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "crypt_varlen_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "crypt_varlen_smoke"), "-std=c11")


def _cpp():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "crypt_varlen_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "crypt_varlen_mirror_test"), "-std=c++17")


def _header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read(), flags=re.S)
    return {name: (0 if params.strip() in ("", "void") else len(params.split(",")))
            for name, params in re.findall(r"\b(p252_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S)}


def _blocks(path):
    """every `extern "C"` block of a Rust source file as {name: number of parameters}, in source order"""
    src = open(path).read()
    return [{name: len([p for p in params.split(",") if p.strip()]) for name, params in re.findall(FN, b, flags=re.S)}
            for b in [b.split("\n}\n")[0] for b in src.split('extern "C" {')[1:]]]


def _c_calls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "crypt_varlen_smoke.c")).read(), flags=re.S)
    return set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "crypt_varlen.rs")) == [WANT]    # one block, exactly the two functions
    assert "mod crypt_varlen;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_crypt_varlen_block():
    block = _blocks(os.path.join(RUST, "crypt_varlen.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    called = _c_calls()
    assert {n for n in called if "varlen" in n} == set(block)
    assert called - set(block) <= set(first)                 # everything else it needs is in the first block of lib.rs


def test_c_crypt_varlen_smoke_cpu():
    res = _c()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "CRYPT_VARLEN_SMOKE_NO_DEVICE" in res.stdout or "CRYPT_VARLEN_SMOKE_OK" in res.stdout


def test_cpp_crypt_varlen_mirror_cpu():
    res = _cpp()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "crypt varlen mirror ok" in res.stdout


def test_output_offset_helpers():
    offsets = np.array([7, 8, 12, 12, 17, 19], dtype=np.uint64)          # offsets[0] != 0; item 2 is empty
    c = pb.cipher_offsets(offsets)
    assert c.dtype == np.uint64 and list(c) == [0, 2, 7, 8, 14, 17]
    # a cipher CSR maps back to the message CSR packed from 0
    assert list(pb.message_offsets(c)) == [0, 1, 5, 5, 10, 12]
    ciph = np.array([3, 5, 10, 13], dtype=np.uint64)
    assert list(pb.message_offsets(ciph)) == [0, 1, 5, 7]
    # lists are accepted; an empty batch has the single offset 0
    assert list(pb.cipher_offsets([4])) == [0] and list(pb.message_offsets(np.array([9], dtype=np.uint64))) == [0]
    # item-by-item: item i of the output starts at offsets[i] - offsets[0] +- i and is one scalar longer / shorter
    rng = np.random.default_rng(1)
    lens = rng.integers(2, 30, 100)
    off = np.concatenate([[5], 5 + np.cumsum(lens)]).astype(np.uint64)
    co, mo = pb.cipher_offsets(off), pb.message_offsets(off)
    assert np.array_equal(np.diff(co.astype(np.int64)), lens + 1) and np.array_equal(np.diff(mo.astype(np.int64)), lens - 1)
    assert co[0] == 0 and mo[0] == 0
    with pytest.raises(pb.EngineError):
        pb.cipher_offsets(np.zeros(0, dtype=np.uint64))


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.encrypt_batch_varlen([np.zeros((3, 4), dtype=np.uint64)], np.zeros((1, 2, 4), dtype=np.uint64),
                                np.zeros((1, 4), dtype=np.uint64))
    res = _c()                                                # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "CRYPT_VARLEN_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout


@pytest.mark.gpu
def test_c_crypt_varlen_smoke_gpu():
    res = _c()
    assert res.returncode == 0 and "CRYPT_VARLEN_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


@pytest.mark.gpu
def test_cpp_crypt_varlen_mirror_gpu():
    res = _cpp()
    assert res.returncode == 0 and "crypt varlen mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
