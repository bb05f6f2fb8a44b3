"""Variable-length digest batches (p252_hash_batch_varlen) through every front end: the header, the library, the ctypes
signature table and the Rust binding's third `extern "C"` block agree; a plain-C program calls exactly that block; the
C++ mirror compiles; the Python packing helper.  CPU part: compile, link, host-only checks, loud failure without a GPU;
GPU part (-m gpu): the same binaries on the device."""
import os
import re
import subprocess

import numpy as np
import pytest

import poseidon252_b200 as pb
from poseidon252_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
HEADER = os.path.join(ROOT, "include", "poseidon252_b200.h")


def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=120)


def _c():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "varlen_smoke.c"), os.path.join(ROOT, "tests", "c", "varlen_smoke"),
                    "-std=c11")


def _cpp():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "varlen_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "varlen_mirror_test"), "-std=c++17")


def _header():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {name: (0 if params.strip() in ("", "void") else len(params.split(",")))
            for name, params in re.findall(r"\b(p252_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S)}


def _rust_blocks():
    """every `extern "C"` block of the Rust binding as {name: number of parameters}, in source order"""
    src = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    blocks = [b.split("\n}\n")[0] for b in src.split('extern "C" {')[1:]]
    return [{name: len([p for p in params.split(",") if p.strip()])
             for name, params in re.findall(r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;", b, flags=re.S)}
            for b in blocks]


def _c_calls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "varlen_smoke.c")).read(), flags=re.S)
    return set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    assert hdr["p252_hash_batch_varlen"] == 11
    assert len(_native.SIGNATURES["p252_hash_batch_varlen"][1]) == 11
    assert hasattr(_native.lib(), "p252_hash_batch_varlen")
    m = re.search(r"#define\s+P252_VARLEN_MAX_LEN\s+(\d+)", open(HEADER).read())
    assert m and int(m.group(1)) == _native.VARLEN_MAX_LEN == 65536
    blocks = _rust_blocks()
    assert len(blocks) == 3
    assert blocks[2] == {"p252_hash_batch_varlen": 11}


def test_c_smoke_calls_exactly_the_third_block():
    first, _, third = _rust_blocks()
    called = _c_calls()
    assert {n for n in called if "varlen" in n} == set(third)
    assert called - set(third) <= set(first)          # everything else it needs is in the first block


def test_c_varlen_smoke_cpu():
    res = _c()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "VARLEN_SMOKE_NO_DEVICE" in res.stdout or "VARLEN_SMOKE_OK" in res.stdout


def test_cpp_varlen_mirror_cpu():
    res = _cpp()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "varlen mirror ok" in res.stdout


def test_pack_varlen():
    rng = np.random.default_rng(3)
    items = [rng.integers(0, 1 << 63, (k, 4), dtype=np.uint64) for k in (3, 1, 0, 7, 2)]
    data, offsets, longest = pb.pack_varlen(items)
    assert data.dtype == np.uint64 and data.shape == (13, 4)
    assert offsets.dtype == np.uint64 and list(offsets) == [0, 3, 4, 4, 11, 13]
    assert longest == 7
    for i, a in enumerate(items):
        assert np.array_equal(data[int(offsets[i]):int(offsets[i + 1])], a)
    # flat (k*4,) inputs are read as k scalars; an empty list packs to nothing
    data, offsets, longest = pb.pack_varlen([np.arange(8, dtype=np.uint64)])
    assert data.shape == (2, 4) and list(offsets) == [0, 2] and longest == 2
    data, offsets, longest = pb.pack_varlen([])
    assert data.shape == (0, 4) and list(offsets) == [0] and longest == 0


def test_no_cpu_fallback_without_gpu():
    import ctypes
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.Hash.digest_batch_varlen(pb.Domain.Other, [np.zeros((3, 4), dtype=np.uint64)])


@pytest.mark.gpu
def test_c_varlen_smoke_gpu():
    res = _c()
    assert res.returncode == 0 and "VARLEN_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


@pytest.mark.gpu
def test_cpp_varlen_mirror_gpu():
    res = _cpp()
    assert res.returncode == 0 and "varlen mirror ok (GPU)" in res.stdout, (res.returncode, res.stdout, res.stderr)
