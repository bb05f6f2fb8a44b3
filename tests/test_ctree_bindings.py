"""The compact sparse tree (p252_ctree) through every front end: the header, the library, the ctypes signature table,
the Rust binding's `extern "C"` block in ctree.rs and the plain-C program that calls exactly that block agree; the C++
CompactTree compiles.  CPU part: compile, link, refusals that need no device, loud failure without a GPU; GPU part
(-m gpu): the same binaries on the device."""
import ctypes
import os
import re
import subprocess

import pytest

import poseidon252_b200 as pb
from poseidon252_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "poseidon252_b200", "lib")
RUST = os.path.join(ROOT, "bindings", "rust", "src")
FN = r"fn\s+(p252_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;"
WANT = {"p252_ctree_layout": 5, "p252_ctree_update": 8, "p252_ctree_open_batch": 6}


def _compile(cmd, src, exe, *flags):
    from poseidon252_b200 import build
    build.build()
    subprocess.check_call([cmd, *flags, "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", LIBDIR, "-lposeidon252_b200", "-Wl,-rpath," + LIBDIR])
    return subprocess.run([exe], input="", capture_output=True, text=True, timeout=120)


def _c():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "ctree_smoke.c"), os.path.join(ROOT, "tests", "c", "ctree_smoke"),
                    "-std=c11")


def _cpp():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "ctree_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "ctree_mirror_test"), "-std=c++17")


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
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "ctree_smoke.c")).read(), flags=re.S)
    return set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    assert {n: hdr[n] for n in hdr if n.startswith("p252_ctree_")} == WANT
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "ctree.rs")) == [WANT]          # one block, exactly the compact-tree functions
    assert not any(n.startswith("p252_ctree_") for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert "mod ctree;" in open(os.path.join(RUST, "lib.rs")).read()
    assert ctypes.sizeof(_native.CTree) == 48


def test_c_smoke_calls_exactly_the_ctree_block():
    block = _blocks(os.path.join(RUST, "ctree.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    called = _c_calls()
    assert {n for n in called if n.startswith("p252_ctree_")} == set(block)
    assert called - set(block) <= set(first)                 # everything else it needs is in the first block of lib.rs


def test_c_ctree_smoke_cpu():
    res = _c()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "CTREE_SMOKE_NO_DEVICE" in res.stdout or "CTREE_SMOKE_OK" in res.stdout


def test_cpp_ctree_mirror_cpu():
    res = _cpp()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "ctree mirror ok (no GPU)" in res.stdout or "root" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.CompactTree(4, 32, 1000)
    res = _c()                                                # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "CTREE_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout


@pytest.mark.gpu
def test_c_ctree_smoke_gpu():
    res = _c()
    assert res.returncode == 0 and "CTREE_SMOKE_OK" in res.stdout, (res.returncode, res.stdout, res.stderr)


@pytest.mark.gpu
def test_cpp_ctree_mirror_gpu():
    res = _cpp()
    assert res.returncode == 0 and "root" in res.stdout, (res.returncode, res.stdout, res.stderr)
