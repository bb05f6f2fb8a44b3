"""Mixed digest batches without a GPU: the bindings of p252_hash_batch_mixed -- the header, the library, the ctypes
signature table, the Rust block in hash_mixed.rs and the plain-C program agree, lib.rs keeps its three blocks, the C and
C++ programs compile with -Wall -Werror -- Hash.finalize_batch's refusals, which need no device, and the absence of a CPU
fallback.  The same C and C++ programs run on the device in test_gpu_hash_mixed.py."""
import ctypes
import os
import re

import numpy as np
import pytest

import poseidon252_b200 as pb
from poseidon252_b200 import _native
from test_notes_cpu import _compile
from test_stealth_cpu import RUST, ROOT, _blocks, _header

WANT = {"p252_hash_batch_mixed": 13}
INVALID_ARGUMENT = -1                                             # P252_ERR_INVALID_ARGUMENT


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "hash_mixed_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "hash_mixed_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "hash_mixed_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "hash_mixed_mirror_test"), "-std=c++17")


# ---- bindings --------------------------------------------------------------------------------------------------------
def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "hash_mixed.rs")) == [WANT]          # one block, exactly the function
    assert "mod hash_mixed;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    assert re.search(r"#define P252_MIXED_TRUNCATED 0x80\b", src)
    assert _native.MIXED_TRUNCATED == 0x80
    assert "pub const MIXED_TRUNCATED: u8 = 0x80;" in open(os.path.join(RUST, "hash_mixed.rs")).read()


def test_c_smoke_calls_exactly_the_hash_mixed_block():
    block = _blocks(os.path.join(RUST, "hash_mixed.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "hash_mixed_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("finalize_batch", "digest_batch_mixed"):
        assert name in pb.__all__ and callable(getattr(pb, name))
        assert getattr(pb, name) is getattr(pb.Hash, name)
    for name in ("hash_batch_mixed", "last_mixed_rejected"):
        assert callable(getattr(pb.Engine, name))


def test_c_hash_mixed_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "HASH_MIXED_SMOKE_NO_DEVICE" in res.stdout or "HASH_MIXED_SMOKE_OK" in res.stdout


def test_cpp_hash_mixed_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "hash_mixed mirror ok" in res.stdout


# ---- refusals that need no device ----------------------------------------------------------------------------------
def _hash(domain, *chunks, out_len=1):
    h = pb.Hash(domain)
    h.output_len(out_len)
    for c in chunks:
        h.update(np.arange(4 * c, dtype=np.uint64).reshape(c, 4))
    return h


class _NoEngine:
    """an engine that fails the test if finalize_batch reaches it"""

    def __getattr__(self, name):
        raise AssertionError("finalize_batch touched the engine (%s)" % name)


def test_finalize_batch_raises_for_the_lowest_index_bad_hash_without_a_device():
    good = [_hash(pb.Domain.Other, 2, 3, out_len=4), _hash(pb.Domain.Merkle4, 1, 3),
            _hash(pb.Domain.Merkle2, 1, 1, out_len=3)]                         # output_len is ignored for Merkle2
    cases = [
        ([_hash(pb.Domain.Merkle4, 3)], pb.IOPatternViolation),                      # arity
        ([_hash(pb.Domain.Other, 2, 0, 1)], pb.InvalidIOPattern),                     # a zero-length chunk
        ([_hash(pb.Domain.Other)], pb.InvalidIOPattern),                              # no input
        ([_hash(pb.Domain.Merkle4, 0, 4)], pb.InvalidIOPattern),                      # arity met, zero-length chunk
        ([_hash(pb.Domain.Merkle4, 0, 3), _hash(pb.Domain.Other, 0)], pb.IOPatternViolation),
        ([_hash(pb.Domain.Other, 0), _hash(pb.Domain.Merkle4, 5)], pb.InvalidIOPattern),
    ]
    for bad, exc in cases:
        with pytest.raises(exc):
            pb.Hash.finalize_batch(good + bad + good, truncated=True, engine=_NoEngine())
        with pytest.raises(exc):                                               # what Hash.finalize raises for it
            bad[0].finalize()
    with pytest.raises(ValueError):
        pb.Hash.finalize_batch(good, truncated=[True], engine=_NoEngine())
    assert pb.Hash.finalize_batch([], engine=_NoEngine()) == []


def test_refused_without_a_context():
    lib = _native.lib()
    mode = (ctypes.c_uint8 * 1)(3)
    data = (ctypes.c_uint64 * 4)()
    off = (ctypes.c_uint64 * 2)(0, 1)
    out = (ctypes.c_uint64 * 4)()
    assert lib.p252_hash_batch_mixed(None, mode, data, 1, off, 1, 1, out, 1, off, 1, None, 0) == INVALID_ARGUMENT


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.Hash.finalize_batch([_hash(pb.Domain.Other, 2, 3, out_len=2), _hash(pb.Domain.Merkle4, 4)], truncated=[True, False])
    with pytest.raises(pb.EngineError):
        pb.Hash.digest_batch_mixed(np.array([3], dtype=np.uint8), np.zeros((2, 4), dtype=np.uint64),
                                   np.array([0, 2], dtype=np.uint64), np.array([0, 1], dtype=np.uint64))
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "HASH_MIXED_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
