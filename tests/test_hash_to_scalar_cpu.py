"""BlsScalar::hash_to_scalar batches without a GPU: the host restatement p252_hash_to_scalar against the oracle
(hashlib's BLAKE2b-512 and a big-integer from_bytes_wide) at the 128-byte block edges and random lengths, the bindings of
the two new calls -- the header, the library, the ctypes signature table, the Rust block in hash_to_scalar.rs and the
plain-C program agree, the C and C++ programs compile with -Wall -Werror -- and the refusals that need no device.  The
same C and C++ programs run on the device in test_gpu_hash_to_scalar.py."""
import ctypes
import os
import re

import numpy as np
import pytest

import hades_oracle as o
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200.hash import hash_to_scalar, pack_bytes
from poseidon252_b200.scalar import P, from_mont
from test_notes_cpu import _compile
from test_stealth_cpu import RUST, ROOT, _blocks, _header

WANT = {"p252_hash_to_scalar_batch": 9, "p252_scalars_from_bytes_wide": 5}
INVALID_ARGUMENT = -1                                             # P252_ERR_INVALID_ARGUMENT
EDGE_LENGTHS = (0, 1, 127, 128, 129, 255, 256, 257)


def _msg(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


# ---- the host restatement against the oracle ----------------------------------------------------------------------
def test_host_hash_to_scalar_matches_the_oracle_at_block_edges_and_random_lengths():
    rng = np.random.default_rng(1)
    lengths = list(EDGE_LENGTHS) + [int(v) for v in rng.integers(0, 4096, 40)]
    for n in lengths:
        m = _msg(rng, n)
        assert int(from_mont(hash_to_scalar(m))) == o.hash_to_scalar(m), n


def test_oracle_from_bytes_wide_is_the_512_bit_integer_mod_p():
    import hashlib
    for m in (b"", b"abc", bytes(range(256))):
        d = hashlib.blake2b(m, digest_size=64).digest()
        assert o.from_bytes_wide(d) == int.from_bytes(d, "little") % P


def test_pack_bytes_layout():
    msgs = [b"", b"ab", b"", b"xyz"]
    data, offsets, longest = pack_bytes(msgs)
    assert data.dtype == np.uint8 and data.tobytes() == b"abxyz"
    assert offsets.dtype == np.uint64 and offsets.tolist() == [0, 0, 2, 2, 5]
    assert longest == 3
    data, offsets, longest = pack_bytes([])
    assert data.shape == (0,) and offsets.tolist() == [0] and longest == 0


# ---- bindings --------------------------------------------------------------------------------------------------------
def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "hash_to_scalar_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "hash_to_scalar_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "hash_to_scalar_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "hash_to_scalar_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "hash_to_scalar.rs")) == [WANT]      # one block, exactly the two functions
    assert "mod hash_to_scalar;" in open(os.path.join(RUST, "lib.rs")).read()
    assert len(_blocks(os.path.join(RUST, "lib.rs"))) == 3
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "lib.rs")) for n in b)
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    assert re.search(r"#define P252_HASH_TO_SCALAR_MAX_LEN \(1u << 20\)", src)
    assert _native.HASH_TO_SCALAR_MAX_LEN == 1 << 20
    assert "pub const HASH_TO_SCALAR_MAX_LEN: usize = 1 << 20;" in open(os.path.join(RUST, "hash_to_scalar.rs")).read()


def test_c_smoke_calls_exactly_the_hash_to_scalar_block():
    block = _blocks(os.path.join(RUST, "hash_to_scalar.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "hash_to_scalar_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_c_smoke_known_answers_are_the_oracle_s():
    """the constants the plain-C program checks on the device are the oracle's values"""
    src = open(os.path.join(ROOT, "tests", "c", "hash_to_scalar_smoke.c")).read()
    limbs = [int(v, 16) for v in re.findall(r"0x([0-9a-f]{16})ULL", src)]
    rows = [sum(limbs[4 * r + k] << (64 * k) for k in range(4)) for r in range(4)]
    msgs = [b"", b"abc", bytes((7 * i + 3) & 255 for i in range(200))]
    R = (1 << 256) % P
    for row, m in zip(rows[:3], msgs):
        assert row == o.hash_to_scalar(m) * R % P
    assert rows[3] == ((1 << 512) - 1) % P * R % P


def test_python_exports():
    for name in ("hash_to_scalar_batch", "pack_bytes"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("hash_to_scalar_batch", "last_hash_to_scalar_rejected", "scalars_from_bytes_wide"):
        assert callable(getattr(pb.Engine, name))


def test_c_hash_to_scalar_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "HASH_TO_SCALAR_SMOKE_NO_DEVICE" in res.stdout or "HASH_TO_SCALAR_SMOKE_OK" in res.stdout


def test_cpp_hash_to_scalar_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "hash_to_scalar mirror ok" in res.stdout


# ---- refusals that need no device ----------------------------------------------------------------------------------
def test_refused_without_a_context():
    lib = _native.lib()
    buf = (ctypes.c_uint8 * 8)()
    off = (ctypes.c_uint64 * 2)(0, 8)
    out = (ctypes.c_uint64 * 4)()
    assert lib.p252_hash_to_scalar_batch(None, buf, 8, off, 1, 8, out, None, 0) == INVALID_ARGUMENT
    assert lib.p252_scalars_from_bytes_wide(None, buf, 0, out, 0) == INVALID_ARGUMENT


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.hash_to_scalar_batch([b"abc", b""])
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "HASH_TO_SCALAR_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
