"""CPU: the C-ABI library loads and exports every symbol include/poseidon252_b200.h declares; host-side
bookkeeping (tags, io-pattern errors) matches the oracle; without a GPU the engine fails loudly."""
import ctypes
import os
import re

import numpy as np
import pytest

import poseidon252_b200 as pb
from poseidon252_b200 import _native
from poseidon252_b200 import hash as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _native.lib()
    names = header_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(_native.SIGNATURES) == names
    assert b"sm_90a" in lib.p252_version()


def test_tag_derivation_matches_oracle(oracle):
    for dom, od, il, ol in [(pb.Domain.Merkle4, oracle.Domain.Merkle4, 4, 1), (pb.Domain.Merkle2, oracle.Domain.Merkle2, 2, 1),
                            (pb.Domain.Other, oracle.Domain.Other, 42, 1), (pb.Domain.Other, oracle.Domain.Other, 7, 3)]:
        pat = [("absorb", il), ("squeeze", ol)]
        assert H.domain_separator(dom) == od
        assert H.tag_input(pat, od) == oracle.tag_input(pat, od)
        assert pb.scalar.from_mont(H.tag(pat, od)) == oracle.hash_to_scalar(oracle.tag_input(pat, od))
    # README.md:40-47: consecutive absorbs aggregate
    assert H.tag_input([("absorb", 3), ("absorb", 39), ("squeeze", 1)], 0) == \
        oracle.tag_input([("absorb", 42), ("squeeze", 1)], 0)
    for msg in (b"", b"abc", bytes(range(256)) * 3):
        assert pb.scalar.from_mont(H.hash_to_scalar(msg)) == oracle.hash_to_scalar(msg)
    # encryption tag
    lib = _native.lib()
    t = np.zeros(4, dtype=np.uint64)
    for L in (1, 2, 42):
        assert lib.p252_encryption_tag(L, t.ctypes.data) == 0
        pat = [("absorb", 2), ("absorb", 1), ("squeeze", L), ("absorb", L), ("squeeze", 1)]
        assert pb.scalar.from_mont(t) == oracle.hash_to_scalar(oracle.tag_input(pat, oracle.Domain.Encryption))


def test_io_pattern_errors():
    lib = _native.lib()
    t = np.zeros(4, dtype=np.uint64)
    assert lib.p252_hash_tag(int(pb.Domain.Merkle4), 3, 1, t.ctypes.data) == 1      # IOPatternViolation
    assert lib.p252_hash_tag(int(pb.Domain.Merkle4), 4, 2, t.ctypes.data) == 1
    assert lib.p252_hash_tag(int(pb.Domain.Merkle2), 4, 1, t.ctypes.data) == 1
    assert lib.p252_hash_tag(int(pb.Domain.Other), 0, 1, t.ctypes.data) == 2        # InvalidIOPattern
    assert lib.p252_hash_tag(int(pb.Domain.Other), 5, 0, t.ctypes.data) == 2
    assert lib.p252_encryption_tag(0, t.ctypes.data) == 2
    assert lib.p252_hash_tag(99, 4, 1, t.ctypes.data) == -1
    with pytest.raises(pb.IOPatternViolation):
        H.io_pattern(pb.Domain.Merkle4, [2, 1], 1)
    assert lib.p252_strerror(5) == b"DecryptionFailed"
    ni, nl = ctypes.c_size_t(0), ctypes.c_int(0)
    assert lib.p252_merkle4_tree_nodes(4 ** 14, ctypes.byref(ni), ctypes.byref(nl)) == 0
    assert ni.value == 89478485 and nl.value == 14                                   # BASELINE config 4
    assert lib.p252_merkle4_tree_nodes(48, ctypes.byref(ni), ctypes.byref(nl)) == 1


def test_scalar_helpers_roundtrip():
    vals = [0, 1, pb.scalar.P - 1, 12345678901234567890]
    assert list(pb.scalar.from_mont(pb.scalar.to_mont(vals))) == vals
    a = pb.scalar.random_limbs_fast(np.random.default_rng(0), (100,))
    assert all(int(v) < pb.scalar.P for v in pb.scalar.from_mont(a))


def test_no_cpu_fallback_without_gpu():
    n = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(n))
    if n.value > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pb.EngineError):
        pb.Engine(0)
    with pytest.raises(pb.EngineError):
        pb.Hash.digest(pb.Domain.Merkle4, pb.scalar.to_mont([1, 2, 3, 4]))


def test_tag_input_random_patterns_match_oracle(oracle):
    """Random valid io-patterns (absorb first, squeeze last, arbitrary alternation and repeats): the library's
    aggregation + big-endian encoding equals the oracle's restatement of dusk-safe's tag input."""
    import random
    rnd = random.Random(2024)
    for _ in range(300):
        n = rnd.randrange(2, 9)
        kinds = ["absorb"] + [rnd.choice(["absorb", "squeeze"]) for _ in range(n - 2)] + ["squeeze"]
        pat = [(k, rnd.randrange(1, 1 << rnd.randrange(1, 20))) for k in kinds]
        dsep = rnd.choice([0, 0xF, 0x3, 1 << 32, rnd.randrange(1 << 64)])
        assert H.tag_input(pat, dsep) == oracle.tag_input(pat, dsep)
        assert pb.scalar.from_mont(H.tag(pat, dsep)) == oracle.hash_to_scalar(oracle.tag_input(pat, dsep))
    # invalid patterns are rejected like dusk-safe's validation
    lib = _native.lib()
    buf = (ctypes.c_uint8 * 64)()
    n = ctypes.c_size_t(64)
    for calls in ([5], [0x80000005], [5, 0x80000001], [0x80000000, 1], [0x80000003, 0]):
        arr = np.array(calls, dtype=np.uint32)
        n.value = 64
        assert lib.p252_tag_input(arr.ctypes.data, len(calls), 0, buf, ctypes.byref(n)) == 2   # InvalidIOPattern
