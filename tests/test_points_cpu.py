"""Point compression without a GPU: the model of points_oracle.py (round trips, the sign bit, the edges), the restatement of
the kernel's sqrt_ratio against Tonelli-Shanks (squares, non-squares, num = 0, every loop round's conditional move both
ways), the constants and the product counts the kernel pins, and the bindings of p252_points_from_bytes /
p252_points_to_bytes -- the header, the library, the ctypes signature table and the Rust block in points.rs agree, lib.rs
keeps its three blocks, the plain-C program calls exactly the new block, the C and C++ programs compile, and the calls
fail loudly without a GPU.  The same C and C++ programs run on the device in test_gpu_points.py."""
import ctypes
import os
import re

import numpy as np
import pytest

import jubjub_oracle as jo
import points_oracle as po
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from test_stealth_cpu import _blocks, _compile, _header

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST = os.path.join(ROOT, "bindings", "rust", "src")
CUH = os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")
WANT = {"p252_points_from_bytes": 7, "p252_points_to_bytes": 7}
P = jo.P


# ---- the model ------------------------------------------------------------------------------------------------------
def _points(rng):
    return ([jo.random_point(rng) for _ in range(20)] + [jo.random_subgroup_point(rng) for _ in range(4)] +
            jo.small_order_points(rng) + [jo.GENERATOR, jo.neg(jo.GENERATOR)])


def test_round_trip_on_full_group_subgroup_and_small_order_points():
    rng = np.random.default_rng(1)
    for pt in _points(rng):
        b = po.encode(pt)
        assert len(b) == 32 and po.decode(b) == pt and po.decode_kernel(b) == pt, pt
        assert int.from_bytes(b, "little") & ((1 << 255) - 1) == pt[1]
        assert b[31] >> 7 == pt[0] & 1


def test_flipped_sign_decodes_to_the_negation():
    rng = np.random.default_rng(2)
    for pt in _points(rng):
        b = bytearray(po.encode(pt))
        b[31] ^= 0x80
        want = pt if pt[0] == 0 else jo.neg(pt)         # u = 0: a set sign bit is accepted, the same point
        assert po.decode(b) == want and po.decode_kernel(b) == want, pt


def test_edges_of_the_encoding():
    enc = lambda v, s=0: (v | s << 255).to_bytes(32, "little")
    for s in (0, 1):
        assert po.decode(enc(1, s)) == (0, 1)           # the identity, either sign
        assert po.decode(enc(P - 1, s)) == (0, P - 1)   # order 2; also the largest canonical v
        u = po.decode(enc(0, s))[0]                      # v = 0: the order-4 points (+-sqrt(-1), 0)
        assert u in (jo.SQRT_M1, P - jo.SQRT_M1) and u & 1 == s and jo.on_curve((u, 0))
        assert po.decode(enc(P, s)) is None             # v = p
    assert po.decode(po.FF) is None and po.decode(bytes(32)) is not None
    assert po.encode((0, 0)) is None and po.encode((P, 1)) is None and po.encode((0, P + 1)) is None
    ns = next(v for v in range(2, 100) if po.decode(enc(v)) is None)  # a v whose u^2 is a non-square
    assert po.decode_kernel(enc(ns)) is None


def test_random_strings_match_between_the_two_decoders():
    rng = np.random.default_rng(3)
    rejected = 0
    for _ in range(400):
        b = rng.integers(0, 256, 32, dtype="uint8").tobytes()
        a = po.decode(b)
        assert a == po.decode_kernel(b)
        if a is None:
            rejected += 1
        else:
            assert jo.on_curve(a) and po.encode(a) == b
    assert 100 < rejected < 300                          # about half of all strings (v >= p or a non-square)


# ---- the kernel's sqrt_ratio ----------------------------------------------------------------------------------------
def test_sqrt_ratio_squares_non_squares_and_zero():
    rng = np.random.default_rng(4)
    seen = set()
    for _ in range(300):
        num = int.from_bytes(rng.integers(0, 256, 32, dtype="uint8").tobytes(), "little") % P
        den = int.from_bytes(rng.integers(0, 256, 32, dtype="uint8").tobytes(), "little") % P or 1
        sq, y = po.sqrt_ratio(num, den)
        x = num * pow(den, -1, P) % P
        assert sq == (jo.sqrt(x) is not None)
        assert y * y % P == (x if sq else po.Z * x % P)
        seen.add(sq)
    assert seen == {True, False}
    for den in (1, 2, P - 1, 12345):
        assert po.sqrt_ratio(0, den) == (True, 0)       # the RFC would report num = 0 as a non-square
    assert po.sqrt_ratio(1, 1)[0] and po.sqrt_ratio(po.Z, 1)[0] is False


def test_sqrt_ratio_every_loop_round_both_ways():
    """num = c6^j, den = 1: c6 generates the 2-Sylow subgroup (order 2^32), so the bits of j steer the loop's moves."""
    seen = {}
    for j in [0] + [1 << a for a in range(32)] + [(1 << 32) - (1 << a) for a in range(32)]:
        num = pow(po.C6, j, P)
        tr = []
        sq, y = po.sqrt_ratio(num, 1, tr)
        assert sq == (j % 2 == 0) and y * y % P == (num if sq else po.Z * num % P)
        for k, e1 in tr:
            seen.setdefault(k, set()).add(e1)
    assert sorted(seen) == list(range(2, 33))
    assert all(seen[k] == {True, False} for k in seen), seen


def _cuh_words(name):
    m = re.search(r"#define %s \{([^}]*)\}" % name, open(CUH).read())
    return sum(int(w.strip().rstrip("u"), 16) << (32 * k) for k, w in enumerate(m.group(1).split(",")))


def test_constants_are_derived_and_match_the_kernel():
    import hades_oracle as ho
    assert (P - 1) % (1 << po.C1) == 0 and po.T % 2 == 1
    assert pow(po.Z, (P - 1) // 2, P) == P - 1                       # Z is a non-residue
    assert jo.SQRT_M1 == pow(po.Z, (P - 1) // 4, P)
    assert _cuh_words("P252_JJ_SQRT_C3") == po.C3
    assert _cuh_words("P252_JJ_SQRT_C6") == po.C6 * ho.R % P
    assert _cuh_words("P252_JJ_SQRT_C7") == po.C7 * ho.R % P
    src = open(CUH).read()
    assert "kSqrtC1 = %d, kSqrtC3Bits = %d, kSqrtC3Ones = %d;" % (po.C1, po.C3.bit_length(), bin(po.C3).count("1")) in src
    assert (po.C3.bit_length(), bin(po.C3).count("1")) == (222, 132)


# ---- product counts -------------------------------------------------------------------------------------------------
def test_product_counts_match_the_kernel():
    src = open(CUH).read()
    assert "kProductsPerSqrtRatio == 986" in src and "kProductsPerDecompress == 989" in src
    assert "kProductsPerCompress == 4" in src
    # den^(2^32 - 1) 31 + 5, steps 3-5 3, c3 221 + 131, steps 7-10 4, step 11 31, steps 13-14 2, loop 465 + 93
    loop = sum(k - 2 for k in range(2, 33)) + 3 * 31
    assert (31 + 5) + 3 + (221 + 131) + 4 + 31 + 2 + loop == 986
    assert 1 + 2 + 986 == 989                                        # Montgomery form of v, v^2, d v^2


# ---- bindings ------------------------------------------------------------------------------------------------------
def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "points_smoke.c"), os.path.join(ROOT, "tests", "c", "points_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "points_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "points_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "points.rs")) == [WANT]          # one block, exactly the two functions
    assert "mod points;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)


def test_c_smoke_calls_exactly_the_points_block():
    block = _blocks(os.path.join(RUST, "points.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "points_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_python_exports():
    for name in ("point_from_bytes", "point_to_bytes", "points_from_bytes_batch", "points_to_bytes_batch"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("points_from_bytes", "points_to_bytes", "last_points_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_c_points_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "POINTS_SMOKE_NO_DEVICE" in res.stdout or "POINTS_SMOKE_OK" in res.stdout


def test_cpp_points_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "points mirror ok" in res.stdout


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])[0]
    with pytest.raises(pb.EngineError):
        pb.point_to_bytes(g)
    with pytest.raises(pb.EngineError):
        pb.point_from_bytes(bytes(32))
    with pytest.raises(pb.EngineError):
        pb.points_from_bytes_batch(np.zeros((3, 32), dtype=np.uint8))
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "POINTS_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
