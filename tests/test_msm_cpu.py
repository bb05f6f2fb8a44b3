"""Multi-scalar multiplication without a GPU: the c-bit signed recoding against big integers on edge scalars, the model of
the kernels' bucket algorithm (msm_oracle.py) against the plain sum on uniform, all-equal and single-window scalars, the
window choice and the counts the source pins, and the bindings of p252_jubjub_msm / p252_schnorr_verify_all -- the
header, the library, the ctypes signature table and the Rust block in msm.rs agree, lib.rs keeps its three blocks, the
plain-C program calls exactly the new block, the C and C++ programs compile, and the calls fail loudly without a GPU.  The
same C and C++ programs run on the device in test_gpu_msm.py."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

import jubjub_oracle as jo
import msm_oracle as mo
import poseidon252_b200 as pb
from poseidon252_b200 import _native
from test_stealth_cpu import _blocks, _compile, _header

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST = os.path.join(ROOT, "bindings", "rust", "src")
CUH = os.path.join(ROOT, "poseidon252_b200", "csrc", "jubjub_device.cuh")
KCU = os.path.join(ROOT, "poseidon252_b200", "csrc", "kernels.cu")
KH = os.path.join(ROOT, "poseidon252_b200", "csrc", "kernels.h")
WANT = {"p252_jubjub_msm": 7, "p252_schnorr_verify_all": 12}
N = jo.R_J


# ---- recoding -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", range(mo.MIN_BITS, mo.MAX_BITS + 1))
def test_recoding_against_big_integers(c):
    rng = random.Random(c)
    W, half = mo.windows(c), 1 << (c - 1)
    assert W * c >= 253 and (W - 1) * c < 253
    for s in mo.edge_scalars() + [rng.randrange(N) for _ in range(200)] + [(1 << 252) - 1]:
        d = mo.recode(s, c)
        assert len(d) == W and sum(e << (c * w) for w, e in enumerate(d)) == s
        assert all(-half <= e < half for e in d[:-1]) and 0 <= d[-1] <= half
    # every low digit at -2^(c-1), and the carry that reaches the top window
    s = mo.all_low_digits_negative(c)
    assert s < N and mo.recode(s, c)[:-1] == [-half] * (W - 1) and mo.recode(s, c)[-1] == 1
    top = ((1 << (252 - (W - 1) * c)) - 1) << ((W - 1) * c) | ((1 << ((W - 1) * c)) - 1)
    assert mo.recode(top, c)[-1] == 1 << (252 - (W - 1) * c)


# ---- the bucket algorithm against the plain sum --------------------------------------------------------------------------
@pytest.mark.parametrize("dist,n", [("uniform", 1 << 16), ("uniform", 1000), ("equal", 1 << 12), ("zero", 4096),
                                    ("single", 1 << 12), ("small", 5000)])
def test_model_against_plain_sum(dist, n):
    rng = random.Random(n)
    sc = {"uniform": lambda: [rng.randrange(N) for _ in range(n)],
          "equal": lambda: [N - 12345] * n,
          "zero": lambda: [0] * n,
          "single": lambda: [rng.randrange(1, 1 << 12) << 130 for _ in range(n)],    # one nonzero window
          "small": lambda: [rng.randrange(3) for _ in range(n)]}[dist]()
    logs = [rng.randrange(N) for _ in range(n)]
    passes = []
    assert mo.msm_model(sc, logs, stats=passes) == mo.plain_sum(sc, logs)
    assert passes[0] >= 1
    assert mo.msm_model(sc[:3000], logs[:3000], c=5, chunk=1024) == mo.plain_sum(sc[:3000], logs[:3000])


def test_each_pass_bounds_the_work_per_piece():
    """all digits of a window in one bucket: every pass adds at most PIECE entries per piece and the list shrinks"""
    n = 1 << 12
    ent = sorted(mo.keys([N - 1] * n, 9), key=lambda e: e[0])
    nb = mo.windows(9) << 8
    buckets, lengths = {}, [len(ent)]
    lst, _ = mo.bucket_pass(ent, nb, buckets, lambda v: 1)
    while lst is not None:
        lengths.append(len(lst))
        lst, _ = mo.bucket_pass(lst, nb, buckets, lambda v: v)
    assert all(b <= 2 * -(-a // mo.PIECE) for a, b in zip(lengths, lengths[1:]))


# ---- window choice and counts pinned in the source --------------------------------------------------------------------
def test_counts_and_window_choice_match_the_source():
    src = open(CUH).read()
    assert "kMsmMinBits = %d, kMsmMaxBits = %d" % (mo.MIN_BITS, mo.MAX_BITS) in src
    assert "kProductsPerMsmRow == 6 && kProductsPerMsmDigit == 7" in src
    assert "kProductsPerMsmCarry == 9 && kProductsPerMsmBucket == 18" in src
    assert "msm_windows(kMsmMaxBits) == 20 && msm_windows(kMsmMinBits) == 64" in src
    assert (mo.windows(13), mo.windows(4)) == (20, 64)
    assert "constexpr int kMsmPiece = %d" % mo.PIECE in open(KH).read()
    assert "constexpr int kMsmThreads = %d" % mo.THREADS in open(KCU).read()
    # the chunk of 2^17 points takes 13-bit windows; a chunk of 2^10 fewer bits
    assert mo.bits_for(1 << 17) == 13 and mo.bits_for(1 << 18) == 13 and mo.bits_for(1024) < 13


# ---- bindings ------------------------------------------------------------------------------------------------------
def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "msm.rs")) == [WANT]
    assert "mod msm;" in open(os.path.join(RUST, "lib.rs")).read()


def test_lib_rs_keeps_three_blocks_without_the_new_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)
    assert not any(n in WANT for b in _blocks(os.path.join(RUST, "schnorr.rs")) for n in b)


def test_header_states_variable_time_and_cofactor():
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    sec = src[src.index("JubJub multi-scalar multiplication"):src.index("int p252_schnorr_verify_all")]
    assert "VARIABLE TIME" in sec and "Cofactored" in sec and "[8]" in sec


def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "msm_smoke.c"), os.path.join(ROOT, "tests", "c", "msm_smoke"),
                    "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "msm_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "msm_mirror_test"), "-std=c++17")


def test_c_smoke_calls_exactly_the_msm_block():
    block = _blocks(os.path.join(RUST, "msm.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "msm_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_c_msm_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "MSM_SMOKE_NO_DEVICE" in res.stdout or "MSM_SMOKE_OK" in res.stdout


def test_cpp_msm_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "msm mirror ok" in res.stdout


def test_python_exports():
    for name in ("jubjub_msm", "schnorr_verify_all"):
        assert name in pb.__all__ and callable(getattr(pb, name))
    for name in ("jubjub_msm", "schnorr_verify_all", "last_msm_invalid", "last_verify_all"):
        assert callable(getattr(pb.Engine, name))


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([jo.GENERATOR])
    with pytest.raises(pb.EngineError):
        pb.jubjub_msm(np.zeros((1, 4), dtype=np.uint64), g)
    with pytest.raises(pb.EngineError):
        pb.schnorr_verify_all(g, np.zeros((1, 4), np.uint64), g, np.zeros((1, 4), np.uint64), g[0])
    res = c_smoke()                                               # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "MSM_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
