"""All-or-nothing verification of double-key signatures without a GPU: the model of verify_double_all_oracle.py against
the AND of the cofactored per-item equations on genuine, tampered, torsion-shifted and cancelling batches, and the
bindings of p252_schnorr_verify_double_all -- the header, the library, the ctypes signature table and the Rust block in
verify_double_all.rs agree, lib.rs keeps its three blocks, msm.rs and schnorr_double.rs keep theirs, the plain-C program
calls exactly the new block, the C and C++ programs compile, and the call fails loudly without a GPU.  The same C and
C++ programs run on the device in test_gpu_verify_double_all.py."""
import ctypes
import functools
import os
import re

import numpy as np
import pytest

import jubjub_oracle as jo
import poseidon252_b200 as pb
import schnorr_double_oracle as sdo
import verify_double_all_oracle as vo
from poseidon252_b200 import _native
from test_stealth_cpu import _blocks, _compile, _header

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST = os.path.join(ROOT, "bindings", "rust", "src")
WANT = {"p252_schnorr_verify_double_all": 16}
N, P, G = jo.R_J, jo.P, jo.GENERATOR


@functools.lru_cache(maxsize=None)
def g_prime():
    return jo.random_subgroup_point(np.random.default_rng(900))


@functools.lru_cache(maxsize=None)
def batch(n=3, seed=901):
    """n genuine signatures by n keys: (pks, pkps, us, Rs, Rps, ms)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        sk, r, m = jo.random_secret(rng), jo.random_secret(rng), int(rng.integers(0, 1 << 62))
        pk, pkp = sdo.key_pair(sk, g_prime())
        u, R, Rp = sdo.sign_double(sk, r, m, g_prime())
        out.append((pk, pkp, u, R, Rp, m))
    return tuple(zip(*out))


def weights(n, seed):
    rng = np.random.default_rng(seed)
    return ([int(x) << 64 | int(y) for x, y in rng.integers(1, 1 << 62, (n, 2))],
            [int(x) << 64 | int(y) for x, y in rng.integers(1, 1 << 62, (n, 2))])


def model(cols, w, wp, one_pair=False):
    pks, pkps, us, Rs, Rps, ms = cols
    if one_pair:
        pks, pkps = pks[:1], pkps[:1]
    return vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w, wp, g_prime())


def per_item(cols):
    return all(vo.cofactored_items(*row, g_prime()) for row in zip(*cols))


# ---- the model against the per-item equations --------------------------------------------------------------------------
def _tampered(cols, what):
    pks, pkps, us, Rs, Rps, ms = [list(c) for c in cols]
    i = 1
    if what == "u+1":
        us[i] = (us[i] + 1) % N
    elif what == "u-1":
        us[i] = (us[i] - 1) % N
    elif what == "m+1":
        ms[i] = (ms[i] + 1) % P
    elif what == "R":
        Rs[i] = jo.add(Rs[i], G)
    elif what == "R'":
        Rps[i] = jo.add(Rps[i], g_prime())
    elif what == "swap":
        Rs[i], Rps[i] = Rps[i], Rs[i]
    elif what == "PK'=PK":
        pkps[i] = pks[i]
    return pks, pkps, us, Rs, Rps, ms


@pytest.mark.parametrize("what", ["genuine", "u+1", "u-1", "m+1", "R", "R'", "swap", "PK'=PK"])
def test_model_equals_and_of_cofactored_items(what):
    cols = _tampered(batch(), what)
    w, wp = weights(3, 902)
    want = per_item(cols)
    assert want == (what == "genuine")
    assert model(cols, w, wp) == want


def test_model_one_key_pair():
    rng = np.random.default_rng(903)
    sk = jo.random_secret(rng)
    pk, pkp = sdo.key_pair(sk, g_prime())
    rows = []
    for m in (3, 4, 5):
        u, R, Rp = sdo.sign_double(sk, jo.random_secret(rng), m, g_prime())
        rows.append((pk, pkp, u, R, Rp, m))
    cols = tuple(zip(*rows))
    w, wp = weights(3, 904)
    assert model(cols, w, wp, one_pair=True) is True
    bad = list(cols)
    bad[5] = (3, 4, 6)
    assert model(tuple(bad), w, wp, one_pair=True) is False


def test_torsion_shifted_R_passes_the_cofactored_check():
    rng = np.random.default_rng(905)
    T = jo.order8_point(rng)
    sk = jo.random_secret(rng)
    pk, pkp = sdo.key_pair(sk, g_prime())
    r, m = jo.random_secret(rng), 77
    for which in ("R", "R'"):
        R, Rp = jo.mul(r, G), jo.mul(r, g_prime())
        if which == "R":
            R = jo.add(R, T)
        else:
            Rp = jo.add(Rp, T)
        u = (r - sdo.challenge2(R, Rp, m) * sk) % N
        assert sdo.verify_double(pk, pkp, u, R, Rp, m, g_prime()) == 0      # the per-item call rejects it
        assert vo.cofactored_items(pk, pkp, u, R, Rp, m, g_prime())
        assert vo.verify_double_all([pk], [pkp], [u], [R], [Rp], [m], [5], [7], g_prime()) is True
        assert vo.verify_double_all([pk], [pkp], [u], [R], [Rp], [m], [5], [7], g_prime(), cofactor=1) is False


def test_cancelling_signature_needs_independent_weights():
    """R = [r] G + D, R' = [r] G' - D: fails per item, passes with weight_p == weight, fails with independent weights"""
    rng = np.random.default_rng(906)
    sk, r, m = jo.random_secret(rng), jo.random_secret(rng), 99
    pk, pkp = sdo.key_pair(sk, g_prime())
    D = jo.random_subgroup_point(rng)
    u, R, Rp = vo.cancelling_signature(sk, r, m, D, g_prime())
    assert sdo.verify_double(pk, pkp, u, R, Rp, m, g_prime()) == 0
    assert not vo.cofactored_items(pk, pkp, u, R, Rp, m, g_prime())
    pks, pkps, us, Rs, Rps, ms = [list(c) for c in batch()]
    pks[1], pkps[1], us[1], Rs[1], Rps[1], ms[1] = pk, pkp, u, R, Rp, m
    w, wp = weights(3, 907)
    assert vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w, w, g_prime()) is True
    assert vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w, wp, g_prime()) is False


def test_zero_weight_leaves_its_equation_unchecked():
    pks, pkps, us, Rs, Rps, ms = [list(c) for c in batch()]
    w, wp = weights(3, 908)
    pks[2] = jo.add(pks[2], G)                                # the first equation of item 2 fails (c is unchanged)
    assert vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w, wp, g_prime()) is False
    w0 = list(w)
    w0[2] = 0
    assert vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w0, wp, g_prime()) is True
    wp0 = list(wp)
    wp0[2] = 0                                                # a zero weight on the other equation does not help
    assert vo.verify_double_all(pks, pkps, us, Rs, Rps, ms, w, wp0, g_prime()) is False


def test_invalid_items_and_off_curve_R():
    cols = [list(c) for c in batch()]
    w, wp = weights(3, 909)
    rng = np.random.default_rng(910)
    for k, bad in ((2, N), (5, P)):                           # u >= r_J, m >= p
        c = [list(x) for x in cols]
        c[k][0] = bad
        assert model(c, w, wp) is False
    assert model(cols, [N] + w[1:], wp) is False and model(cols, w, wp[:2] + [N]) is False
    c = [list(x) for x in cols]
    c[3][0] = jo.off_curve_point(rng)                         # canonical R off the curve: not invalid, still False
    assert vo.item_valid(*[x[0] for x in c], w[0], wp[0]) and model(c, w, wp) is False


# ---- bindings ------------------------------------------------------------------------------------------------------
def c_smoke():
    return _compile("gcc", os.path.join(ROOT, "tests", "c", "verify_double_all_smoke.c"),
                    os.path.join(ROOT, "tests", "c", "verify_double_all_smoke"), "-std=c11")


def cpp_mirror():
    return _compile("g++", os.path.join(ROOT, "tests", "cpp", "verify_double_all_mirror_test.cpp"),
                    os.path.join(ROOT, "tests", "cpp", "verify_double_all_mirror_test"), "-std=c++17")


def test_header_library_signatures_and_rust_block_agree():
    hdr = _header()
    lib = _native.lib()
    for name, nparams in WANT.items():
        assert hdr[name] == nparams, name
        assert hasattr(lib, name) and len(_native.SIGNATURES[name][1]) == nparams, name
    assert _blocks(os.path.join(RUST, "verify_double_all.rs")) == [WANT]   # one block, exactly the new function
    assert "mod verify_double_all;" in open(os.path.join(RUST, "lib.rs")).read()


def test_existing_blocks_keep_their_functions():
    blocks = _blocks(os.path.join(RUST, "lib.rs"))
    assert len(blocks) == 3
    assert not any(n in WANT for b in blocks for n in b)
    assert _blocks(os.path.join(RUST, "msm.rs")) == [{"p252_jubjub_msm": 7, "p252_schnorr_verify_all": 12}]
    assert [set(b) for b in _blocks(os.path.join(RUST, "schnorr_double.rs"))] == [
        {"p252_schnorr_sign_double_batch", "p252_schnorr_verify_double_batch", "p252_note_sign_double_batch"}]


def test_header_states_variable_time_cofactor_and_independent_weights():
    src = open(os.path.join(ROOT, "include", "poseidon252_b200.h")).read()
    sec = src[src.index("All-or-nothing batch verification of double-key"):src.index("int p252_schnorr_verify_double_all")]
    assert "VARIABLE TIME" in sec and "Cofactored" in sec and "[8]" in sec and "independently" in sec


def test_c_smoke_calls_exactly_the_new_block():
    block = _blocks(os.path.join(RUST, "verify_double_all.rs"))[0]
    first = _blocks(os.path.join(RUST, "lib.rs"))[0]
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "tests", "c", "verify_double_all_smoke.c")).read(), flags=re.S)
    called = set(re.findall(r"\b(p252_[a-z0-9_]+)\s*\(", src))
    assert {n for n in called if n in WANT} == set(block)
    assert called - set(block) <= set(first)


def test_c_verify_double_all_smoke_cpu():
    res = c_smoke()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "VERIFY_DOUBLE_ALL_SMOKE_NO_DEVICE" in res.stdout or "VERIFY_DOUBLE_ALL_SMOKE_OK" in res.stdout


def test_cpp_verify_double_all_mirror_cpu():
    res = cpp_mirror()
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    assert "verify double all mirror ok" in res.stdout


def test_python_exports():
    assert "schnorr_verify_double_all" in pb.__all__ and callable(pb.schnorr_verify_double_all)
    for name in ("schnorr_verify_double_all", "last_verify_double_all", "last_schnorr_double_invalid"):
        assert callable(getattr(pb.Engine, name))


def test_no_cpu_fallback_without_gpu():
    cnt = ctypes.c_int(0)
    _native.lib().p252_device_count(ctypes.byref(cnt))
    if cnt.value > 0:
        pytest.skip("a GPU is present")
    g = jo.points_mont([G])
    one = np.ones((1, 4), np.uint64)
    with pytest.raises(pb.EngineError):
        pb.schnorr_verify_double_all(g, g, one, g, g, one, g[0], g[0])
    res = c_smoke()                                           # P252_ERR_NO_DEVICE, reported by name
    assert res.returncode == 0 and "VERIFY_DOUBLE_ALL_SMOKE_NO_DEVICE no usable sm_90 CUDA device" in res.stdout, res.stdout
