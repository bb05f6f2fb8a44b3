"""The constant fold of the scaled-lazy Hades (cfold in hades_device.cuh): the partial rounds' lane-4 correction and the
output multiplication are products C w / R by a table constant C, computed as S = sum_j w_j T_j over the 32-bit limbs
w_j of w with T_j = C 2^(32j - 192) mod p, then two Montgomery rows z = (S + m0 p + m1 p 2^32) / 2^64.  In a partial
round the fold is taken on lane 4's S-box input u (g = G u / R) and enters the S-box's last product,
montmul(g, u^4 / R^3).

CPU:
* The emulated PTX rows (tools/gen_field_ptx.py) equal the integer definition at their carry edges (all-ones w, every
  T_j = p - 1, zero) and on random operands, and give the residue montmul(C, w) gives.
* Upper bounds propagated through all 68 rounds with the real fold tables prove S < 2^290, z < p + 2^226 (so z is a
  valid row operand, z + p <= 2^256), the corrected S-box output < 1.887 p, the FP64 column sums < 2^52, T < 2^288 and
  a final value < 2p.
* Constructed states reach the fold's results >= p at every partial round: z == p (a true zero: the stored lane 4 of a
  partial round's S-box input is p, and S is a nonzero multiple of p below 2^64 p) and z == 1 + p
  (stored class 1: S + m p == 2^64 is impossible for S >= 2^64, so the rows land on 1 + p); the output fold likewise at
  output lane values 0 and R^-1 (Montgomery 1).  A class s in (1, 2^226) lands on s or s + p depending on the low bits
  of S, which the backward construction does not choose, so those are left to the model's bound.
GPU (-m gpu): every permutation path on those states, bit for bit against the C oracle."""
import functools
import random
from collections import defaultdict

import numpy as np
import pytest

import c_oracle
import gen_field_ptx as g
import hades_edges as he
import hades_model as hm
import hades_oracle as o
from conftest import mont

P = hm.P
PINV64 = pow(P, -1, 1 << 64)
PARTIAL = range(hm.HALF_FULL, hm.HALF_FULL + hm.PARTIAL_ROUNDS)


def fold_def(tab, w):
    """The integer the fold computes, from its definition: one 64-bit Montgomery digit on S."""
    s = sum(((w >> (32 * j)) & hm.M32) * t for j, t in enumerate(tab))
    m = (-s * PINV64) % (1 << 64)
    assert (s + m * P) % (1 << 64) == 0
    return (s + m * P) >> 64


def mm(x, y):
    return hm.montmul(x, y, "test")


# ---- emulated PTX == definition -------------------------------------------------------------------------------------------
def test_fold_tables():
    tb = hm.TABLES
    for c, tab in [(tb.G[r], tb.GT[r]) for r in PARTIAL] + [(tb.F, tb.FT)]:
        assert len(tab) == 8 and all(0 <= t < P for t in tab)
        w = sum(1 << (32 * j) for j in range(8))
        assert sum(tab) % P == c * w * pow(2, -192, P) % P


def test_fold_rows_at_carry_edges():
    tb = hm.TABLES
    tabs = [[P - 1] * 8, [0] * 8, tb.FT, tb.GT[hm.HALF_FULL], tb.GT[hm.HALF_FULL + hm.PARTIAL_ROUNDS - 1]]
    ws = [0, 1, hm.TWO256 - 1, P - 1, P, 2 * P - 1, hm.M32, hm.TWO256 - (1 << 32), (1 << 255) - 1]
    for tab in tabs:
        for w in ws:
            z = g.emu_cfold(tab, w)
            assert z == fold_def(tab, w) == hm.cfold(tab, w, "test")
            assert z < P + (1 << 226)
    # the largest sum: every limb all-ones times every T_j = p - 1
    s = 8 * hm.M32 * (P - 1)
    assert s < 1 << 290 and g.emu_cfold([P - 1] * 8, hm.TWO256 - 1) == fold_def([P - 1] * 8, hm.TWO256 - 1)


def test_fold_random_and_residue():
    rnd = random.Random(11)
    tb = hm.TABLES
    consts = [(tb.G[r], tb.GT[r]) for r in PARTIAL] + [(tb.F, tb.FT)]
    for _ in range(300):
        c, tab = rnd.choice(consts)
        w = rnd.choice([rnd.randrange(hm.TWO256), rnd.randrange(2 * P), hm.TWO256 - 1 - rnd.randrange(1 << 40),
                        rnd.randrange(1 << rnd.randrange(1, 256))])
        z = g.emu_cfold(tab, w)
        assert z == fold_def(tab, w)
        assert z % P == mm(c, w) % P, "fold residue differs from montmul(C, w)"
    rt = [rnd.randrange(P) for _ in range(8)]
    assert g.emu_cfold(rt, hm.TWO256 - 1) == fold_def(rt, hm.TWO256 - 1)


def test_fold_wide_op_count():
    assert g.cfold_wide_ops() == 8 * 8 + 2 * 7
    assert "constexpr int kWideOps_fr_cfold = 78;" in g.emit_header()


# ---- operand bounds with the fold, proved ------------------------------------------------------------------------------
def fold_bound(tab, w):
    """(S, z) upper bounds of the fold over every w' <= w: limb j of w' is at most min(2^32 - 1, w >> 32j)."""
    s = sum(min(hm.M32, w >> (32 * j)) * t for j, t in enumerate(tab))
    return s, (s + ((1 << 64) - 1) * P) >> 64


def proved_bounds():
    """As test_hades_edges.proved_bounds, with the lane-4 correction and the output product as constant folds."""
    tb, C, M = hm.TABLES, hm.CMAT, hm.TWO256

    def mm_bound(x, y, row):
        assert row + P <= M
        return (x * y + (M - 1) * P) >> 256

    def sq(x):
        return (x * x + (M - 1) * P) >> 256

    worst = defaultdict(int)
    u = [P - 1] * he.W
    for r in range(he.ROUNDS):
        z = []
        for i in range(he.W):
            if r:
                worst["u"] = max(worst["u"], u[i])
            if hm.is_full(r) or i == 4:
                a = sq(u[i])
                b = sq(a)
                for k, v in (("sqr1", a), ("sqr2", b)):
                    worst[k] = max(worst[k], v)
                if hm.is_full(r):
                    x = mm_bound(u[i], b, u[i])
                    worst["x5"] = max(worst["x5"], x)
                else:
                    s, gu = fold_bound(tb.GT[r], u[i])
                    assert s < 1 << 290, "round %d: fold sum may reach 2^290" % r
                    worst["S"], worst["gfold"] = max(worst["S"], s), max(worst["gfold"], gu)
                    x = mm_bound(gu, b, gu)
                    worst["gmul"] = max(worst["gmul"], x)
                z.append(x)
            else:
                z.append(u[i])
        nxt = []
        for i in range(he.W):
            t = (tb.A[r + 1][i] if r + 1 < he.ROUNDS else 0) + sum(C[i][j] * z[j] for j in range(he.W))
            assert t < 1 << 288, "round %d lane %d: T may reach 2^288" % (r, i)
            worst["T"] = max(worst["T"], t)
            for k in range(8):
                col = sum(C[i][j] * min(hm.M32, z[j] >> (32 * k)) for j in range(he.W))
                assert col < 1 << 52, "round %d lane %d limb %d: FP64 column may reach 2^52" % (r, i, k)
                worst["col"] = max(worst["col"], col)
            nxt.append((t + hm.M32 * P) >> 32)
        u = nxt
    for x in u:
        s, f = fold_bound(tb.FT, x)
        worst["S"], worst["final"] = max(worst["S"], s), max(worst["final"], f)
    return worst


def test_operand_bounds_with_fold_proved():
    b = proved_bounds()
    for site, lim in (("u", 10003), ("sqr1", 14534), ("sqr2", 19565), ("x5", 18862), ("gmul", 18870)):
        assert b[site] * 10000 < lim * P, "%s bound %.6f p exceeds %.4f p" % (site, b[site] / P, lim / 1e4)
    assert b["u"] < P + (1 << 243)
    assert b["S"] < 1 << 290
    assert b["gfold"] < P + (1 << 226) and b["final"] < P + (1 << 226)
    assert b["final"] < 2 * P                        # one conditional subtraction gives [0, p)
    assert b["T"] < 1 << 288 and b["col"] < 1 << 52


# ---- constructed states at the fold's edges ----------------------------------------------------------------------------
def _case(r, true4, rng):
    v = [rng.randrange(P) for _ in range(he.W)]
    v[4] = true4
    return he.state_at_round_to_input(r, v)


@functools.lru_cache(maxsize=None)
def fold_corpus():
    """(name, canonical input, site, (round, lane), wanted traced value): per partial round the lane-4 fold at p and at
    1 + p; per output lane the output fold at p and 1 + p."""
    rng = random.Random("fold-%d" % he.SEED)
    cases = []
    for r in PARTIAL:
        kappa = hm.TABLES.kappa[r]
        # the fold g = G u / R of the S-box input: class 0 for a true zero; class 1 for stored u = R / G, i.e. the
        # true value kappa_r R / G
        cases.append(("gfold_p@r%d" % r, _case(r, 0, rng), "gfold", (r, 4), P))
        true1 = kappa * hm.R * pow(hm.TABLES.G[r], -1, P) % P
        cases.append(("gfold_1_plus_p@r%d" % r, _case(r, true1, rng), "gfold", (r, 4), 1 + P))
    for lane in range(he.W):
        for name, y, want in (("final_p", 0, P), ("final_1_plus_p", o.R_INV, 1 + P)):
            out = [rng.randrange(P) for _ in range(he.W)]
            out[lane] = y
            cases.append(("%s@l%d" % (name, lane), he.output_to_input(out), "final", (he.ROUNDS, lane), want))
    return tuple(cases)


def test_fold_corpus_reaches_its_edges():
    miss = []
    for name, x, site, key, want in fold_corpus():
        t = he.trace(x)
        if t.sites[site][key] != want:
            miss.append(name)
        assert t.out == [he.mont(y) for y in o.perm(x)], name
    assert not miss, "fold edges not reached: %s" % miss
    assert len(fold_corpus()) == 2 * hm.PARTIAL_ROUNDS + 2 * he.W


@pytest.mark.gpu
def test_gpu_permute_on_fold_edges(engine):
    x = mont([c[1] for c in fold_corpus()]).reshape(-1, 5, 4)
    want = c_oracle.permute(x)
    assert np.array_equal(engine.permute_batch(x), want)
    big = np.tile(x, (max(1, (1 << 16) // x.shape[0]) + 1, 1, 1))
    assert np.array_equal(engine.permute_batch(big), np.tile(want, (big.shape[0] // x.shape[0], 1, 1)))
    y = x.copy()
    engine.permute_batch_inplace(y)
    assert np.array_equal(y, want)
