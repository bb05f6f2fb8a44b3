"""Build-time model of the Hades kernel's *scaled lazy* formulation (product tooling; it does
not import oracle/).  It (1) regenerates the base constants from the published recipe
(assets/HOWTO.md:23-41,70-97), (2) derives the per-round tables the CUDA kernel
uses, and (3) provides an integer-exact model of the kernel's arithmetic (same montmul /
redc1 / cond-sub definitions, same operand bounds) that tests compare with the oracle.

Why a different formulation is bit-exact
----------------------------------------
The reference's MDS entries are the integers stored in assets/mds.bin read with from_raw
(src/hades/mds_matrix.rs:25-32) = R/(i+j+5) mod p.  With LAMBDA = lcm(5..13) = 360360 and
c_ij = LAMBDA/(i+j+5) (integers <= 72072):  MDS = K * C,  K = R/LAMBDA mod p.
The kernel keeps every lane as an integer `stored` with  true = kappa_r * stored (mod p)  for a
round-dependent, data-independent scale kappa_r:

  * montmul(a,b) = (a*b + m*p)/2^256 (m = -a*b/p mod 2^256)  -- unreduced Montgomery product
  * full round   : z = montmul(u, montsqr(montsqr(u)))            (scale kappa^5 R^4)
  * partial round: lane 4 is multiplied by G_r = kappa_r^4 R^5 (result scale G_r / R, as a montmul) so that its
                   scale equals the scale kappa_r of the four linear lanes: z = montmul(cfold(G_r, u), montsqr^2(u)),
                   the fold taken on the S-box input so that it does not wait for the squarings
  * constant fold: a product C w / R by a table constant C (G_r, F) is  S = sum_j w_j T_j  over w's 32-bit
                   limbs with T_j = C 2^(32j-192) mod p, then two Montgomery rows (S + m0 p + m1 p 2^32)/2^64:
                   64 + 14 limb products instead of a montmul's 120, result < p + 2^226
  * mix          : T_i = A_{r+1,i} + sum_j c_ij z_j  (plain small-integer MADs, 9 limbs), then one
                   Montgomery row  u_i = (T_i + m p)/2^32  (m = -T_i mod 2^32)
                   => kappa_{r+1} = K * sigma_r * 2^32,  A_{r+1,i} = arc_{r+1,i} / (K sigma_r)
  * last round   : out_i = fold of redc1(T_i) by F,  F = K sigma R^2 2^32, then one conditional
                   subtraction -> standard Montgomery form in [0,p), i.e. BlsScalar.0 bit-exact.

Per permutation: 300 Montgomery products + 65 constant folds + 340 small mixes instead of the reference's
2000 products (src/hades/permutation/scalar.rs:54-64 does 25 per round).
"""
from __future__ import annotations

import hashlib
from math import lcm
from typing import List, Sequence

P = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
R = (1 << 256) % P
R_INV = pow(R, -1, P)
WIDTH, FULL_ROUNDS, PARTIAL_ROUNDS = 5, 8, 60
ROUNDS = FULL_ROUNDS + PARTIAL_ROUNDS
HALF_FULL = FULL_ROUNDS // 2
LAMBDA = lcm(*range(WIDTH, 3 * WIDTH - 1))          # lcm(5..13) = 360360
CMAT = [[LAMBDA // (i + j + WIDTH) for j in range(WIDTH)] for i in range(WIDTH)]
M32 = (1 << 32) - 1
TWO256 = 1 << 256
PINV = pow(P, -1, TWO256)
# exponent words (0x433 << 20) of the eight IEEE-double column sums the FP64 mix folds into 9 limbs
K_OFF = 0x43300000 * sum(1 << (32 * k) for k in range(1, 9))


def inv(x: int) -> int:
    return pow(x % P, -1, P)


# ---- base constants (file integers; see module docstring) -----------------------------------
def arc_file_ints() -> List[int]:
    out, prev, data = [], 1, b"poseidon-for-plonk"
    for _ in range(ROUNDS * WIDTH):
        data = hashlib.sha512(data).digest()
        c = (int.from_bytes(data, "little") + prev) % P
        prev = c
        out.append(c * R % P)
    return out


def mds_file_ints() -> List[List[int]]:
    return [[inv(i + j + WIDTH) * R % P for j in range(WIDTH)] for i in range(WIDTH)]


ARC = arc_file_ints()                       # ARC[r*5+i] : field element (canonical integer)
MDS = mds_file_ints()
K_MDS = R * inv(LAMBDA) % P
assert all(MDS[i][j] == K_MDS * CMAT[i][j] % P for i in range(5) for j in range(5))


def is_full(r: int) -> bool:
    return r < HALF_FULL or r >= HALF_FULL + PARTIAL_ROUNDS


# ---- derived tables ---------------------------------------------------------------------------
class Tables:
    """kappa[r]: scale at the S-box input of round r.  A[r][i]: ARC term added inside the mix that
    *produces* round r's input (r >= 1); A[0] is the explicit first add.  G[r]: lane-4 correction
    (partial rounds).  F: final output multiplier.  GT[r], FT: their constant-fold tables (fold_table)."""

    def __init__(self):
        self.kappa = [0] * ROUNDS
        self.A = [[0] * WIDTH for _ in range(ROUNDS)]
        self.G = [0] * ROUNDS
        kappa = R_INV                                   # input is standard Montgomery form
        self.A[0] = [ARC[i] * inv(kappa) % P for i in range(WIDTH)]
        for r in range(ROUNDS):
            self.kappa[r] = kappa
            if is_full(r):
                sigma = pow(kappa, 5, P) * pow(R, 4, P) % P
            else:
                self.G[r] = pow(kappa, 4, P) * pow(R, 5, P) % P
                sigma = kappa
            ks = K_MDS * sigma % P
            if r + 1 < ROUNDS:
                self.A[r + 1] = [ARC[(r + 1) * WIDTH + i] * inv(ks) % P for i in range(WIDTH)]
                kappa = ks * (1 << 32) % P
            else:
                self.F = ks * pow(R, 2, P) * (1 << 32) % P
        self.GT = [fold_table(g) if g else None for g in self.G]
        self.FT = fold_table(self.F)


def fold_table(c: int) -> List[int]:
    """T_j = c 2^(32j - 192) mod p, j = 0..7: sum_j w_j T_j = c w 2^-192 (mod p) for w = sum_j w_j 2^(32j)."""
    i192 = inv(1 << 192)
    return [c * pow(2, 32 * j, P) * i192 % P for j in range(8)]


TABLES = Tables()


# ---- integer-exact primitives (the CUDA code computes exactly these integers) -----------------
class Bounds:
    """Tracks the largest value/p ever seen per site, to back the overflow analysis in DESIGN.md."""
    seen = {}

    @classmethod
    def note(cls, site: str, v: int):
        f = v / P
        if f > cls.seen.get(site, 0.0):
            cls.seen[site] = f


def montmul(x: int, y: int, site: str = "montmul") -> int:
    """(x*y + m*p) / 2^256 with m = -x*y*p^-1 mod 2^256.  `x` is the row operand of the CUDA
    routine (all 8 limbs multiplied each row): the 9-limb window needs x + p <= 2^256."""
    assert 0 <= x and x + P <= TWO256, "row operand too large for the 9-limb window"
    assert 0 <= y < TWO256
    t = x * y
    m = (-t * PINV) % TWO256
    r = (t + m * P) >> 256
    assert (t + m * P) & (TWO256 - 1) == 0
    assert r < TWO256, "montmul result overflows 8 limbs"
    Bounds.note(site, r)
    return r


def redc1(t: int, site: str = "redc1") -> int:
    """One Montgomery row on a 9-limb value: (t + m p)/2^32, m = -t mod 2^32 (p = 1 mod 2^32)."""
    assert 0 <= t < (1 << 288)
    m = (-t) & M32
    r = (t + m * P) >> 32
    assert r < TWO256
    Bounds.note(site, r)
    return r


def cfold(tab: Sequence[int], w: int, site: str = "cfold") -> int:
    """Constant fold (hades_device.cuh cfold): S = sum_j w_j tab[j] over the 32-bit limbs of w, then two Montgomery
    rows.  Equals C w / R (mod p) for tab = fold_table(C), like montmul(C, w), with a different representative."""
    assert 0 <= w < TWO256
    s = sum(((w >> (32 * j)) & M32) * t for j, t in enumerate(tab))
    assert s < 1 << 290, "fold sum overflows the 10-limb window"
    for _ in range(2):
        m = (-s) & M32
        s = (s + m * P) >> 32
    assert s < TWO256
    Bounds.note(site, s)
    return s


def condsub255(a: int) -> int:
    """if bit 255 set: a -= p   (=> a < 2^255 afterwards, since p > 2^254)."""
    if a >> 255:
        a -= P
    assert 0 <= a < (1 << 255)
    return a


def condsub(a: int) -> int:
    """full conditional subtraction, a < 2p -> [0,p)."""
    if a >= P:
        a -= P
    assert 0 <= a < P
    return a


def montsqr(a: int, site: str = "montsqr") -> int:
    """(a*a + m*p) / 2^256: product first (36 limb products), then eight Montgomery rows on the low half
    plus the high half.  No row-operand constraint; only the result must fit 8 limbs."""
    assert 0 <= a < TWO256
    t = a * a
    m = (-t * PINV) % TWO256
    r = (t + m * P) >> 256
    assert r < TWO256, "montsqr result overflows 8 limbs"
    Bounds.note(site, r)
    return r


def sbox(u: int, trace=None) -> int:
    a = montsqr(u, "sqr1")
    b = montsqr(a, "sqr2")
    x5 = montmul(u, b, "x5")
    if trace is not None:
        trace("sqr1", a)
        trace("sqr2", b)
        trace("x5", x5)
    return x5


def mix(z: Sequence[int], arc_next: Sequence[int] | None, trace=None) -> List[int]:
    """trace(lane, T): called with each lane's 9-limb total before the Montgomery row."""
    out = []
    zl = [limbs32(v) for v in z]
    for i in range(WIDTH):
        # every limb column must be exact in an IEEE double next to the 2^52 bias (FP64-pipe mix)
        for k in range(8):
            col = sum(CMAT[i][j] * zl[j][k] for j in range(WIDTH))
            assert col < (1 << 52) and float(col + (1 << 52)) == col + (1 << 52)
        t = sum(CMAT[i][j] * z[j] for j in range(WIDTH))
        if arc_next is not None:
            t += arc_next[i]
        if trace is not None:
            trace(i, t)
        out.append(redc1(t))
    return out


def permute_model(state_mont: Sequence[int], trace=None) -> List[int]:
    """state_mont: 5 integers < p in standard Montgomery form (BlsScalar.0 as an integer).
    Returns the permuted state in the same form -- must equal the reference bit for bit.

    trace(r, site, lane, value), if given, sees every intermediate integer: per round r the S-box
    input or linear lane `u`, the S-box's `sqr1`, `sqr2`, `x5` (full rounds; in partial rounds lane 4's `gfold` =
    cfold(G, u) and the corrected S-box output `gmul` = montmul(gfold, sqr2) instead of `x5`), and the
    mix total `T` that produces round r+1's `u` (round 67: the final mix); then, under r = ROUNDS,
    each lane's `final` value before the last conditional subtraction."""
    T = TABLES
    u = [condsub(s + a) for s, a in zip(state_mont, T.A[0])]
    for r in range(ROUNDS):
        def lane_trace(lane):
            return None if trace is None else (lambda name, v: trace(r, name, lane, v))
        if trace is not None:
            for i, x in enumerate(u):
                trace(r, "u", i, x)
        if is_full(r):
            z = [sbox(x, lane_trace(i)) for i, x in enumerate(u)]
        else:
            # lane 4: G u^5 / R^5 = montmul(cfold(G, u), u^4 / R^3); the fold of u runs beside the squarings
            gu = cfold(T.GT[r], u[4], "gfold")
            a = montsqr(u[4], "sqr1")
            b = montsqr(a, "sqr2")
            g = montmul(gu, b, "gmul")
            if trace is not None:
                for name, v in (("gfold", gu), ("sqr1", a), ("sqr2", b), ("gmul", g)):
                    trace(r, name, 4, v)
            z = list(u[:4]) + [g]
        mix_trace = None if trace is None else (lambda i, t: trace(r, "T", i, t))
        if r + 1 < ROUNDS:
            u = mix(z, T.A[r + 1], mix_trace)
        else:
            v = mix(z, None, mix_trace)
            w = [cfold(T.FT, x, "final") for x in v]
            if trace is not None:
                for i, x in enumerate(w):
                    trace(ROUNDS, "final", i, x)
            return [condsub(x) for x in w]
    raise AssertionError


def limbs32(v: int, n: int = 8) -> List[int]:
    return [(v >> (32 * i)) & M32 for i in range(n)]


def permute_dense(state_mont: Sequence[int]) -> List[int]:
    """The reference's dense formulation on canonical integers (src/hades/permutation.rs:105-123 with
    scalar.rs:39-64), used only to self-check the scaled-lazy model inside this build tool."""
    s = [x * R_INV % P for x in state_mont]
    for r in range(ROUNDS):
        s = [(x + ARC[r * WIDTH + i]) % P for i, x in enumerate(s)]
        if is_full(r):
            s = [pow(x, 5, P) for x in s]
        else:
            s[4] = pow(s[4], 5, P)
        s = [sum(MDS[i][j] * s[j] for j in range(WIDTH)) % P for i in range(WIDTH)]
    return [x * R % P for x in s]


if __name__ == "__main__":
    import random

    rnd = random.Random(7)
    cases = [[0] * 5, [1] * 5, [P - 1] * 5, [17] * 5, list(range(5))]
    cases += [[rnd.randrange(P) for _ in range(5)] for _ in range(100)]
    for c in cases:
        m = [x * R % P for x in c]
        assert permute_model(m) == permute_dense(m), c
    print("scaled-lazy model == dense formulation on", len(cases), "states")
    for k, v in sorted(Bounds.seen.items()):
        print("  max %-8s %.5f p   (2^256 = %.5f p)" % (k, v, TWO256 / P))
