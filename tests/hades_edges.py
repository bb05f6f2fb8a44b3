"""Test support (CPU): inputs that drive the scaled-lazy Hades (tools/hades_model.py, hades_device.cuh) through the
exact edges of its non-canonical arithmetic, at chosen rounds and lanes.

The kernel never reduces mod p between the first round-constant add and the output.  A lane of round r holds an
integer `u` with  true = kappa_r * u (mod p)  and u < p + 2^242; the last product lies in [0, 2p) before one
conditional subtraction.  The sites where a wrong comparison, a dropped carry or a bad table row shows are the
non-canonical ones: u == p (true value 0), u = s + p for a small or mid-sized class s, and a final value == p (an
output lane 0).  On random inputs each has a chance of about 1/p or 2^-16 per site, so they are constructed here:
Hades is invertible (the MDS is a Cauchy matrix; x^5 is a bijection on F_p because gcd(5, p-1) = 1), so a chosen
state at any round's S-box input, or at the output, is run backwards to the input that reaches it.

Sponge inputs have fixed lanes (the tag in lane 0, zero-padded rate lanes).  Through the round-0 S-box each fixed
input lane j is one linear equation in the round-1 state v:  (MDS^-1 (v - ARC_1))_j = (in_j + ARC_0,j)^5, so a round-1
target stays reachable while at least one lane is free.

All values are canonical integers unless a name says Montgomery (`mont`)."""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import hades_model as hm
import hades_oracle as o

P = o.P
W = o.WIDTH
ROUNDS = o.ROUNDS
ARC = o.ROUND_CONSTANTS
MDS = o.MDS_MATRIX
INV5 = pow(5, -1, P - 1)                  # x -> x^INV5 inverts the S-box
SEED = 2024


# ---- linear algebra mod p ----------------------------------------------------------------------------------------------
def solve(a: Sequence[Sequence[int]], b: Sequence[int]) -> List[int]:
    """x with a x = b (mod p), a square and invertible; Gauss-Jordan elimination."""
    n = len(a)
    m = [[v % P for v in row] + [bv % P] for row, bv in zip(a, b)]
    for c in range(n):
        piv = next(r for r in range(c, n) if m[r][c])
        m[c], m[piv] = m[piv], m[c]
        f = pow(m[c][c], -1, P)
        m[c] = [v * f % P for v in m[c]]
        for r in range(n):
            if r != c and m[r][c]:
                g = m[r][c]
                m[r] = [(v - g * w) % P for v, w in zip(m[r], m[c])]
    return [m[r][n] for r in range(n)]


def mat_inv(a: Sequence[Sequence[int]]) -> List[List[int]]:
    n = len(a)
    cols = [solve(a, [int(i == j) for i in range(n)]) for j in range(n)]
    return [[cols[j][i] for j in range(n)] for i in range(n)]


MDS_INV = mat_inv(MDS)


def matvec(a, v):
    return [sum(x * y for x, y in zip(row, v)) % P for row in a]


# ---- forward and inverse rounds --------------------------------------------------------------------------------------
def is_full(r: int) -> bool:
    return hm.is_full(r)


def state_at_round(x: Sequence[int], r: int) -> List[int]:
    """The oracle's state at round r's S-box input (after the round-constant add) for input x; r = ROUNDS: the output."""
    s = [v % P for v in x]
    for k in range(r):
        (o.apply_full_round if is_full(k) else o.apply_partial_round)(k, s)
    if r < ROUNDS:
        o.add_round_constants(r, s)
    return s


def _undo_sbox(r: int, z: List[int]) -> List[int]:
    if is_full(r):
        return [pow(v, INV5, P) for v in z]
    return z[:4] + [pow(z[4], INV5, P)]


def state_at_round_to_input(r: int, v: Sequence[int]) -> List[int]:
    """The input x whose state at round r's S-box input is v (0 <= r < ROUNDS)."""
    v = [t % P for t in v]
    for k in range(r, 0, -1):
        w = [(t - a) % P for t, a in zip(v, ARC[k])]
        v = _undo_sbox(k - 1, matvec(MDS_INV, w))
    return [(t - a) % P for t, a in zip(v, ARC[0])]


def output_to_input(y: Sequence[int]) -> List[int]:
    """perm^-1(y)."""
    return state_at_round_to_input(ROUNDS - 1, _undo_sbox(ROUNDS - 1, matvec(MDS_INV, y)))


def mont(x: int) -> int:
    return x * o.R % P


# ---- traced model ------------------------------------------------------------------------------------------------------
@dataclass
class Trace:
    """Every intermediate integer of one permutation of the model: site -> {(r, lane): value}."""
    sites: Dict[str, Dict[Tuple[int, int], int]] = field(default_factory=dict)
    out: List[int] = field(default_factory=list)

    def __call__(self, r, site, lane, value):
        self.sites.setdefault(site, {})[(r, lane)] = value

    def u(self, r, lane):
        return self.sites["u"][(r, lane)]

    def final(self, lane):
        return self.sites["final"][(ROUNDS, lane)]


def trace(x: Sequence[int]) -> Trace:
    """Trace the model on canonical input x (fed in Montgomery form, as the kernels take it)."""
    t = Trace()
    t.out = hm.permute_model([mont(v) for v in x], t)
    return t


def stored_class(r: int, true: int) -> int:
    """The residue mod p of round r's stored lane for a true value (true = kappa_r * stored)."""
    return true * pow(hm.TABLES.kappa[r], -1, P) % P


def true_of_class(r: int, s: int) -> int:
    return hm.TABLES.kappa[r] * s % P


# ---- raw-permutation corpus ------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """One constructed state.  kind names the edge; r the round (ROUNDS: the output), lanes the targeted lanes, s the
    stored class each targeted lane should hold (mod p), x the canonical input of the permutation that reaches it.
    `perm` is the index of the targeted permutation within a sponge item (0: the first), `data` the item's inputs."""
    kind: str
    r: int
    lanes: Tuple[int, ...]
    s: Optional[int]
    x: List[int]
    perm: int = 0
    data: Optional[List[int]] = None

    @property
    def name(self):
        return "%s@r%d/l%s" % (self.kind, self.r, "".join(map(str, self.lanes)))


# S-box / linear-lane targets at every (round 1..67, lane): stored u == p (true 0), u == 1 + p, u == p - 1, true +-1
U_KINDS = ("u_eq_p", "u_1_plus_p", "u_p_minus_1", "true_plus_1", "true_minus_1")
# u = s + p with s in [2^k, 2^(k+1)), kept where the model confirms u > p.  A mix output is below p + 2^242 and mostly
# below p + 2^241, so s >= 2^241 almost never lands above p; s near 2^240 does in a few percent of the sites.
S_PLUS_P_BITS = (238, 239, 240)


def _target_true(kind: str, r: int, rng) -> Tuple[int, int]:
    """(true value, stored class) of one targeted lane."""
    if kind == "u_eq_p":
        return 0, 0
    if kind == "u_1_plus_p":
        return true_of_class(r, 1), 1
    if kind == "u_p_minus_1":
        return true_of_class(r, P - 1), P - 1
    if kind == "true_plus_1":
        return 1, stored_class(r, 1)
    if kind == "true_minus_1":
        return P - 1, stored_class(r, P - 1)
    if kind.startswith("s_plus_p_"):
        k = int(kind.rsplit("_", 1)[1])
        s = rng.randrange(1 << k, 1 << (k + 1))
        return true_of_class(r, s), s
    raise ValueError(kind)


def _raw_case(kind, r, lanes, rng) -> Case:
    v = [rng.randrange(P) for _ in range(W)]
    s = None
    for lane in lanes:
        v[lane], s = _target_true(kind, r, rng)
    return Case(kind, r, tuple(lanes), s, state_at_round_to_input(r, v))


def _s_plus_p_case(r, lane, k, rng) -> Optional[Case]:
    """A case with stored class s in [2^k, 2^(k+1)) at (r, lane), or None if the model stores s rather than s + p."""
    c = _raw_case("s_plus_p_%d" % k, r, (lane,), rng)
    return c if trace(c.x).u(r, lane) == c.s + P else None


@functools.lru_cache(maxsize=None)
def raw_corpus() -> Tuple[Case, ...]:
    """Every (round 1..67, lane) with each U_KINDS edge and the s + p edges the model confirms; round 0's first add at
    true 0, true p - 1 and stored p - 1; all five lanes zero at rounds 1, 3, 64, 67; output lanes 0 and p - 1 (canonical
    and Montgomery), and perm^-1(0)."""
    rng = random.Random(SEED)
    cases = []
    for lane in range(W):
        for kind in ("true_zero", "true_minus_1", "u_p_minus_1"):
            true = {"true_zero": 0, "true_minus_1": P - 1, "u_p_minus_1": true_of_class(0, P - 1)}[kind]
            v = [rng.randrange(P) for _ in range(W)]
            v[lane] = true
            cases.append(Case("r0_" + kind, 0, (lane,), stored_class(0, true), state_at_round_to_input(0, v)))
    for r in range(1, ROUNDS):
        for lane in range(W):
            for kind in U_KINDS:
                cases.append(_raw_case(kind, r, (lane,), rng))
            kept = [c for c in (_s_plus_p_case(r, lane, k, rng) for k in S_PLUS_P_BITS) if c]
            k = S_PLUS_P_BITS[0]
            while not kept and k > 200:              # none landed above p: smaller classes until one does
                k -= 1
                kept = [c for c in [_s_plus_p_case(r, lane, k, rng)] if c]
            cases += kept
    for r in (1, 3, 64, ROUNDS - 1):
        cases.append(_raw_case("u_eq_p", r, tuple(range(W)), rng))
    for lane in range(W):
        for kind, y in (("out_zero", 0), ("out_minus_1", P - 1), ("out_mont_minus_1", (P - 1) * o.R_INV % P)):
            out = [rng.randrange(P) for _ in range(W)]
            out[lane] = y
            cases.append(Case(kind, ROUNDS, (lane,), mont(y), output_to_input(out)))
    cases.append(Case("out_zero", ROUNDS, tuple(range(W)), 0, output_to_input([0] * W)))
    return tuple(cases)


# ---- sponge corpora ----------------------------------------------------------------------------------------------------
def constrained_input(fixed: Dict[int, int], r: int, targets: Dict[int, int], rng) -> List[int]:
    """A permutation input whose lanes in `fixed` hold the given values and whose state at round r (0 or 1) holds the
    true values `targets` on the targeted lanes; every other choice random."""
    if r == 0:
        x = [rng.randrange(P) for _ in range(W)]
        for j, t in targets.items():
            assert j not in fixed
            x[j] = (t - ARC[0][j]) % P
        for j, c in fixed.items():
            x[j] = c
        return x
    assert r == 1
    # unknowns: the untargeted round-1 lanes; len(fixed) of them are solved for, the rest random
    unknown = [j for j in range(W) if j not in targets]
    assert len(unknown) >= len(fixed), "no round-1 freedom left"
    v = [0] * W
    for j, t in targets.items():
        v[j] = t
    rand, solved = unknown[:len(unknown) - len(fixed)], unknown[len(unknown) - len(fixed):]
    for j in rand:
        v[j] = rng.randrange(P)
    rows = sorted(fixed)
    # fixed lane i:  sum_k MDS_INV[i][k] v_k = (c_i + ARC_0,i)^5 + sum_k MDS_INV[i][k] ARC_1,k
    a = [[MDS_INV[i][k] for k in solved] for i in rows]
    b = [(pow(fixed[i] + ARC[0][i], 5, P) + sum(MDS_INV[i][k] * ARC[1][k] for k in range(W))
          - sum(MDS_INV[i][k] * v[k] for k in range(W) if k not in solved)) % P for i in rows]
    for k, val in zip(solved, solve(a, b)):
        v[k] = val
    x = state_at_round_to_input(1, v)
    assert all(x[i] == fixed[i] % P for i in fixed), "fixed lanes not reproduced"
    return x


def hash_tag(domain: int, in_len: int, out_len: int) -> int:
    return o.hash_to_scalar(o.tag_input([o.Absorb(in_len), o.Squeeze(out_len)], domain))


def crypt_tag(L: int) -> int:
    return o.hash_to_scalar(o.tag_input([o.Absorb(2), o.Absorb(1), o.Squeeze(L), o.Absorb(L), o.Squeeze(1)],
                                        o.Domain.Encryption))


SPONGE_KINDS = (("u_eq_p", 1), ("u_1_plus_p", 1), ("u_p_minus_1", 1), ("r0_true_zero", 0), ("r0_true_minus_1", 0))


def _sponge_cases(fixed: Dict[int, int], free: Sequence[int], rng, perm=0) -> List[Case]:
    """Round-1 edges on every lane (a fixed lane too: the round-1 state has freedom left) and round-0 edges on the free
    lanes of one permutation whose fixed input lanes are `fixed`."""
    cases = []
    for kind, r in SPONGE_KINDS:
        for lane in (range(W) if r == 1 else free):
            if r == 1:
                true, s = _target_true(kind, 1, rng)
            else:
                true = 0 if kind == "r0_true_zero" else P - 1
                s = stored_class(0, true)
            x = constrained_input(fixed, r, {lane: true}, rng)
            cases.append(Case(kind, r, (lane,), s, x, perm))
    return cases


@dataclass(frozen=True)
class DigestCorpus:
    domain: str
    in_len: int
    out_len: int
    tag: int
    cases: Tuple[Case, ...]          # case.data: the item's in_len inputs; case.x: the targeted permutation's input

    @property
    def data(self) -> List[List[int]]:
        return [c.data for c in self.cases]


DIGEST_SHAPES = (("Merkle4", 4, 1), ("Merkle2", 2, 1), ("Other", 3, 1), ("Other", 8, 5))


@functools.lru_cache(maxsize=None)
def digest_corpus(domain: str, in_len: int, out_len: int) -> DigestCorpus:
    """Digest items whose first permutation (and, for in_len in 5..8, also the second absorb permutation) reaches the
    SPONGE_KINDS edges.  The first permutation's input is [tag, d_1, .., d_k, 0, ..]; the second's lane 0 is fixed by
    the first permutation and its lanes 1..4 are free through d_5..d_8."""
    assert in_len <= 8
    rng = random.Random("digest-%d-%s-%d-%d" % (SEED, domain, in_len, out_len))
    tag = hash_tag(getattr(o.Domain, domain), in_len, out_len)
    k = min(in_len, 4)
    fixed = {0: tag}
    fixed.update({j: 0 for j in range(k + 1, W)})
    cases = []
    for c in _sponge_cases(fixed, range(1, k + 1), rng):
        c.data = c.x[1:k + 1] + [rng.randrange(P) for _ in range(in_len - k)]
        cases.append(c)
    if in_len > 4:
        # second absorb permutation: input [s1_0, s1_1 + d_5, .., s1_4 + d_8] for the first permutation's output s1
        head = [rng.randrange(P) for _ in range(4)]
        s1 = o.perm([tag] + head)
        free2 = list(range(1, in_len - 3))
        for c in _sponge_cases({j: s1[j] for j in range(W) if j not in free2}, free2, rng, perm=1):
            c.data = head + [(c.x[j] - s1[j]) % P for j in free2]
            cases.append(c)
    return DigestCorpus(domain, in_len, out_len, tag, tuple(cases))


@dataclass(frozen=True)
class CryptCorpus:
    L: int
    tag: int
    cases: Tuple[Case, ...]          # case.data: [u, v, nonce]; case.x: [tag, u, v, nonce, 0]
    messages: Tuple[Tuple[int, ...], ...]


@functools.lru_cache(maxsize=None)
def crypt_corpus(L: int) -> CryptCorpus:
    """Encryptions of L-scalar messages whose first permutation [tag, u, v, nonce, 0] reaches the SPONGE_KINDS edges
    (two fixed lanes); the messages are random."""
    rng = random.Random("crypt-%d-%d" % (SEED, L))
    tag = crypt_tag(L)
    cases = _sponge_cases({0: tag, 4: 0}, (1, 2, 3), rng)
    for c in cases:
        c.data = c.x[1:4]
    msgs = tuple(tuple(rng.randrange(P) for _ in range(L)) for _ in cases)
    return CryptCorpus(L, tag, tuple(cases), msgs)
