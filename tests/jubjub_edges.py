"""Test support (CPU): JubJub points whose coordinates, Niels components and products sit at the edges of the field, and
the inputs that place such a point on a kernel's input, on a fixed-base table entry or on a result.

The device holds a coordinate as its Montgomery image m = x R mod p (8 x u32, fully reduced, jubjub_device.cuh), so the
edges are edges of m: p - 1 (the largest canonical value), a value whose top limb equals p's top limb (where a reduction
that looks at the top limb alone would go wrong), an all-ones limb, a sum m_u + m_v just below or just above p (where
fr_add_mod's conditional subtraction flips), a difference m_v - m_u that borrows by one, and a product T = u v at 1 or
p - 1.  A random point reaches one of them with a chance between 2^-32 and 2^-250 per operation, so they are constructed.

Classes (`Edge.kind`), the site each reaches, and why it reaches it:

  "u", "v"    m_u or m_v is a value of M.  (u, v) = a solution of the curve equation for the other coordinate.
              As an input (dhke public, stealth A / B, scan R, host-read base / spend_B) the limbs are consumed as they are
              by fr_is_canonical, on_curve, to_cached / to_niels and the host checks; as a table entry (below) they are the
              outputs of the affine conversion fmul(X, 1/Z) and its fr_condsub; as a result, the same last two fmuls.
  "sum"       m_u + m_v = p +- k as integers, k = 1..4: the Niels / cached Y + X of fr_add_mod (to_cached, to_niels,
              fixed_base_entry) and of the host's add_mod (jubjub_niels), just below p and just above it (the
              subtraction runs).  p +- 1 have no point; p - 2 and p + 2 are the closest.
  "diff"      m_v - m_u = +-k, k = 1..4, and +-2^32, +-(2^32 - 1): Y - X of fr_sub_mod / the host's sub_mod with and
              without the borrow (a borrow by 2 leaves p - 2).  With v = u + c the curve equation is the quartic
              d u^4 + 2cd u^3 + dc^2 u^2 - 2c u - (c^2 - 1) = 0 (a sum is the same with u -> -u), solved by `roots`.
              m_u + m_v = p and v = +-u are impossible: c = 0 leaves d u^4 = -1, and -1/d is not a square.
  "uv"        Mont(u v) at 1..40, p - 1, p - 2, p - 3 and limb edges: the T = fmul(u, v) of the input point
              (scalar_mul, fixed_base_entry, to_niels) and of the host's mont_mul.
  "kt"        Mont(2d u v) at k and p - k, k = 1..7 (the first with a point is 6): the Niels / cached 2d T, and
              select_niels' negation 0 - kt = p - k / k when a negative digit selects the entry.  With v = c / u the
              curve equation is a quadratic in u^2.

Every class also has prime-subgroup members (`subgroup_edges`, [r_J] E = O), searched past the named targets where none
of them is in the subgroup; a table entry (w, j) can only be placed at a subgroup point in general.

Placements (the group is cyclic of order 8 r_J, and the fixed-base and stealth calls take their base as an argument):
  output      [s] P = Q for odd s < r_J and P = [s^-1 mod 8 r_J] Q: k_dhke's public, k_fixed_base's base.  The result is
              the last two fmuls of the affine conversion and their fr_condsub.
  table       entry (w, j) = j 16^w B = E for B = [(j 16^w)^-1 mod r_J] E: the affine entry is Niels-formed right after the
              inversion (fixed_base_entry), then selected, swapped and negated by select_niels.  Paired with secrets whose
              signed recoding selects the entry with every sign it can take there (magnitude 8 only as -8, window 63 only
              +1).
  stealth     the sender's note_pk = Q for B = Q - [h] G, h = hash([r] A); R = Q for G = [r^-1 mod 8 r_J] Q.  The scan's
              note_pk = Q for spend_B = Q - [h] G, h = hash([a] R).
  boundary    raw coordinate limbs m + p, m + 2p and 2^256 - 1 (2p < 2^256 < 3p) whose residue is a curve coordinate:
              only the canonical check tells them from their valid twin (m, the other coordinate).

Values named Montgomery (`m`, `mont`) are the limbs the device sees; everything else is a canonical integer."""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

import hades_oracle as ho
import jubjub_oracle as jo
import stealth_oracle as so

P = jo.P
R = ho.R                      # 2^256 mod p: the Montgomery image of 1
R_INV = ho.R_INV
D = jo.D
R_J = jo.R_J
N8 = 8 * R_J                  # the order of the full group
G = jo.GENERATOR
TOP = P >> 224                # p's top 32-bit limb


def mont(x: int) -> int:
    return x % P * R % P


def unmont(m: int) -> int:
    return m % P * R_INV % P


# ---- the edge value set M (Montgomery values) ---------------------------------------------------------------------------
def _dedupe(pairs):
    seen, out = set(), []
    for name, v in pairs:
        if v not in seen:
            seen.add(v)
            out.append((name, v))
    return tuple(out)


M: Tuple[Tuple[str, int], ...] = _dedupe(
    [("0", 0), ("1", 1), ("2", 2), ("3", 3), ("p-1", P - 1), ("p-2", P - 2), ("p-3", P - 3), ("(p-1)/2", (P - 1) // 2),
     ("(p+1)/2", (P + 1) // 2), ("R", R), ("2^32-1", (1 << 32) - 1), ("2^32", 1 << 32), ("2^64-1", (1 << 64) - 1),
     ("2^64", 1 << 64), ("2^128-1", (1 << 128) - 1), ("2^224-1", (1 << 224) - 1), ("2^224", 1 << 224),
     ("2^254-1", (1 << 254) - 1), ("2^254", 1 << 254), ("p-2^32", P - (1 << 32)), ("p-2^64", P - (1 << 64)),
     ("p-2^192", P - (1 << 192))]
    + [("limb%d" % k, 0xffffffff << (32 * k)) for k in range(7)])
# the values of M whose top limb is p's: a reduction deciding on the top limb alone subtracts p from them
TOP_LIMB_NAMES = tuple(name for name, m in M if m >> 224 == TOP)

# The sums, differences and products closest to each edge that have points; the ones without are pinned by the CPU test.
SUM_TARGETS = tuple(("p%+d" % k, P + k) for k in (-1, 1, -2, 2, -3, 3, -4, 4))             # m_u + m_v
DIFF_TARGETS = tuple((str(k), k) for k in (1, -1, 2, -2, 3, -3, 4, -4)) + (
    ("2^32", 1 << 32), ("-2^32", -(1 << 32)), ("2^32-1", (1 << 32) - 1), ("-(2^32-1)", 1 - (1 << 32)))   # m_v - m_u
UV_TARGETS = tuple((str(k), k) for k in range(1, 41)) + (
    ("p-1", P - 1), ("p-2", P - 2), ("p-3", P - 3), ("2^32-1", (1 << 32) - 1), ("2^32", 1 << 32),
    ("2^64-1", (1 << 64) - 1), ("p-2^32", P - (1 << 32)), ("p-2^64", P - (1 << 64)), ("R", R))   # Mont(u v)
KT_TARGETS = tuple((n, t) for k in range(1, 8) for n, t in ((str(k), k), ("p-%d" % k, P - k)))   # Mont(2d u v)
KINDS = ("u", "v", "sum", "diff", "uv", "kt")


@dataclass(frozen=True)
class Edge:
    kind: str                 # one of KINDS
    name: str                 # the named edge, e.g. "p-1"
    target: int               # the value the site sees (Montgomery; an integer sum or difference for "sum" / "diff")
    pt: Tuple[int, int]       # canonical affine (u, v)

    @property
    def label(self):
        return "%s=%s" % (self.kind, self.name)


def site_value(kind: str, pt) -> int:
    """The value of a point at the site of `kind`, computed from its coordinates: what Edge.target claims."""
    u, v = pt
    return {"u": mont(u), "v": mont(v), "sum": mont(u) + mont(v), "diff": mont(v) - mont(u), "uv": mont(u * v),
            "kt": mont(2 * D * u * v)}[kind]


# ---- polynomials over F_q and their roots -------------------------------------------------------------------------------
# coefficient lists, lowest degree first, no trailing zeros ([] is the zero polynomial)
def _trim(a):
    while a and a[-1] == 0:
        a.pop()
    return a


def _divmod(a, b, q):
    a = _trim([x % q for x in a])
    inv, db = pow(b[-1], -1, q), len(b) - 1
    quo = [0] * max(len(a) - db, 0)
    while len(a) - 1 >= db:
        f, s = a[-1] * inv % q, len(a) - 1 - db
        quo[s] = f
        for i, c in enumerate(b):
            a[s + i] = (a[s + i] - f * c) % q
        _trim(a)
    return quo, a


def _mulmod(a, b, m, q):
    r = [0] * (len(a) + len(b) - 1) if a and b else []
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            r[i + j] = (r[i + j] + x * y) % q
    return _divmod(r, m, q)[1]


def _powmod(a, e, m, q):
    r, a = [1], _divmod(a, m, q)[1]
    while e:
        if e & 1:
            r = _mulmod(r, a, m, q)
        a = _mulmod(a, a, m, q)
        e >>= 1
    return r


def _sub(a, b, q):
    n = max(len(a), len(b))
    return _trim([((a[i] if i < len(a) else 0) - (b[i] if i < len(b) else 0)) % q for i in range(n)])


def _gcd(a, b, q):
    a, b = _trim([x % q for x in a]), _trim([x % q for x in b])
    while b:
        a, b = b, _divmod(a, b, q)[1]
    inv = pow(a[-1], -1, q)
    return [x * inv % q for x in a]


def roots(f: Sequence[int], q: int = P, seed: int = 1) -> List[int]:
    """The distinct roots in F_q (q an odd prime) of f: gcd(f, x^q - x) keeps the product of f's linear factors, then
    equal-degree splitting (Cantor-Zassenhaus) by gcd(g, (x + a)^((q-1)/2) - 1) for random a."""
    f = _trim([x % q for x in f])
    if len(f) < 2:
        return []
    g = _gcd(f, _sub(_powmod([0, 1], q, f, q), [0, 1], q), q)
    rng, out = random.Random(seed), []

    def split(g):
        d = len(g) - 1
        if d == 1:
            out.append(-g[0] % q)
        while d > 1:
            k = _gcd(g, _sub(_powmod([rng.randrange(q), 1], (q - 1) // 2, g, q), [1], q), q)
            if 0 < len(k) - 1 < d:
                split(k)
                split(_divmod(g, k, q)[0])
                return

    split(g)
    return sorted(out)


def quartic(c: int) -> List[int]:
    """The curve equation with v = u + c as a polynomial in u: d u^4 + 2cd u^3 + dc^2 u^2 - 2c u - (c^2 - 1)."""
    return [(1 - c * c) % P, -2 * c % P, D * c * c % P, 2 * c * D % P, D]


# ---- solving the curve equation for one coordinate ---------------------------------------------------------------------
def v_from_u(u: int) -> List[int]:
    """Every v with (u, v) on the curve: v^2 = (1 + u^2) / (1 - d u^2) (1 - d u^2 != 0: d is not a square)."""
    r = jo.sqrt((1 + u * u) * pow((1 - D * u * u) % P, -1, P))
    return [] if r is None else sorted({r, -r % P})


def u_from_v(v: int) -> List[int]:
    pt = jo.point_from_v(v)
    return [] if pt is None else sorted({pt[0], -pt[0] % P})


def points_with_uv(c: int) -> List[Tuple[int, int]]:
    """Every curve point with u v = c != 0: with v = c / u, u^4 + (1 + d c^2) u^2 - c^2 = 0, a quadratic in u^2."""
    b = (1 + D * c * c) % P
    s = jo.sqrt(b * b + 4 * c * c)
    if s is None:
        return []
    pts = set()
    for w in ((-b + s) * pow(2, -1, P) % P, (-b - s) * pow(2, -1, P) % P):
        r = jo.sqrt(w)
        for u in ({r, -r % P} if r else ()):
            pts.add((u, c * pow(u, -1, P) % P))
    return sorted(pts)


def _class(kind: str, name: str, t: int) -> List[Edge]:
    """Every point of one class whose site value is exactly t (an integer sum or difference is checked as such)."""
    if kind == "u":
        pts = [(unmont(t), v) for v in v_from_u(unmont(t))]
    elif kind == "v":
        pts = [(u, unmont(t)) for u in u_from_v(unmont(t))]
    elif kind in ("sum", "diff"):
        c = unmont(t)
        us = [-x % P for x in roots(quartic(c))] if kind == "sum" else roots(quartic(c))
        pts = [(u, (c - u) % P if kind == "sum" else (u + c) % P) for u in us]
    elif kind == "uv":
        pts = points_with_uv(unmont(t))
    else:
        pts = points_with_uv(unmont(t) * pow(2 * D, -1, P) % P)
    return [Edge(kind, name, t, pt) for pt in sorted(pts) if site_value(kind, pt) == t]


_TARGETS = {"u": M, "v": M, "sum": SUM_TARGETS, "diff": DIFF_TARGETS, "uv": UV_TARGETS, "kt": KT_TARGETS}


@functools.lru_cache(maxsize=None)
def edges(kind: str) -> Tuple[Edge, ...]:
    """Every point of the class at its named targets, in target order."""
    return tuple(e for name, t in _TARGETS[kind] for e in _class(kind, name, t))


@functools.lru_cache(maxsize=None)
def all_edges() -> Tuple[Edge, ...]:
    return tuple(e for k in KINDS for e in edges(k))


@functools.lru_cache(maxsize=None)
def no_point() -> Tuple[Tuple[str, str], ...]:
    """(kind, name) of every named target that no curve point reaches."""
    return tuple((k, name) for k in KINDS for name, t in _TARGETS[k] if not _class(k, name, t))


# ---- scalar multiples (memoized: the oracle's double-and-add costs ~25 ms per 252-bit scalar) ----------------------
@functools.lru_cache(maxsize=None)
def mul(k: int, pt) -> Tuple[int, int]:
    return jo.mul(k, tuple(pt))


def in_subgroup(pt) -> bool:
    return mul(R_J, pt) == jo.IDENTITY


@functools.lru_cache(maxsize=None)
def subgroup_edges() -> Tuple[Edge, ...]:
    """One prime-subgroup point of every class other than the identity: the first in class order with [r_J] E = O
    (about one point in 8; every class has one)."""
    return tuple(next(e for e in edges(k) if e.pt != jo.IDENTITY and in_subgroup(e.pt)) for k in KINDS)


# ---- placements ---------------------------------------------------------------------------------------------------------
OUTPUT_SECRETS = (3, int("f" * 62, 16), R_J - 2, (1 << 251) + 1)     # odd, < r_J
OUTPUT_COORD_NAMES = TOP_LIMB_NAMES + ("0", "1", "R", "2^254-1", "limb3")


@functools.lru_cache(maxsize=None)
def output_edges() -> Tuple[Edge, ...]:
    """The results placed at an edge: every sum / diff / uv / kt point and the coordinate points at the top-limb values
    (where a reduction deciding on the top limb alone goes wrong) and a few others."""
    return tuple(e for e in all_edges() if e.kind not in ("u", "v") or e.name in OUTPUT_COORD_NAMES)


@functools.lru_cache(maxsize=None)
def output_placements() -> Tuple[Tuple[Edge, int, Tuple[int, int]], ...]:
    """(Q, s, P) with [s] P = Q: P = [s^-1 mod 8 r_J] Q (s odd, so invertible mod 8 r_J; Q's order divides 8 r_J)."""
    out = []
    for i, e in enumerate(output_edges()):
        s = OUTPUT_SECRETS[i % len(OUTPUT_SECRETS)]
        out.append((e, s, mul(pow(s, -1, N8), e.pt)))
    return tuple(out)


WINDOWS = 64
TABLE_ENTRIES = ((0, 1), (0, 8), (1, 1), (62, 8), (63, 1))


def recode(s: int) -> List[int]:
    """The kernel's signed 4-bit recoding (recode_digit): 64 digits in [-8, 8), least significant first."""
    digits, carry = [], 0
    for _ in range(WINDOWS):
        x = (s & 15) + carry
        s >>= 4
        carry = (x + 8) >> 4
        digits.append(x - (carry << 4))
    return digits


def signs_at(w: int, j: int) -> Tuple[int, ...]:
    """The digit signs the recoding can give entry (w, j): magnitude 8 only as -8, window 63 only 0 or +1."""
    if w == WINDOWS - 1:
        return (1,) if j == 1 else ()
    return (-1,) if j == 8 else (1, -1)


def secret_selecting(w: int, e: int, seed: int) -> int:
    """A secret s < r_J whose recoding has digit e at window w, every other digit random."""
    rng = random.Random("select-%d-%d-%d" % (w, e, seed))
    while True:
        d = [rng.randrange(-8, 8) for _ in range(WINDOWS - 1)] + [rng.randrange(0, 2)]
        d[w] = e
        s = sum(x << (4 * k) for k, x in enumerate(d))
        if 0 <= s < R_J:
            assert recode(s) == d
            return s


@dataclass(frozen=True)
class TablePlacement:
    w: int
    j: int
    edge: Edge                          # the entry's point
    base: Tuple[int, int]               # B with j 16^w B = edge.pt
    secrets: Tuple[Tuple[int, int], ...]   # (sign, s): s selects entry (w, j) with that sign


@functools.lru_cache(maxsize=None)
def table_placements() -> Tuple[TablePlacement, ...]:
    """Every entry of TABLE_ENTRIES at every class's subgroup point; entry (0, 1) also at the first point of every
    class (any order: B = E)."""
    out = []
    for w, j in TABLE_ENTRIES:
        es = subgroup_edges() + (tuple(edges(k)[0] for k in KINDS) if (w, j) == (0, 1) else ())
        for i, e in enumerate(es):
            k = j << (4 * w)
            base = e.pt if k == 1 else mul(pow(k, -1, R_J), e.pt)
            secs = tuple((sg, secret_selecting(w, sg * j, i)) for sg in signs_at(w, j))
            out.append(TablePlacement(w, j, e, base, secs))
    return tuple(out)


# ---- stealth placements -------------------------------------------------------------------------------------------------
STEALTH_R = 0x0bad_5eed_0dd_c0ffee_1234567 | 1          # the sender's r (odd) for the placements
SCAN_A, SCAN_B = 0x5ca1ab1e_7ea_f00d, 0xb0b_cafe_b0ba      # the receiver's view key a and spend key b


def hash_point(pt) -> int:
    return so.hash_point(pt)


@functools.lru_cache(maxsize=None)
def receiver():
    """(a, A, B) = (view key, [a] G, [b] G)"""
    return SCAN_A, mul(SCAN_A, G), mul(SCAN_B, G)


@functools.lru_cache(maxsize=None)
def sender_hG(r: int = STEALTH_R, G_: Tuple[int, int] = G) -> Tuple[int, int]:
    """[hash([r] A)] G for the receiver's A"""
    _, A, _ = receiver()
    return mul(hash_point(mul(r, A)), G_)


def note_pk_placement(Q) -> Tuple[int, int]:
    """B with note_pk = [hash([r] A)] G + B = Q (r = STEALTH_R)"""
    return jo.add(Q, jo.neg(sender_hG()))


@functools.lru_cache(maxsize=None)
def R_placement(Q) -> Tuple[Tuple[int, int], Tuple[int, int], Tuple[int, int]]:
    """(G', B', note_pk) for R = [r] G' = Q: G' = [r^-1 mod 8 r_J] Q, B' = [b] G', note_pk = [hash([r] A)] G' + B'"""
    Gq = mul(pow(STEALTH_R, -1, N8), Q)
    B = mul(SCAN_B, Gq)
    return Gq, B, jo.add(sender_hG(STEALTH_R, Gq), B)


@functools.lru_cache(maxsize=None)
def scan_note():
    """(R, [hash([a] R)] G) of one note the receiver scans: R = [r] G"""
    Rp = mul(STEALTH_R, G)
    return Rp, mul(hash_point(mul(SCAN_A, Rp)), G)


def spend_B_placement(Q) -> Tuple[int, int]:
    """spend_B with the scan's note key [hash([a] R)] G + spend_B = Q"""
    return jo.add(Q, jo.neg(scan_note()[1]))


def near_misses(Q) -> List[Tuple[str, Tuple[int, int]]]:
    """Canonical points next to Q that are not Q: -Q, Q + (0, -1), the coordinates swapped, v + 1 and v - 1."""
    u, v = Q
    cands = [("neg", jo.neg(Q)), ("plus_t2", jo.add(Q, (0, P - 1))), ("swap", (v, u)), ("v+1", (u, (v + 1) % P)),
             ("v-1", (u, (v - 1) % P))]
    return [(n, c) for n, c in cands if c != tuple(Q)]


# ---- exact-boundary invalid inputs ----------------------------------------------------------------------------------
BOUNDARY_RAW = (("p", P), ("p+1", P + 1), ("2p-1", 2 * P - 1), ("2p", 2 * P), ("2p+1", 2 * P + 1),
                ("2^256-1", (1 << 256) - 1))


@dataclass(frozen=True)
class Boundary:
    name: str                   # e.g. "u=2p-1"
    raw: Tuple[int, int]        # Montgomery limbs as ints, one coordinate >= p
    twin: Tuple[int, int]       # the same residues, canonical: a curve point

    @property
    def pt(self):
        return unmont(self.twin[0]), unmont(self.twin[1])


@functools.lru_cache(maxsize=None)
def boundaries() -> Tuple[Boundary, ...]:
    """Every raw value of BOUNDARY_RAW as u and as v wherever its residue is a curve coordinate, the other coordinate
    solved for (the first root)."""
    out = []
    for name, x in BOUNDARY_RAW:
        m = x % P
        for v in v_from_u(unmont(m))[:1]:
            out.append(Boundary("u=" + name, (x, mont(v)), (m, mont(v))))
        for u in u_from_v(unmont(m))[:1]:
            out.append(Boundary("v=" + name, (mont(u), x), (mont(u), m)))
    return tuple(out)


# ---- device rows ------------------------------------------------------------------------------------------------------
def raw_rows(pairs) -> np.ndarray:
    """(m_u, m_v) raw Montgomery ints (any value < 2^256) -> (n, 2, 4) uint64"""
    out = np.zeros((len(pairs), 2, 4), dtype=np.uint64)
    for i, pair in enumerate(pairs):
        for j, c in enumerate(pair):
            for k in range(4):
                out[i, j, k] = (c >> (64 * k)) & ((1 << 64) - 1)
    return out


def rows(points) -> np.ndarray:
    """canonical affine points -> (n, 2, 4) Montgomery rows"""
    return raw_rows([(mont(u), mont(v)) for u, v in points])
