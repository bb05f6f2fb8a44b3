"""Generator for poseidon252_b200/csrc/fr_ptx.cuh: the carry-chain primitives of the B200 Hades
kernel as inline-PTX blocks (mad.lo.cc / madc.hi.cc pairs that ptxas fuses into IMAD.WIDE.U32[.X]).

Every primitive is first built as a small IR (list of PTX ops on named 32-bit registers), which
  * `Prog.run` EMULATES instruction by instruction (32-bit wrap, CC.CF carry flag, predicates) so
    the sequences are verified here, without a GPU, against the integer definitions in
    tools/hades_model.py (see tests/test_field_ptx.py), and
  * `Prog.emit` prints as one `asm` statement per primitive (no carry flag ever crosses an asm
    boundary).
Ops tagged nocarry=True are the chain ends where the analysis says no carry can leave; the
emulator asserts that.

Field: BLS12-381 Fr, 8 x 32-bit limbs, p = 1 mod 2^32  =>  the Montgomery digit is m = -t0 and
m*p0 needs no multiplier (p0 = 1): 15 IMAD.WIDE per interleaved row instead of 16.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List, Sequence, Union

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hades_model import P, M32  # noqa: E402

PL = [(P >> (32 * i)) & M32 for i in range(8)]
assert PL[0] == 1 and PL[1] == M32
# p1 = 2^32 - 1: m*p1 = (m << 32) - m, i.e. lo = -m = w0 (the limb being cancelled) and hi = m - (m != 0).
# With P1_ALU the two halves are formed on the ALU pipe (borrow of 0 - w0) instead of an IMAD.HI.
P1_ALU = os.environ.get("P252_P1_ALU", "0") == "1"
FUSE_FRESH = os.environ.get("P252_FUSE_FRESH", "1") == "1"

Operand = Union[str, int]


class Prog:
    def __init__(self, name: str, doc: str):
        self.name, self.doc = name, doc
        self.ops: List[tuple] = []
        self.ins: List[str] = []        # read-only C operands
        self.outs: List[str] = []       # write-only C operands
        self.inouts: List[str] = []     # read-write C operands
        self.temps: List[str] = []
        self.preds: List[str] = []

    # -- declaration helpers
    def inp(self, *names):
        self.ins += names
        return names if len(names) > 1 else names[0]

    def out(self, *names):
        self.outs += names
        return names if len(names) > 1 else names[0]

    def inout(self, *names):
        self.inouts += names
        return names if len(names) > 1 else names[0]

    def tmp(self, *names):
        self.temps += names
        return names if len(names) > 1 else names[0]

    def pred(self, name):
        self.preds.append(name)
        return name

    def op(self, opc: str, d: str, *src: Operand, nocarry: bool = False, guard: str | None = None):
        self.ops.append((opc, d, src, nocarry, guard))

    # -- emulator
    def run(self, env: Dict[str, int]) -> Dict[str, int]:
        reg = dict(env)
        cf = 0
        cf_kind = None          # "add" or "sub": which flavour produced the live carry flag
        preds: Dict[str, bool] = {}

        def val(x):
            return x & M32 if isinstance(x, int) else reg[x]

        for opc, d, src, nocarry, guard in self.ops:
            if guard is not None and not preds[guard]:
                continue
            base = opc.split(".")[0]
            if base == "setp":          # setp.ge.u32 p, a, b
                cmp = opc.split(".")[1]
                a, b = val(src[0]), val(src[1])
                preds[d] = {"ge": a >= b, "eq": a == b, "ne": a != b, "lt": a < b}[cmp]
                continue
            if base == "selp":          # selp d, a, b, p
                reg[d] = val(src[0]) if preds[src[2]] else val(src[1])
                continue
            if base == "mov":
                reg[d] = val(src[0])
                continue
            if base == "mulwide":       # (lo|hi) = a * b as ONE 64-bit product (mul.wide.u32 + mov.b64 unpack)
                lo, hi = d.split("|")
                prod = val(src[0]) * val(src[1])
                reg[lo], reg[hi] = prod & M32, prod >> 32
                continue
            if base == "and":
                reg[d] = val(src[0]) & val(src[1])
                continue
            if base == "min":
                reg[d] = min(val(src[0]), val(src[1]))
                continue
            if base == "shf":           # shf.l.wrap.b32 d, lo, hi, n : upper word of (hi:lo) << n
                n = val(src[2]) & 31
                reg[d] = (((val(src[1]) << 32) | val(src[0])) << n >> 32) & M32
                continue
            uses_c = base.endswith("c") and base in ("madc", "addc", "subc")
            sets_cc = opc.endswith(".cc.u32") or ".cc" in opc
            cin = cf if uses_c else 0
            kind = "sub" if base in ("sub", "subc") else "add"
            if uses_c:
                # On the GPU a borrow written by sub.cc is NOT a carry for addc/madc (and vice versa) even though
                # PTX names one flag: found on the GPU (DESIGN.md, alternatives).  Never mix flavours.
                assert cf_kind == kind, "carry chain mixes add and sub flavours in %s at %s" % (self.name, opc)
            if sets_cc:
                cf_kind = kind
            if base in ("mul",):
                prod = val(src[0]) * val(src[1])
                full = (prod & M32) if ".lo" in opc else (prod >> 32)
            elif base in ("mad", "madc"):
                prod = val(src[0]) * val(src[1])
                part = (prod & M32) if ".lo" in opc else (prod >> 32)
                full = part + val(src[2]) + cin
            elif base in ("add", "addc"):
                full = val(src[0]) + val(src[1]) + cin
            elif base in ("sub", "subc"):
                full = val(src[0]) - val(src[1]) - cin
                if full < 0:
                    full += 1 << 32
                    bout = 1
                else:
                    bout = 0
                if sets_cc:
                    cf = bout
                else:
                    assert not (nocarry and bout), (self.name, opc, d)
                reg[d] = full & M32
                continue
            else:
                raise ValueError(opc)
            cout = full >> 32
            assert cout <= 1, (self.name, opc)
            if sets_cc:
                cf = cout
            else:
                assert not (nocarry and cout), "carry lost in %s at %s %s" % (self.name, opc, d)
            reg[d] = full & M32
        return reg

    # -- CUDA emitter
    def emit(self) -> str:
        order = self.outs + self.inouts + self.ins
        idx = {n: i for i, n in enumerate(order)}

        def fmt(x):
            if isinstance(x, int):
                return "0x%08x" % (x & M32)
            return "%%%d" % idx[x] if x in idx else x

        lines = []
        if self.temps:
            lines.append(".reg .u32 %s;" % ", ".join(self.temps))
        if self.preds:
            lines.append(".reg .pred %s;" % ", ".join(self.preds))
        n64 = 0
        for opc, d, src, _nc, guard in self.ops:
            g = "@%s " % guard if guard else ""
            if opc == "mulwide":
                lo, hi = d.split("|")
                w = "wd%d" % n64
                n64 += 1
                lines.append("mul.wide.u32 %s, %s, %s;" % (w, fmt(src[0]), fmt(src[1])))
                lines.append("mov.b64 {%s, %s}, %s;" % (fmt(lo), fmt(hi), w))
                continue
            lines.append("%s%s %s;" % (g, opc, ", ".join([fmt(d)] + [fmt(s) for s in src])))
        if n64:
            lines.insert(0, ".reg .u64 %s;" % ", ".join("wd%d" % i for i in range(n64)))
        body = "\n".join('        "%s\\n\\t"' % ln for ln in ["{"] + lines + ["}"])
        cons_out = ", ".join(['"=&r"(%s)' % n for n in self.outs] + ['"+r"(%s)' % n for n in self.inouts])
        cons_in = ", ".join('"r"(%s)' % n for n in self.ins)
        return "    asm(\n%s\n        : %s\n        : %s);\n" % (body, cons_out, cons_in)


def arr(name: str, n: int) -> List[str]:
    return ["%s[%d]" % (name, i) for i in range(n)]


# ------------------------------------------------------------------------------------------------
# Interleaved Montgomery product: 8 rows over an even/odd pair of 8-limb accumulators
#   window value  W = sum ev[k] 2^(32k) + sum od[k] 2^(32(k+1))      (9 limbs)
#   row:  W += x * y_i ;  m = -W mod 2^32 ;  W += m p ;  W >>= 32  (roles of ev/od swap)
# Needs x + p <= 2^256 (window stays below 2^288); y is arbitrary (< 2^256).
# ------------------------------------------------------------------------------------------------
def _reduce_row(pg: Prog, ev, od, m):
    if P1_ALU:
        h = m + "h"
        if h not in pg.temps:
            pg.tmp(h)
        pg.op("sub.cc.u32", m, 0, ev[0])                            # m = -W mod 2^32, borrow = (W0 != 0)
        pg.op("subc.u32", h, m, 0)                                  # hi(m * p1) = m - (m != 0)
        pg.op("add.cc.u32", od[0], od[0], ev[0])                    # lo(m * p1) = -m = W0
        pg.op("addc.cc.u32", od[1], od[1], h)
    else:
        pg.op("sub.u32", m, 0, ev[0])                               # m = -W mod 2^32
        # odd columns (1,2),(3,4),(5,6),(7,8) += m * p1,p3,p5,p7
        pg.op("mad.lo.cc.u32", od[0], m, PL[1], od[0])
        pg.op("madc.hi.cc.u32", od[1], m, PL[1], od[1])
    for k in (2, 4):
        pg.op("madc.lo.cc.u32", od[k], m, PL[k + 1], od[k])
        pg.op("madc.hi.cc.u32", od[k + 1], m, PL[k + 1], od[k + 1])
    pg.op("madc.lo.cc.u32", od[6], m, PL[7], od[6])
    pg.op("madc.hi.u32", od[7], m, PL[7], od[7], nocarry=True)
    # even columns: limb 0 + m*p0 = ev0 + m = 0 (mod 2^32), carry = (ev0 != 0); then p2,p4,p6
    pg.op("add.cc.u32", ev[0], ev[0], m)
    pg.op("addc.cc.u32", ev[1], ev[1], 0)
    for k in (2, 4, 6):
        pg.op("madc.lo.cc.u32", ev[k], m, PL[k], ev[k])
        pg.op("madc.hi.cc.u32", ev[k + 1], m, PL[k], ev[k + 1])
    pg.op("addc.u32", od[7], od[7], 0, nocarry=True)


def gen_row_first() -> Prog:
    pg = Prog("fr_row_first", "ev/od = x * yi, then one reduction row (ev[0] becomes 0)")
    ev = pg.out(*arr("ev", 8))
    od = pg.out(*arr("od", 8))
    x = pg.inp(*arr("x", 8))
    yi = pg.inp("yi")
    m = pg.tmp("m")
    # outputs are written before all inputs are read -> early-clobber is avoided by the C wrapper
    for k in (0, 2, 4, 6):
        pg.op("mul.lo.u32", ev[k], x[k], yi)
        pg.op("mul.hi.u32", ev[k + 1], x[k], yi)
        pg.op("mul.lo.u32", od[k], x[k + 1], yi)
        pg.op("mul.hi.u32", od[k + 1], x[k + 1], yi)
    _reduce_row(pg, ev, od, m)
    return pg


def gen_row() -> Prog:
    pg = Prog("fr_row", "shift window by one limb (od[0] dead, od[1] orphan), += x*yi, reduce")
    ev = pg.inout(*arr("ev", 8))
    od = pg.inout(*arr("od", 8))
    x = pg.inp(*arr("x", 8))
    yi = pg.inp("yi")
    m = pg.tmp("m")
    pg.op("add.cc.u32", ev[0], ev[0], od[1])
    for k in (0, 2, 4):
        pg.op("madc.lo.cc.u32", od[k], x[k + 1], yi, od[k + 2])
        pg.op("madc.hi.cc.u32", od[k + 1], x[k + 1], yi, od[k + 3])
    pg.op("madc.lo.cc.u32", od[6], x[7], yi, 0)
    pg.op("madc.hi.u32", od[7], x[7], yi, 0, nocarry=True)
    pg.op("mad.lo.cc.u32", ev[0], x[0], yi, ev[0])
    pg.op("madc.hi.cc.u32", ev[1], x[0], yi, ev[1])
    for k in (2, 4, 6):
        pg.op("madc.lo.cc.u32", ev[k], x[k], yi, ev[k])
        pg.op("madc.hi.cc.u32", ev[k + 1], x[k], yi, ev[k + 1])
    pg.op("addc.u32", od[7], od[7], 0, nocarry=True)
    _reduce_row(pg, ev, od, m)
    return pg


def gen_merge() -> Prog:
    pg = Prog("fr_merge", "r = (od + ev>>32): result of the last row, 8 limbs")
    r = pg.out(*arr("r", 8))
    ev = pg.inp(*arr("ev", 8))
    od = pg.inp(*arr("od", 8))
    pg.op("add.cc.u32", r[0], od[0], ev[1])
    for k in range(1, 7):
        pg.op("addc.cc.u32", r[k], od[k], ev[k + 1])
    pg.op("addc.u32", r[7], od[7], 0, nocarry=True)
    return pg


# ------------------------------------------------------------------------------------------------
# Mix tail: T = E + O<<32 (+ A), one Montgomery row
# ------------------------------------------------------------------------------------------------
def gen_mix_sum() -> Prog:
    pg = Prog("fr_mix_sum", "t[0..8] = e[0..7] + (o[0..7] << 32)")
    t = pg.out(*arr("t", 9))
    e = pg.inp(*arr("e", 8))
    o = pg.inp(*arr("o", 8))
    pg.op("mov.u32", t[0], e[0])
    pg.op("add.cc.u32", t[1], e[1], o[0])
    for k in range(2, 8):
        pg.op("addc.cc.u32", t[k], e[k], o[k - 1])
    pg.op("addc.u32", t[8], o[7], 0, nocarry=True)
    return pg


def gen_redc1(with_arc: bool, n: int = 9) -> Prog:
    """t (9 limbs) holds the folded FP64 column sums INCLUDING the double-exponent offsets
    K_off = 0x43300000 * sum_{k=1..8} 2^(32k); a (9 limbs) = (A - K_off) mod 2^288, so that t + a wraps to the
    true T + A < 2^288.  Then one Montgomery row, kept in even/odd form so that every IMAD.WIDE accumulator is
    one fixed (even, odd) register pair: the even products m*p2, m*p4, m*p6 chain into t itself, the odd
    products m*p1..p7 go to a fresh odd-aligned array (plain mul.wide), and one add chain merges them.
    n = 10 (no constant): the same row on a 10-limb t, giving 9 limbs (first row of the constant fold)."""
    assert n == 9 or not with_arc
    name = "fr_arc_redc1" if with_arc else ("fr_redc1" if n == 9 else "fr_redc1_%d" % n)
    pg = Prog(name, "u = (t + a (mod 2^288) + m p) >> 32 with m = -(t+a) mod 2^32; t, a are 9 limbs" if with_arc else
              "u = (t + m p) >> 32 with m = -t mod 2^32; t is %d limbs, u %d" % (n, n - 1))
    u = pg.out(*arr("u", n - 1))
    t = pg.inout(*arr("t", n))
    if with_arc:
        a = pg.inp(*arr("a", 9))
        pg.op("add.cc.u32", t[0], t[0], a[0])
        for k in range(1, 8):
            pg.op("addc.cc.u32", t[k], t[k], a[k])
        pg.op("addc.u32", t[8], t[8], a[8])          # wraps mod 2^288 by construction
    m = pg.tmp("m")
    o = pg.tmp(*["o%d" % k for k in range(1, 9)])     # o[k-1] <-> limb k
    pg.op("sub.u32", m, 0, t[0])
    for idx, pj in enumerate((1, 3, 5, 7)):           # odd columns (1,2),(3,4),(5,6),(7,8): fresh
        if FUSE_FRESH and pj != 1:
            # one 64-bit product: ONE IMAD.WIDE.U32 instead of the IMAD + IMAD.HI pair ptxas makes of mul.lo / mul.hi
            pg.op("mulwide", o[2 * idx] + "|" + o[2 * idx + 1], m, PL[pj])
        else:
            pg.op("mul.lo.u32", o[2 * idx], m, PL[pj])
            pg.op("mul.hi.u32", o[2 * idx + 1], m, PL[pj])
    pg.op("add.cc.u32", t[0], t[0], m)                # limb 0 cancels; carry = (t0 != 0)
    pg.op("addc.cc.u32", t[1], t[1], 0)
    for k in (2, 4, 6):                               # even columns (2,3),(4,5),(6,7)
        pg.op("madc.lo.cc.u32", t[k], m, PL[k], t[k])
        pg.op("madc.hi.cc.u32", t[k + 1], m, PL[k], t[k + 1])
    for k in range(8, n - 1):
        pg.op("addc.cc.u32", t[k], t[k], 0)
    pg.op("addc.u32", t[n - 1], t[n - 1], 0, nocarry=True)
    pg.op("add.cc.u32", u[0], t[1], o[0])
    for k in range(1, 7):
        pg.op("addc.cc.u32", u[k], t[k + 1], o[k])
    if n == 9:
        pg.op("addc.u32", u[7], t[8], o[7], nocarry=True)
    else:
        pg.op("addc.cc.u32", u[7], t[8], o[7])
        for k in range(8, n - 2):
            pg.op("addc.cc.u32", u[k], t[k + 1], 0)
        pg.op("addc.u32", u[n - 2], t[n - 1], 0, nocarry=True)
    return pg


# ------------------------------------------------------------------------------------------------
# Product by a table constant C:  S = sum_j w_j T_j  with  T_j = C 2^(32j - 192) mod p  (eight 32 x 256-bit rows, all
# at the same alignment, S < 8 * 2^32 p < 2^290), then two Montgomery rows (fr_redc1_10, fr_redc1):
#   z = (S + m0 p + m1 p 2^32) / 2^64  ==  C w / R  (mod p),  z < p + 2^226.
# Same residue as montmul(C, w) with 64 + 2 * 7 multiplier instructions instead of 8 * 15.
# Window: ev[k] = limb k (0..8) takes the products with T_j's even limbs, od[k] = limb k + 1 (1..9) the odd ones; each
# row's carry stops in the top limb (< 8 after eight rows).
# ------------------------------------------------------------------------------------------------
def gen_fold_row(first: bool) -> Prog:
    name = "fr_fold_row_first" if first else "fr_fold_row"
    pg = Prog(name, "ev/od = t * wj (first row)" if first else "ev/od += t * wj  (t: 8 limbs, wj: one 32-bit limb)")
    ev = (pg.out if first else pg.inout)(*arr("ev", 9))
    od = (pg.out if first else pg.inout)(*arr("od", 9))
    t = pg.inp(*arr("t", 8))
    wj = pg.inp("wj")
    if first:
        for k in (0, 2, 4, 6):
            pg.op("mul.lo.u32", ev[k], t[k], wj)
            pg.op("mul.hi.u32", ev[k + 1], t[k], wj)
            pg.op("mul.lo.u32", od[k], t[k + 1], wj)
            pg.op("mul.hi.u32", od[k + 1], t[k + 1], wj)
        pg.op("mov.u32", ev[8], 0)
        pg.op("mov.u32", od[8], 0)
        return pg
    for acc, off in ((ev, 0), (od, 1)):
        for k in (0, 2, 4, 6):
            pg.op("mad.lo.cc.u32" if k == 0 else "madc.lo.cc.u32", acc[k], t[k + off], wj, acc[k])
            pg.op("madc.hi.cc.u32", acc[k + 1], t[k + off], wj, acc[k + 1])
        pg.op("addc.u32", acc[8], acc[8], 0, nocarry=True)
    return pg


def gen_fold_merge() -> Prog:
    pg = Prog("fr_fold_merge", "s[0..9] = ev[0..8] + (od[0..8] << 32)")
    s = pg.out(*arr("s", 10))
    ev = pg.inp(*arr("ev", 9))
    od = pg.inp(*arr("od", 9))
    pg.op("mov.u32", s[0], ev[0])
    pg.op("add.cc.u32", s[1], ev[1], od[0])
    for k in range(2, 9):
        pg.op("addc.cc.u32", s[k], ev[k], od[k - 1])
    pg.op("addc.u32", s[9], od[8], 0, nocarry=True)
    return pg


# ------------------------------------------------------------------------------------------------
# Conditional subtractions / modular add / sub
# ------------------------------------------------------------------------------------------------
def gen_condsub255() -> Prog:
    pg = Prog("fr_condsub255", "if (a >= 2^255) a -= p   => a < 2^255")
    a = pg.inout(*arr("a", 8))
    q = pg.pred("q")
    pg.op("setp.ge.u32", q, a[7], 0x80000000)
    pg.op("sub.cc.u32", a[0], a[0], PL[0], guard=q)
    for k in range(1, 7):
        pg.op("subc.cc.u32", a[k], a[k], PL[k], guard=q)
    pg.op("subc.u32", a[7], a[7], PL[7], guard=q, nocarry=True)
    return pg


def gen_condsub() -> Prog:
    pg = Prog("fr_condsub", "a < 2p  ->  a mod p in [0,p)")
    a = pg.inout(*arr("a", 8))
    t = pg.tmp(*["t%d" % i for i in range(8)])
    brw = pg.tmp("brw")
    q = pg.pred("q")
    pg.op("sub.cc.u32", t[0], a[0], PL[0])
    for k in range(1, 8):
        pg.op("subc.cc.u32", t[k], a[k], PL[k])
    pg.op("subc.u32", brw, 0, 0)                   # 0xffffffff if a < p
    pg.op("setp.eq.u32", q, brw, 0)
    for k in range(8):
        pg.op("selp.u32", a[k], t[k], a[k], q)
    return pg


def gen_add() -> Prog:
    pg = Prog("fr_add_lazy", "r = a + b (no reduction; caller guarantees a + b < 2^256)")
    r = pg.out(*arr("r", 8))
    a = pg.inp(*arr("a", 8))
    b = pg.inp(*arr("b", 8))
    pg.op("add.cc.u32", r[0], a[0], b[0])
    for k in range(1, 7):
        pg.op("addc.cc.u32", r[k], a[k], b[k])
    pg.op("addc.u32", r[7], a[7], b[7], nocarry=True)
    return pg


def gen_submod() -> Prog:
    pg = Prog("fr_sub_mod", "r = a - b mod p for a, b in [0,p)  (BlsScalar -)")
    r = pg.out(*arr("r", 8))
    a = pg.inp(*arr("a", 8))
    b = pg.inp(*arr("b", 8))
    brw = pg.tmp("brw")
    msk = pg.tmp(*["k%d" % i for i in range(8)])
    pg.op("sub.cc.u32", r[0], a[0], b[0])
    for k in range(1, 8):
        pg.op("subc.cc.u32", r[k], a[k], b[k])
    pg.op("subc.u32", brw, 0, 0)                   # all-ones if a < b
    for k in range(8):
        pg.op("and.b32", msk[k], brw, PL[k])
    pg.op("add.cc.u32", r[0], r[0], msk[0])
    for k in range(1, 7):
        pg.op("addc.cc.u32", r[k], r[k], msk[k])
    pg.op("addc.u32", r[7], r[7], msk[7])
    return pg



# ------------------------------------------------------------------------------------------------
# Chain builder with "fresh" (not yet written, logically zero) accumulator limbs
# ------------------------------------------------------------------------------------------------
class Acc:
    """Accumulator limbs by absolute index; a limb is 'fresh' until first written."""

    def __init__(self, pg: Prog, prefix: str, n: int, preset: Dict[int, str] | None = None):
        self.pg, self.n = pg, n
        self.name = {k: "%s%d" % (prefix, k) for k in range(n)}
        self.defined = set()
        if preset:
            for k, nm in preset.items():
                self.name[k] = nm
                self.defined.add(k)
        self.temps = [self.name[k] for k in range(n) if not (preset and k in preset)]

    def src(self, k) -> Operand:
        return self.name[k] if k in self.defined else 0


def chain_products(pg: Prog, acc: Acc, prods: Sequence[tuple], cf_live: bool = False, capture: bool = True) -> None:
    """prods: [(a, b, pos)] with consecutive 64-bit columns pos, pos+2, ...: acc[pos,pos+1] += a*b, carry
    running through the columns; the final carry is captured into acc[last+2] (asserted not to overflow)."""
    for (a, b, pos) in prods:
        for half, k in (("lo", pos), ("hi", pos + 1)):
            d = acc.name[k]
            if k in acc.defined or cf_live:
                opc = ("madc.%s.cc.u32" if cf_live else "mad.%s.cc.u32") % half
                pg.op(opc, d, a, b, acc.src(k))
                cf_live = True
            else:
                pg.op("mul.%s.u32" % half, d, a, b)
            acc.defined.add(k)
    if cf_live and capture:
        k = prods[-1][2] + 2
        pg.op("addc.u32", acc.name[k], acc.src(k), 0, nocarry=True)
        acc.defined.add(k)


def gen_sqr_product() -> Prog:
    """t[0..15] = a^2: 28 off-diagonal products once (even/odd columns), doubled by a funnel shift that is
    folded into the carry chain of the 8 diagonal squares  =>  36 IMAD.WIDE instead of 64."""
    pg = Prog("fr_sqr_wide", "t[0..15] = a * a (full 512-bit square)")
    t = pg.out(*arr("t", 16))
    a = pg.inp(*arr("a", 8))
    E, O = Acc(pg, "e", 17), Acc(pg, "o", 17)
    pg.tmp(*E.temps)
    pg.tmp(*O.temps)
    for i in range(7):
        odd = [(a[i], a[j], i + j) for j in range(i + 1, 8, 2)]
        even = [(a[i], a[j], i + j) for j in range(i + 2, 8, 2)]
        if odd:
            chain_products(pg, O, odd)
        if even:
            chain_products(pg, E, even)
    # S = E + O  (limb 0 is empty: the lowest off-diagonal product sits at limb 1)
    S = ["s%d" % k for k in range(16)]
    pg.tmp(*S)
    first = True
    for k in range(1, 16):
        if k not in E.defined and k not in O.defined and first:
            pg.op("mov.u32", S[k], 0)
            continue
        pg.op("add.cc.u32" if first else "addc.cc.u32", S[k], E.src(k), O.src(k))
        first = False
    assert 16 not in E.defined and 16 not in O.defined
    # t = 2 S + sum a_i^2 2^(64 i): x_k = (S_k << 1) | (S_{k-1} >> 31), folded into the diagonal chain
    X = ["x%d" % k for k in range(16)]
    pg.tmp(*X)
    pg.op("shf.l.wrap.b32", X[1], 0, S[1], 1)
    for k in range(2, 16):
        pg.op("shf.l.wrap.b32", X[k], S[k - 1], S[k], 1)
    pg.op("mul.lo.u32", t[0], a[0], a[0])
    pg.op("mad.hi.cc.u32", t[1], a[0], a[0], X[1])
    for i in range(1, 8):
        pg.op("madc.lo.cc.u32", t[2 * i], a[i], a[i], X[2 * i])
        if i < 7:
            pg.op("madc.hi.cc.u32", t[2 * i + 1], a[i], a[i], X[2 * i + 1])
        else:
            pg.op("madc.hi.u32", t[15], a[7], a[7], X[15], nocarry=True)
    return pg


def gen_redc_wide() -> Prog:
    """r = (t_lo + M p) / 2^256 + t_hi with M = -t_lo / p mod 2^256: eight Montgomery rows on the low half
    (9-limb even/odd window, pure register renaming between rows), then one 8-limb addition."""
    pg = Prog("fr_redc_wide", "r = redc(t[0..7]) + t[8..15]  (t is a 512-bit product)")
    r = pg.out(*arr("r", 8))
    t = pg.inp(*arr("t", 16))
    uid = [0]

    def fresh(prefix):
        uid[0] += 1
        nm = "%s%d" % (prefix, uid[0])
        pg.tmp(nm)
        return nm

    # window limbs as register names or None (= zero / not yet written)
    EV: List = [fresh("w") for _ in range(8)]
    for k in range(8):
        pg.op("mov.u32", EV[k], t[k])
    OD: List = [None] * 8
    orphan = None
    for row in range(8):
        cf = False
        if orphan is not None:
            pg.op("add.cc.u32", EV[0], EV[0], orphan)
            cf = True
        m = fresh("m")
        pg.op("sub.u32", m, 0, EV[0])
        odd_cols = (0, 2, 4, 6)
        if P1_ALU:
            # m * p1 = (EV0, m - (m != 0)) formed without the multiplier and without touching the carry flag
            one, h = fresh("c"), fresh("h")
            pg.op("min.u32", one, m, 1)
            pg.op("sub.u32", h, m, one)
            for kk, val in ((0, EV[0]), (1, h)):
                if OD[kk] is not None or cf:
                    src = OD[kk] if OD[kk] is not None else 0
                    if OD[kk] is None:
                        OD[kk] = fresh("w")
                    pg.op("addc.cc.u32" if cf else "add.cc.u32", OD[kk], src, val)
                    cf = True
                else:
                    OD[kk] = fresh("w")
                    pg.op("mov.u32", OD[kk], val)
            odd_cols = (2, 4, 6)
        # odd columns += m * (p1, p3, p5, p7)
        for idx, k in enumerate(odd_cols):
            pj = PL[k + 1]
            if FUSE_FRESH and OD[k] is None and OD[k + 1] is None and not cf and k + 1 != 7:
                OD[k], OD[k + 1] = fresh("w"), fresh("w")
                pg.op("mulwide", OD[k] + "|" + OD[k + 1], m, pj)     # one IMAD.WIDE.U32 (see gen_redc1)
                continue
            for half, kk in (("lo", k), ("hi", k + 1)):
                last = (kk == 7)
                if OD[kk] is not None or cf:
                    src = OD[kk] if OD[kk] is not None else 0
                    if OD[kk] is None:
                        OD[kk] = fresh("w")
                    opc = ("madc.%s" if cf else "mad.%s") % half + (".u32" if last else ".cc.u32")
                    pg.op(opc, OD[kk], m, pj, src, nocarry=last)
                    cf = not last
                else:
                    OD[kk] = fresh("w")
                    pg.op("mul.%s.u32" % half, OD[kk], m, pj)
        # even columns: limb 0 cancels (carry = EV0 != 0), then p2, p4, p6; carry out joins limb 8
        junk = fresh("j")
        pg.op("add.cc.u32", junk, EV[0], m)
        pg.op("addc.cc.u32", EV[1], EV[1], 0)
        for k in (2, 4, 6):
            pg.op("madc.lo.cc.u32", EV[k], m, PL[k], EV[k])
            pg.op("madc.hi.cc.u32", EV[k + 1], m, PL[k], EV[k + 1])
        pg.op("addc.u32", OD[7], OD[7], 0, nocarry=True)
        # shift the window down one limb: pure renaming
        orphan = EV[1]
        EV, OD = OD, [EV[2], EV[3], EV[4], EV[5], EV[6], EV[7], None, None]
    # merge window + orphan, then add the high half of t
    s = [fresh("q") for _ in range(8)]
    pg.op("add.cc.u32", s[0], EV[0], orphan)
    for k in range(1, 7):
        pg.op("addc.cc.u32", s[k], EV[k], OD[k - 1])
    pg.op("addc.u32", s[7], EV[7], 0, nocarry=True)
    pg.op("add.cc.u32", r[0], s[0], t[8])
    for k in range(1, 7):
        pg.op("addc.cc.u32", r[k], s[k], t[8 + k])
    pg.op("addc.u32", r[7], s[7], t[15], nocarry=True)
    return pg


ALL = [gen_row_first(), gen_row(), gen_merge(), gen_redc1(True),
       gen_condsub255(), gen_condsub(), gen_add(), gen_submod(),
       gen_sqr_product(), gen_redc_wide(),
       gen_fold_row(True), gen_fold_row(False), gen_fold_merge(), gen_redc1(False, 10), gen_redc1(False)]
BY_NAME = {p.name: p for p in ALL}

SIGS = {
    "fr_row_first": "uint32_t (&ev)[8], uint32_t (&od)[8], const uint32_t (&x)[8], uint32_t yi",
    "fr_row": "uint32_t (&ev)[8], uint32_t (&od)[8], const uint32_t (&x)[8], uint32_t yi",
    "fr_merge": "uint32_t (&r)[8], const uint32_t (&ev)[8], const uint32_t (&od)[8]",
    "fr_arc_redc1": "uint32_t (&u)[8], uint32_t (&t)[9], const uint32_t (&a)[9]",
    "fr_condsub255": "uint32_t (&a)[8]",
    "fr_condsub": "uint32_t (&a)[8]",
    "fr_add_lazy": "uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]",
    "fr_sub_mod": "uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]",
    "fr_sqr_wide": "uint32_t (&t)[16], const uint32_t (&a)[8]",
    "fr_redc_wide": "uint32_t (&r)[8], const uint32_t (&t)[16]",
    "fr_fold_row_first": "uint32_t (&ev)[9], uint32_t (&od)[9], const uint32_t (&t)[8], uint32_t wj",
    "fr_fold_row": "uint32_t (&ev)[9], uint32_t (&od)[9], const uint32_t (&t)[8], uint32_t wj",
    "fr_fold_merge": "uint32_t (&s)[10], const uint32_t (&ev)[9], const uint32_t (&od)[9]",
    "fr_redc1_10": "uint32_t (&u)[9], uint32_t (&t)[10]",
    "fr_redc1": "uint32_t (&u)[8], uint32_t (&t)[9]",
}


# ---- emulator-level compositions (mirror the C++ wrappers in fr_ptx.cuh) -----------------------
def _get(reg, name, n):
    return [reg["%s[%d]" % (name, i)] for i in range(n)]


def _put(name, vals):
    return {"%s[%d]" % (name, i): v for i, v in enumerate(vals)}


def emu_montmul(x: int, y: int) -> int:
    xl = [(x >> (32 * i)) & M32 for i in range(8)]
    yl = [(y >> (32 * i)) & M32 for i in range(8)]
    env = {**_put("x", xl), "yi": yl[0]}
    reg = BY_NAME["fr_row_first"].run(env)
    A, B = _get(reg, "ev", 8), _get(reg, "od", 8)
    for i in range(1, 8):
        # roles swap each row: previous od becomes ev
        env = {**_put("x", xl), "yi": yl[i], **_put("ev", B), **_put("od", A)}
        reg = BY_NAME["fr_row"].run(env)
        A, B = _get(reg, "ev", 8), _get(reg, "od", 8)
    reg = BY_NAME["fr_merge"].run({**_put("ev", A), **_put("od", B)})
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "r", 8)))


def emu_montsqr(a: int) -> int:
    reg = BY_NAME["fr_sqr_wide"].run(_put("a", [(a >> (32 * i)) & M32 for i in range(8)]))
    t = _get(reg, "t", 16)
    assert sum(v << (32 * i) for i, v in enumerate(t)) == a * a, "square product wrong"
    reg = BY_NAME["fr_redc_wide"].run(_put("t", t))
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "r", 8)))


def emu_redc_wide(t: int) -> int:
    reg = BY_NAME["fr_redc_wide"].run(_put("t", [(t >> (32 * i)) & M32 for i in range(16)]))
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "r", 8)))


K_OFF = 0x43300000 * sum(1 << (32 * k) for k in range(1, 9))     # exponent words of the 8 double columns


def emu_mix_lane(cols: Sequence[int], arc: int | None) -> int:
    """cols[k]: the exact column sum of limb k (< 2^52), as produced by the DFMA chain.  Mirrors the CUDA mix:
    raw = bits(2^52 + col) ; t[k] = lo_k + hi_raw_{k-1} + carry ; then fr_arc_redc1 with a = A - K_off."""
    t, hi_prev, carry = [], 0, 0
    for k in range(8):
        assert 0 <= cols[k] < (1 << 52)
        raw = 0x4330000000000000 + cols[k]
        sm = (raw & M32) + hi_prev + carry
        t.append(sm & M32)
        carry = sm >> 32
        hi_prev = raw >> 32
    t.append((hi_prev + carry) & M32)
    a = ((arc or 0) - K_OFF) % (1 << 288)
    reg = BY_NAME["fr_arc_redc1"].run({**_put("t", t), **_put("a", [(a >> (32 * i)) & M32 for i in range(9)])})
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "u", 8)))


def emu_cfold(tab: Sequence[int], w: int) -> int:
    """The constant fold as hades_device.cuh's cfold() composes it: eight rows, the merge, two Montgomery rows."""
    wl = hm_limbs(w)
    reg = BY_NAME["fr_fold_row_first"].run({**_put("t", hm_limbs(tab[0])), "wj": wl[0]})
    for j in range(1, 8):
        env = {**_put("t", hm_limbs(tab[j])), "wj": wl[j], **_put("ev", _get(reg, "ev", 9)), **_put("od", _get(reg, "od", 9))}
        reg = BY_NAME["fr_fold_row"].run(env)
    reg = BY_NAME["fr_fold_merge"].run({**_put("ev", _get(reg, "ev", 9)), **_put("od", _get(reg, "od", 9))})
    reg = BY_NAME["fr_redc1_10"].run(_put("t", _get(reg, "s", 10)))
    reg = BY_NAME["fr_redc1"].run(_put("t", _get(reg, "u", 9)))
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "u", 8)))


def hm_limbs(v: int) -> List[int]:
    return [(v >> (32 * i)) & M32 for i in range(8)]


def emu_unary(name: str, a: int) -> int:
    reg = BY_NAME[name].run(_put("a", [(a >> (32 * i)) & M32 for i in range(8)]))
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "a", 8)))


def emu_binary(name: str, a: int, b: int) -> int:
    reg = BY_NAME[name].run({**_put("a", [(a >> (32 * i)) & M32 for i in range(8)]),
                             **_put("b", [(b >> (32 * i)) & M32 for i in range(8)])})
    return sum(v << (32 * i) for i, v in enumerate(_get(reg, "r", 8)))


HEADER = '''// GENERATED by tools/gen_field_ptx.py -- do not edit by hand.
// Carry-chain primitives for BLS12-381 Fr on 8 x 32-bit limbs (sm_90a).  Each primitive is ONE asm
// statement (the carry flag never crosses a statement); mad.lo.cc/madc.hi.cc pairs become
// IMAD.WIDE.U32[.X] in SASS.  Verified instruction-by-instruction by the emulator in the generator
// (tests/test_field_ptx.py) against the integer definitions of tools/hades_model.py.
#pragma once
#include <stdint.h>

namespace p252 {

'''


def wide_ops(pg: Prog) -> int:
    """32x32->64-bit multiplier instructions a primitive issues: every *.hi half (its .lo partner fuses into the same
    IMAD.WIDE; a lone .hi is an IMAD.HI) and every mul.wide."""
    return sum(1 for opc, *_ in pg.ops if opc == "mulwide" or ".hi" in opc)


def cfold_wide_ops() -> int:
    return sum(wide_ops(BY_NAME[n]) * k for n, k in (("fr_fold_row_first", 1), ("fr_fold_row", 7), ("fr_redc1_10", 1),
                                                      ("fr_redc1", 1)))


def emit_header() -> str:
    s = HEADER
    s += "// multiplier instructions (IMAD.WIDE / IMAD.HI class) per primitive, counted by the generator\n"
    for pg in ALL:
        if wide_ops(pg):
            s += "constexpr int kWideOps_%s = %d;\n" % (pg.name, wide_ops(pg))
    s += "// the whole constant fold: eight rows + two Montgomery rows (cfold in hades_device.cuh)\n"
    s += "constexpr int kWideOps_fr_cfold = %d;\n" % cfold_wide_ops()
    s += "\n"
    for pg in ALL:
        s += "// %s\n" % pg.doc
        s += "__device__ __forceinline__ void %s(%s) {\n" % (pg.name, SIGS[pg.name])
        s += pg.emit()
        s += "}\n\n"
    s += "}  // namespace p252\n"
    return s


if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "poseidon252_b200", "csrc",
                       "fr_ptx.cuh")
    with open(out, "w") as f:
        f.write(emit_header())
    print("wrote", os.path.normpath(out))
