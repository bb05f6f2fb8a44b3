"""CPU: the constructed edge corpus of tests/hades_edges.py, and the operand bounds of the scaled-lazy Hades proved for
every round.

* The inverse rounds undo the oracle's rounds one by one.
* The C oracle (what every GPU test compares with) equals the Python oracle on every corpus state.
* The corpus reaches its edges: the traced model shows stored u == p, u = s + p, a final value == p at exactly the
  targeted (round, lane) sites.  A change to the tables that moved the stored classes would make the corpus toothless;
  this test fails first.
* The model equals the oracle on every corpus state.
* Upper bounds propagated through all 68 rounds with the real tables prove the bounds DESIGN.md section 3.4 lists, the
  row-operand condition of every montmul, T < 2^288 and the FP64 column sums < 2^52."""
import functools
import random
from collections import defaultdict

import numpy as np
import pytest

import hades_edges as he
import hades_model as hm
import hades_oracle as o
from conftest import mont

P = o.P


# ---- shared, traced once per session --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def traced_raw():
    """(case, u values of the case's round, final values, model output) for every raw-corpus state."""
    out = []
    for c in he.raw_corpus():
        t = he.trace(c.x)
        r = min(c.r, he.ROUNDS - 1)
        out.append((c, [t.u(r, i) for i in range(he.W)], [t.final(i) for i in range(he.W)], t.out))
    return out


def sponge_corpora():
    return [he.digest_corpus(*s) for s in he.DIGEST_SHAPES] + [he.crypt_corpus(L) for L in (1, 3)]


def sponge_perm_input(corpus, c):
    """The input of permutation c.perm of corpus item c, recomputed from the item itself through the oracle's sponge."""
    if isinstance(corpus, he.CryptCorpus):
        assert c.perm == 0
        return [corpus.tag] + list(c.data) + [0]
    k = min(corpus.in_len, 4)
    s = [corpus.tag] + list(c.data[:k]) + [0] * (4 - k)
    for n in range(1, c.perm + 1):
        s = o.perm(s)
        chunk = c.data[4 * n:4 * n + 4]
        s = [s[0]] + [(a + b) % P for a, b in zip(s[1:], chunk)] + s[1 + len(chunk):]
    return s


# ---- inverse rounds ------------------------------------------------------------------------------------------------------
def test_inverse_rounds_round_trip():
    rng = random.Random(5)
    for x in [[0] * 5, [P - 1] * 5] + [[rng.randrange(P) for _ in range(5)] for _ in range(2)]:
        for r in range(he.ROUNDS):
            assert he.state_at_round_to_input(r, he.state_at_round(x, r)) == x, "round %d" % r
        y = o.perm(x)
        assert he.state_at_round(x, he.ROUNDS) == y
        assert he.output_to_input(y) == x
    assert all(sum(a * b for a, b in zip(row, col)) % P == int(i == j)
               for i, row in enumerate(he.MDS) for j, col in enumerate(zip(*he.MDS_INV)))


def test_sponge_corpora_are_sponge_states():
    """Every sponge case's targeted permutation input is what the sponge actually permutes for that item."""
    for corpus in sponge_corpora():
        for c in corpus.cases:
            assert sponge_perm_input(corpus, c) == c.x, c.name


# ---- C oracle == Python oracle on the corpus ----------------------------------------------------------------------------
def test_c_oracle_equals_python_oracle_on_corpus(coracle):
    xs = [c.x for c in he.raw_corpus()]
    got = coracle.permute(mont(xs).reshape(-1, 5, 4))
    assert np.array_equal(got, mont([o.perm(x) for x in xs]).reshape(-1, 5, 4))
    for corpus in sponge_corpora():
        if isinstance(corpus, he.CryptCorpus):
            L, n = corpus.L, len(corpus.cases)
            secret = mont([c.data[:2] for c in corpus.cases]).reshape(n, 2, 4)
            nonce = mont([c.data[2] for c in corpus.cases]).reshape(n, 4)
            cipher = coracle.encrypt(mont(corpus.tag), mont(corpus.messages).reshape(n, L, 4), L, secret, nonce)
            want = [o.encrypt(m, c.data[:2], c.data[2]) for m, c in zip(corpus.messages, corpus.cases)]
            assert np.array_equal(cipher, mont(want).reshape(n, L + 1, 4))
            msg, ok = coracle.decrypt(mont(corpus.tag), cipher, L, secret, nonce)
            assert ok.all() and np.array_equal(msg, mont(corpus.messages).reshape(n, L, 4))
        else:
            dom = getattr(o.Domain, corpus.domain)
            want = []
            for d in corpus.data:
                h = o.Hash(dom)
                h.output_len(corpus.out_len)
                h.update(d)
                want.append(h.finalize())
            got = coracle.digest(mont(corpus.tag), mont(corpus.data), corpus.in_len, corpus.out_len)
            assert np.array_equal(got, mont(want).reshape(got.shape)), corpus.domain


# ---- the corpus reaches its edges ---------------------------------------------------------------------------------------
def _expect_raw(c, us, finals):
    """The misses of one raw case: (round, lane, kind) names whose traced value is not the targeted one."""
    miss = []
    for lane in c.lanes:
        name = "r%d/lane%d/%s" % (c.r, lane, c.kind)
        if c.r == he.ROUNDS:
            v = finals[lane]
            ok = v % P == c.s and {"out_zero": v == P, "out_minus_1": True, "out_mont_minus_1": v in (P - 1, 2 * P - 1)}[c.kind]
        else:
            v = us[lane]
            ok = v % P == c.s and {
                "u_eq_p": v == P, "u_1_plus_p": v == 1 + P, "u_p_minus_1": v == P - 1,
                "true_plus_1": v < 2 * P, "true_minus_1": v < 2 * P,
                "r0_true_zero": v == 0, "r0_true_minus_1": v < P, "r0_u_p_minus_1": v == P - 1,
            }.get(c.kind, c.kind.startswith("s_plus_p_") and v == c.s + P and v > P)
        if not ok:
            miss.append(name)
    return miss


def test_raw_corpus_reaches_its_edges():
    miss, covered = [], defaultdict(set)
    deepest = defaultdict(int)                       # round -> largest u - p over the s + p cases
    for c, us, finals, _ in traced_raw():
        miss += _expect_raw(c, us, finals)
        for lane in c.lanes:
            covered[c.kind].add((c.r, lane))
        if c.kind.startswith("s_plus_p_"):
            deepest[c.r] = max(deepest[c.r], us[c.lanes[0]] - P)
    assert not miss, "%d targeted sites not reached: %s" % (len(miss), miss[:20])
    every = {(r, lane) for r in range(1, he.ROUNDS) for lane in range(he.W)}
    for kind in he.U_KINDS:
        assert covered[kind] >= every, "%s: no case at %s" % (kind, sorted(every - covered[kind])[:10])
    s_plus_p = set().union(*(v for k, v in covered.items() if k.startswith("s_plus_p_")))
    assert s_plus_p == every, "u = s + p missing at (round, lane) %s" % sorted(every - s_plus_p)[:10]
    shallow = [r for r in range(1, he.ROUNDS) if deepest[r] < 1 << 238]
    assert not shallow, "rounds without a case u >= p + 2^238: %s" % shallow
    for kind in ("r0_true_zero", "r0_true_minus_1", "r0_u_p_minus_1"):
        assert covered[kind] == {(0, lane) for lane in range(he.W)}, kind
    assert covered["u_eq_p"] >= {(r, lane) for r in (1, 3, 64, 67) for lane in range(he.W)}
    assert sum(c.kind == "u_eq_p" and len(c.lanes) == he.W for c in he.raw_corpus()) == 4
    for kind in ("out_zero", "out_minus_1", "out_mont_minus_1"):
        assert covered[kind] == {(he.ROUNDS, lane) for lane in range(he.W)}, kind
    assert any(c.kind == "out_zero" and len(c.lanes) == he.W for c in he.raw_corpus())


@pytest.mark.parametrize("which", ["%s-%d-%d" % s for s in he.DIGEST_SHAPES] + ["crypt-1", "crypt-3"])
def test_sponge_corpus_reaches_its_edges(which):
    corpus = dict(zip(["%s-%d-%d" % s for s in he.DIGEST_SHAPES] + ["crypt-1", "crypt-3"], sponge_corpora()))[which]
    miss, hit = [], set()
    for c in corpus.cases:
        t = he.trace(c.x)
        lane = c.lanes[0]
        v = t.u(c.r, lane)
        want = {"u_eq_p": P, "u_1_plus_p": 1 + P, "u_p_minus_1": P - 1, "r0_true_zero": 0}.get(c.kind)
        if v % P != c.s or (want is not None and v != want):
            miss.append("perm%d/r%d/lane%d/%s" % (c.perm, c.r, lane, c.kind))
        hit.add((c.perm, c.r, lane, c.kind))
        assert t.out == [he.mont(y) for y in o.perm(c.x)], c.name
    assert not miss, "%s: targeted sites not reached: %s" % (which, miss)
    perms = {c.perm for c in corpus.cases}
    for perm in perms:
        assert {(perm, 1, lane, "u_eq_p") for lane in range(he.W)} <= hit, "%s: round-1 u == p missing" % which


# ---- model == oracle ----------------------------------------------------------------------------------------------------
def test_model_equals_oracle_on_corpus():
    bad = [c.name for c, _, _, out in traced_raw() if out != [he.mont(y) for y in o.perm(c.x)]]
    assert not bad, "model differs from the oracle on %s" % bad[:20]


# ---- operand bounds, proved -------------------------------------------------------------------------------------------
def proved_bounds():
    """Upper bounds of every intermediate of the scaled-lazy permutation over all canonical inputs, propagated round by
    round with the real tables: a Montgomery product of operands <= x, y is <= (x y + (2^256 - 1) p) / 2^256, a
    Montgomery row on T is <= (T + (2^32 - 1) p) / 2^32.  Asserts the conditions the CUDA code needs on the way;
    returns the largest bound per site."""
    tb, C, M = hm.TABLES, hm.CMAT, hm.TWO256

    def mm(x, y, row):
        assert row + P <= M, "montmul row operand %d may exceed 2^256 - p" % row
        return (x * y + (M - 1) * P) >> 256

    def sq(x):
        return (x * x + (M - 1) * P) >> 256

    worst = defaultdict(int)
    u = [P - 1] * he.W                               # the first add's conditional subtraction: [0, p)
    for r in range(he.ROUNDS):
        z = []
        for i in range(he.W):
            if r:
                worst["u"] = max(worst["u"], u[i])
            if hm.is_full(r) or i == 4:
                a = sq(u[i])
                b = sq(a)
                x = mm(u[i], b, u[i])
                for k, v in (("sqr1", a), ("sqr2", b), ("x5", x)):
                    worst[k] = max(worst[k], v)
                if not hm.is_full(r):
                    x = mm(tb.G[r], x, tb.G[r])
                    worst["gmul"] = max(worst["gmul"], x)
                z.append(x)
            else:
                z.append(u[i])
        nxt = []
        for i in range(he.W):
            t = (tb.A[r + 1][i] if r + 1 < he.ROUNDS else 0) + sum(C[i][j] * z[j] for j in range(he.W))
            assert t < 1 << 288, "round %d lane %d: T may reach 2^288" % (r, i)
            worst["T"] = max(worst["T"], t)
            for k in range(8):                      # FP64 column sums: every limb <= min(2^32 - 1, bound >> 32k)
                col = sum(C[i][j] * min(hm.M32, z[j] >> (32 * k)) for j in range(he.W))
                assert col < 1 << 52, "round %d lane %d limb %d: FP64 column may reach 2^52" % (r, i, k)
                worst["col"] = max(worst["col"], col)
            nxt.append((t + hm.M32 * P) >> 32)
        u = nxt
    for x in u:
        worst["final"] = max(worst["final"], mm(tb.F, x, tb.F))
    return worst


def test_operand_bounds_proved():
    b = proved_bounds()
    # DESIGN.md section 3.4, "Operand bounds": k/10^4 p bounds as exact integer comparisons
    for site, lim in (("u", 10003), ("sqr1", 14534), ("sqr2", 19565), ("x5", 18862), ("gmul", 18550)):
        assert b[site] * 10000 < lim * P, "%s bound %.6f p exceeds %.4f p" % (site, b[site] / P, lim / 1e4)
    assert b["u"] < P + (1 << 243)
    assert b["final"] < 2 * P                      # one conditional subtraction gives [0, p)
    assert b["T"] < 1 << 288 and b["col"] < 1 << 52
    assert max(b.values()) < 1 << 288
    assert all(b[k] < hm.TWO256 for k in ("u", "sqr1", "sqr2", "x5", "gmul", "final"))
