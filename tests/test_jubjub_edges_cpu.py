"""The constructions of jubjub_edges.py are what they claim (CPU only): every edge point is a curve point whose site value
is the named edge, subgroup members are in the subgroup, placements put their point where they say, the paired secrets
select their table entry with the claimed sign, the pinned targets without a point have none, the impossible classes are
impossible and the quartic root finder agrees with brute force."""
import random

import pytest

import jubjub_edges as je
import jubjub_oracle as jo
from test_fixed_base_cpu import niels

P = je.P

# named targets that no curve point reaches (kind, name); a construction that silently loses cases changes this list
NO_POINT = {
    ("u", "(p-1)/2"), ("u", "(p+1)/2"), ("u", "R"), ("u", "2^32"), ("u", "2^224-1"), ("u", "p-2^32"), ("u", "limb2"),
    ("u", "limb4"), ("u", "limb6"),
    ("v", "2"), ("v", "p-2"), ("v", "2^32-1"), ("v", "2^32"), ("v", "2^64"), ("v", "2^254-1"), ("v", "2^254"),
    ("v", "p-2^32"), ("v", "p-2^64"), ("v", "limb2"), ("v", "limb4"),
    ("sum", "p-1"), ("sum", "p+1"),
    ("diff", "1"), ("diff", "-1"), ("diff", "2^32"), ("diff", "-2^32"),
    ("kt", "1"), ("kt", "p-1"), ("kt", "2"), ("kt", "p-2"), ("kt", "3"), ("kt", "p-3"), ("kt", "4"), ("kt", "p-4"),
    ("kt", "5"), ("kt", "p-5"),
} | {("uv", n) for n in ("1", "2", "3", "4", "5", "6", "10", "11", "12", "15", "16", "17", "18", "19", "21", "22", "23",
                         "24", "25", "26", "27", "29", "30", "31", "32", "33", "34", "35", "38", "39", "40", "p-1",
                         "p-2", "p-3", "2^32-1", "2^32", "2^64-1", "p-2^32", "p-2^64", "R")}


def test_edge_value_set():
    vals = dict(je.M)
    assert len(vals) == len(je.M) and all(0 <= m < P for m in vals.values())
    assert vals["R"] == je.mont(1) and vals["(p-1)/2"] * 2 + 1 == P
    assert {vals["limb%d" % k] for k in range(1, 7)} | {vals["2^32-1"]} == {0xffffffff << (32 * k) for k in range(7)}
    assert set(je.TOP_LIMB_NAMES) == {"p-1", "p-2", "p-3", "p-2^32", "p-2^64", "p-2^192"}


@pytest.mark.parametrize("kind", je.KINDS)
def test_every_edge_is_a_curve_point_at_its_named_value(kind):
    es = je.edges(kind)
    assert es, kind                                               # every class is non-empty
    targets = dict(je._TARGETS[kind])
    for e in es:
        assert jo.on_curve(e.pt), e
        assert e.target == targets[e.name] == je.site_value(kind, e.pt), e
    assert len(set(e.pt for e in es)) == len(es)


def test_niels_components_in_montgomery_form():
    """The Niels form (v - u, v + u, 2d u v) of each sum / diff / kt point holds the edge in its Montgomery image, and the
    limbs the device adds or subtracts are the exact integers claimed."""
    for e in je.edges("sum") + je.edges("diff") + je.edges("kt") + je.edges("uv"):
        ymx, ypx, kt = (je.mont(x) for x in niels(e.pt))
        mu, mv = je.mont(e.pt[0]), je.mont(e.pt[1])
        if e.kind == "sum":
            assert ypx == e.target % P and mu + mv == e.target and (e.target >= P) == (ypx < mu)
        elif e.kind == "diff":
            assert ymx == e.target % P and mv - mu == e.target and (e.target < 0) == (mv < mu)
        elif e.kind == "kt":
            assert kt == e.target and (P - kt) % P == je.mont(-2 * je.D * e.pt[0] * e.pt[1])
        else:
            assert je.mont(e.pt[0] * e.pt[1]) == e.target


def test_pinned_targets_without_a_point():
    assert set(je.no_point()) == NO_POINT
    # the statistics of the curve equation: p - k for k = 1..40 is a u coordinate 20 times, Mont(u v) = k for 7 k <= 29
    assert sum(1 for k in range(1, 41) if je.v_from_u(je.unmont(P - k))) == 20
    assert sum(1 for k in range(1, 30) if je.points_with_uv(je.unmont(k))) == 7


def test_impossible_classes():
    """m_u + m_v = p and m_v = m_u (v = -u, v = u) have no point: with c = 0 the quartic is d u^4 + 1, and -1/d is not a
    square."""
    assert pow(-pow(je.D, -1, P) % P, (P - 1) // 2, P) == P - 1
    assert je.roots(je.quartic(0)) == []
    for kind, t in (("sum", P), ("diff", 0)):
        assert je._class(kind, "", t) == []


@pytest.mark.parametrize("q", [10007, 10009, 65537])
def test_root_finder_matches_brute_force(q):
    rng = random.Random(q)
    for _ in range(60):
        f = [rng.randrange(q) for _ in range(rng.randrange(0, 5))] + [rng.randrange(1, q)]
        if rng.random() < 0.3:                                    # a product of linear factors, some repeated
            f = [1]
            for _ in range(4):
                r = rng.randrange(8)
                f = [(a - r * b) % q for a, b in zip([0] + f, f + [0])]
        want = [x for x in range(q) if sum(c * pow(x, i, q) for i, c in enumerate(f)) % q == 0]
        assert je.roots(f, q) == want, f


def test_quartic_roots_are_the_points_with_that_difference():
    rng = __import__("numpy").random.default_rng(5)
    for _ in range(4):
        u, v = jo.random_point(rng)
        assert u in je.roots(je.quartic((v - u) % P))


def test_subgroup_edges():
    sg = je.subgroup_edges()
    assert [e.kind for e in sg] == list(je.KINDS)
    for e in sg:
        assert e in je.edges(e.kind) and e.pt != jo.IDENTITY and je.mul(je.R_J, e.pt) == jo.IDENTITY


def test_output_placements():
    outs = je.output_placements()
    assert {e.kind for e, _, _ in outs} == set(je.KINDS)
    for kind in ("u", "v"):                                       # results at the top-limb values, as u and as v
        assert {e.name for e, _, _ in outs if e.kind == kind} >= {e.name for e in je.edges(kind)
                                                                  if e.name in je.TOP_LIMB_NAMES} != set()
    for e, s, pub in outs:
        assert s % 2 == 1 and 0 < s < je.R_J and jo.on_curve(pub)
        assert je.mul(s, pub) == e.pt, e


def test_table_placements_and_their_secrets():
    tps = je.table_placements()
    assert {(t.w, t.j) for t in tps} == set(je.TABLE_ENTRIES)
    for t in tps:
        k = t.j << (4 * t.w)
        assert jo.on_curve(t.base) and je.mul(k, t.base) == t.edge.pt, (t.w, t.j, t.edge)
        # every sign the recoding can give this entry, each selected by its secret
        assert sorted(sg for sg, _ in t.secrets) == sorted(je.signs_at(t.w, t.j)) and t.secrets
        for sg, s in t.secrets:
            assert 0 <= s < je.R_J and je.recode(s)[t.w] == sg * t.j
    # the recoding model is the kernel's (the model in test_fixed_base_cpu.py), and its sign limits are real
    from test_fixed_base_cpu import recode
    for t in tps:
        for _, s in t.secrets:
            assert recode(s) == je.recode(s)
    assert je.signs_at(0, 8) == (-1,) and je.signs_at(63, 1) == (1,) and je.signs_at(1, 3) == (1, -1)
    rng = random.Random(7)
    for _ in range(300):
        d = je.recode(rng.randrange(je.R_J))
        assert 8 not in d and d[63] in (0, 1)


def test_stealth_placements():
    a, A, B = je.receiver()
    h_send = je.sender_hG()
    for e in je.output_edges()[::7]:
        Bq = je.note_pk_placement(e.pt)
        assert jo.on_curve(Bq) and jo.add(h_send, Bq) == e.pt
        Sb = je.spend_B_placement(e.pt)
        Rn, hG = je.scan_note()
        assert jo.add(hG, Sb) == e.pt and je.so.owns(a, Sb, Rn, e.pt) == 1
        for _, q in je.near_misses(e.pt):
            assert q != e.pt and all(0 <= c < P for c in q) and je.so.owns(a, Sb, Rn, q) == 0
    for e in je.output_edges()[::23]:
        Gq, Bq, pk = je.R_placement(e.pt)
        assert je.mul(je.STEALTH_R, Gq) == e.pt and je.so.stealth_address(je.STEALTH_R, A, Bq, Gq) == (e.pt, pk)


def test_boundaries():
    bs = je.boundaries()
    assert {b.name.split("=")[1] for b in bs} == {n for n, _ in je.BOUNDARY_RAW}
    assert 2 * P < 1 << 256 < 3 * P
    for b in bs:
        assert jo.on_curve(b.pt) and b.twin == (je.mont(b.pt[0]), je.mont(b.pt[1]))
        i = 0 if b.name.startswith("u=") else 1
        assert b.raw[i] >= P and b.raw[i] % P == b.twin[i] and b.raw[1 - i] == b.twin[1 - i] and b.raw[i] < 1 << 256
    # u = p with v = Mont(1): the identity with a non-canonical u; u = 2p with v = Mont(+-1) likewise
    assert je.Boundary("u=p", (P, je.mont(1)), (0, je.mont(1))) in bs


def test_rows():
    r = je.raw_rows([((1 << 256) - 1, P)])
    assert (r[0, 0] == 0xFFFFFFFFFFFFFFFF).all() and sum(int(r[0, 1, k]) << (64 * k) for k in range(4)) == P
    assert (je.rows([jo.GENERATOR]) == jo.points_mont([jo.GENERATOR])).all()
