"""Regenerates tests/golden/hades_golden.json from the Python oracle (oracle/hades_oracle.py), which
reproduces the 6 known-answer vectors of src/hades.rs:134-162.  The reference is Rust
and cannot be executed here (no cargo/rustc; deps not vendored), so these are ORACLE-derived vectors:
the KAT block is pinned by the reference, the rest by the oracle that passes those KATs.
All values are canonical big-endian hex (the `{:?}` format of BlsScalar)."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import hades_oracle as o  # noqa: E402


def hx(v):
    return "0x%064x" % v


def main():
    rnd = random.Random(0xBEEF)
    g = {"comment": __doc__.strip().split("\n")[0]}
    g["kat_inputs_le_hex"] = o.KAT_INPUTS_LE_HEX
    g["kat_expected"] = {str(k): v for k, v in o.KAT_EXPECTED.items()}
    states = [[0] * 5, [0, 1, 2, 3, 4], [17] * 5, [19] * 5, [5000] * 5, [o.P - 1] * 5, [1, 0, 0, 0, 0]]
    states += [[rnd.randrange(o.P) for _ in range(5)] for _ in range(8)]
    g["perm"] = [{"in": [hx(x) for x in s], "out": [hx(x) for x in o.perm(s)]} for s in states]
    digests = []
    x42 = [rnd.randrange(o.P) for _ in range(42)]
    for name, dom, data, out_len in [
        ("merkle4", o.Domain.Merkle4, x42[:4], 1),
        ("merkle2", o.Domain.Merkle2, x42[:2], 1),
        ("other42", o.Domain.Other, x42, 1),
        ("other4", o.Domain.Other, x42[:4], 1),
        ("other1", o.Domain.Other, x42[:1], 1),
        ("other5_out2", o.Domain.Other, x42[:5], 2),
        ("other3_out3", o.Domain.Other, x42[:3], 3),
        ("other4_out7", o.Domain.Other, x42[:4], 7),
        ("other9_out5", o.Domain.Other, x42[:9], 5),
    ]:
        h = o.Hash(dom)
        h.output_len(out_len)
        h.update(data)
        digests.append({"name": name, "domain": dom, "in": [hx(v) for v in data], "out_len": out_len,
                        "out": [hx(v) for v in h.finalize()]})
    g["digest"] = digests
    enc = []
    for L in (1, 2, 3, 4, 5, 8, 21, 42):
        msg = [rnd.randrange(o.P) for _ in range(L)]
        sec = [rnd.randrange(o.P), rnd.randrange(o.P)]
        nonce = rnd.randrange(o.P)
        enc.append({"L": L, "msg": [hx(v) for v in msg], "secret": [hx(v) for v in sec], "nonce": hx(nonce),
                    "cipher": [hx(v) for v in o.encrypt(msg, sec, nonce)]})
    g["encrypt"] = enc
    g["tags"] = {
        "merkle4": hx(o.hash_to_scalar(o.tag_input([o.Absorb(4), o.Squeeze(1)], o.Domain.Merkle4))),
        "other42": hx(o.hash_to_scalar(o.tag_input([o.Absorb(42), o.Squeeze(1)], o.Domain.Other))),
        "encrypt2": hx(o.hash_to_scalar(o.tag_input(
            [o.Absorb(2), o.Absorb(1), o.Squeeze(2), o.Absorb(2), o.Squeeze(1)], o.Domain.Encryption))),
    }
    # Merkle trees (node = Hash::digest(Domain::Merkle4 | Merkle2, children), src/hash.rs:22-31): all internal levels
    # bottom-up + one opening (per level: the sibling group of the path node) -- for the tree / opening entry points
    trees = []
    for arity, k, leaf in ((4, 3, 37), (2, 5, 19)):
        dom = o.Domain.Merkle4 if arity == 4 else o.Domain.Merkle2
        leaves = [rnd.randrange(o.P) for _ in range(arity ** k)]
        leaves[5] = 0                                            # an empty slot is the zero scalar
        levels, cur = [leaves], leaves
        while len(cur) > 1:
            cur = [o.Hash.digest(dom, cur[i:i + arity])[0] for i in range(0, len(cur), arity)]
            levels.append(cur)
        path, i = [], leaf
        for l in range(k):
            g0 = i // arity * arity
            path.append([hx(v) for v in levels[l][g0:g0 + arity]])
            i //= arity
        trees.append({"arity": arity, "leaves": [hx(v) for v in leaves],
                      "nodes": [hx(v) for lv in levels[1:] for v in lv], "opening_leaf": leaf, "opening": path})
    g["merkle"] = trees
    with open(os.path.join(HERE, "hades_golden.json"), "w") as f:
        json.dump(g, f, indent=1)
    print("wrote hades_golden.json")


if __name__ == "__main__":
    main()
