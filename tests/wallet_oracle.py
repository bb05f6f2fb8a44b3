"""Pure-Python model of the multi-key wallet scan of p252_wallet_scan_batch.

    keys (a_j, b_j), j < k:  B_j = [b_j] G;  key j is bad iff a_j >= r_J or b_j >= r_J
    note i (R, note_pk, pos, nonce, cipher, C):
      invalid iff R is not a curve point with u, v < p or a coordinate of note_pk is >= p
      owner      = the smallest good j with stealth_oracle.owns(a_j, B_j, R, note_pk) == 1, else -1
      nullifier  = nullifier_oracle.nullifier(a_owner, b_owner, R, pos, G')
      (value, blinder), opened = note_oracle.open_note(a_owner, R, nonce, cipher, C, G')
    totals[j] = (sum of the opened values of the notes j owns, mod 2^64 and its high word; owned count; opened count)

Composed from stealth_oracle, nullifier_oracle and note_oracle only: no formula of its own."""
import jubjub_oracle as jo
import note_oracle as nto
import nullifier_oracle as nuo
import stealth_oracle as so

G = jo.GENERATOR


def key_ok(a, b):
    return 0 <= a < jo.R_J and 0 <= b < jo.R_J


def note_ok(R, note_pk):
    return jo.on_curve(R) and all(0 <= c < jo.P for c in note_pk)


def owner(keys, R, note_pk, base=G, spend=None):
    """the smallest index of a good key that owns the note, -1 if none does or the note is invalid; spend: the keys' B_j,
    if already computed"""
    if not note_ok(R, note_pk):
        return -1
    for j, (a, b) in enumerate(keys):
        if key_ok(a, b) and so.owns(a, spend[j] if spend else jo.mul(b, base), R, note_pk, base) == 1:
            return j
    return -1


def scan(keys, notes, Gp, base=G):
    """keys [(a, b)], notes [(R, note_pk, pos, nonce, cipher, C)] -> dict of the call's outputs: owner, nullifier, value,
    blinder, opened (per note; None / 0 where zeroed), totals (per key: [lo, hi, n_owned, n_opened]), n_invalid,
    n_bad_keys"""
    out = {"owner": [], "nullifier": [], "value": [], "blinder": [], "opened": [],
           "totals": [[0, 0, 0, 0] for _ in keys], "n_invalid": 0,
           "n_bad_keys": sum(not key_ok(a, b) for a, b in keys)}
    sums = [0] * len(keys)
    spend = [jo.mul(b, base) if key_ok(a, b) else None for a, b in keys]
    for R, pk, pos, nonce, cipher, C in notes:
        out["n_invalid"] += not note_ok(R, pk)
        j = owner(keys, R, pk, base, spend)
        out["owner"].append(j)
        nul, opening = None, None
        if j >= 0:
            a, b = keys[j]
            nul = nuo.nullifier(a, b, R, pos, Gp)
            opening = nto.open_note(a, R, nonce, cipher, C, Gp, base)
            out["totals"][j][2] += 1
            if opening is not None:
                out["totals"][j][3] += 1
                sums[j] += opening[0]
        out["nullifier"].append(nul)
        out["value"].append(opening[0] if opening else 0)
        out["blinder"].append(opening[1] if opening else 0)
        out["opened"].append(int(opening is not None))
    for j, s in enumerate(sums):
        out["totals"][j][0], out["totals"][j][1] = s & ((1 << 64) - 1), s >> 64
    return out
