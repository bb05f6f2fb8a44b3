"""Pure-Python model of the double-key Schnorr signatures of p252_schnorr_sign_double_batch /
p252_schnorr_verify_double_batch and of the note signer p252_note_sign_double_batch.

    challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0]      (< 2^250 < r_J)
    sign_double   (sk, r; m):                R = [r] G,  R' = [r] G',  u = (r - c sk) mod r_J
    verify_double ((PK, PK'); (u, R, R'), m):  [u] G + [c] PK == R  AND  [u] G' + [c] PK' == R'
    note_sk(a, b, R_note) = (hash([a] R_note) + b) mod r_J                    (nullifier_oracle.note_sk)
    note spend key: (PK, PK') = ([note_sk] G, [note_sk] G')

Built from jubjub_oracle.py (affine complete addition, double-and-add), hades_oracle.Hash.digest_truncated,
stealth_oracle.hash_point and nullifier_oracle.note_sk -- formulas independent of the kernels' (table walks, extended
coordinates, projective comparison).  The formulas are jubjub-schnorr's SecretKey::sign_double / SignatureDouble::verify
and phoenix-core's note key as recalled, not checked against those crates (they are not vendored): the library's
contract is the formulas above."""
import hades_oracle as ho
import jubjub_oracle as jo
import nullifier_oracle as no

G = jo.GENERATOR


def challenge2(R, Rp, m):
    """c of the model: the truncated digest of (R.u, R.v, R'.u, R'.v, m), a canonical JubJub scalar < 2^250"""
    return ho.Hash.digest_truncated(ho.Domain.Other, [R[0], R[1], Rp[0], Rp[1], m])[0]


def key_pair(sk, Gp, base=G):
    """(PK, PK') = ([sk] G, [sk] G')"""
    return jo.mul(sk, base), jo.mul(sk, Gp)


def sign_double(sk, r, m, Gp, base=G):
    """(u, R, R'), or None where the batch call reports ok = 0 (sk or r >= r_J, m >= p)"""
    if not (0 <= sk < jo.R_J) or not (0 <= r < jo.R_J) or not (0 <= m < jo.P):
        return None
    R, Rp = jo.mul(r, base), jo.mul(r, Gp)
    return (r - challenge2(R, Rp, m) * sk) % jo.R_J, R, Rp


def verify_double(pk, pkp, u, R, Rp, m, Gp, base=G):
    """1 verified, 0 not verified, None invalid (u >= r_J, m >= p, a coordinate of R or R' >= p, PK or PK' not a curve
    point)"""
    if not (0 <= u < jo.R_J) or not (0 <= m < jo.P) or not all(0 <= x < jo.P for x in tuple(R) + tuple(Rp)):
        return None
    if not jo.on_curve(pk) or not jo.on_curve(pkp):
        return None
    c = challenge2(R, Rp, m)
    ok = jo.add(jo.mul(u, base), jo.mul(c, pk)) == tuple(R)
    ok_p = jo.add(jo.mul(u, Gp), jo.mul(c, pkp)) == tuple(Rp)
    return int(ok and ok_p)


def note_sign_double(a, b, R_note, r, m, Gp, base=G):
    """((u, R, R'), pk') of the note's spend signature, or None where the batch call reports ok = 0 (a, b or r >= r_J,
    R_note not a curve point, m >= p)"""
    sk = no.note_sk(a, b, R_note)
    if sk is None:
        return None
    sig = sign_double(sk, r, m, Gp, base)
    if sig is None:
        return None
    return sig, jo.mul(sk, Gp)
