"""Pure-Python model of the note nullifiers of p252_nullifier_batch.

    hash(P)   = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]                 (the stealth calls' hash, < 2^250)
    note_sk   = (hash([a] R) + b) mod r_J
    pk'       = [note_sk] G'
    nullifier = Hash::digest(Domain::Other, [pk'.u, pk'.v, pos])[0]                (not truncated)

Built from stealth_oracle.hash_point, jubjub_oracle.py (affine complete addition, double-and-add) and
hades_oracle.Hash.digest -- formulas independent of the kernels'.  The formulas are phoenix-core's
SecretKey::gen_note_sk and Note::gen_nullifier as recalled, not checked against that crate (it is not vendored): the
library's contract is the formulas above."""
import hades_oracle as ho
import jubjub_oracle as jo
import stealth_oracle as so


def note_sk(a, b, R):
    """hash([a] R) + b mod r_J, or None where the batch call reports ok = 0 (a or b >= r_J, R not a curve point)"""
    if not (0 <= a < jo.R_J and 0 <= b < jo.R_J) or not jo.on_curve(R):
        return None
    return (so.hash_point(jo.mul(a, R)) + b) % jo.R_J


def nullifier(a, b, R, pos, Gp):
    """the nullifier of the note with ephemeral key R at tree position pos (0 <= pos < 2^64) for the secret key (a, b),
    G' = Gp; None for an invalid item"""
    sk = note_sk(a, b, R)
    if sk is None:
        return None
    pk = jo.mul(sk, Gp)
    return ho.Hash.digest(ho.Domain.Other, [pk[0], pk[1], pos])[0]
