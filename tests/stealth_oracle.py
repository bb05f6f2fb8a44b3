"""Pure-Python model of the stealth addresses of p252_stealth_address_batch / p252_stealth_owns_batch.

    hash(P)                       = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]     (P affine; < 2^250 < r_J)
    sender   (r; A, B):             R = [r] G,   note_pk = [hash([r] A)] G + B
    receiver (a, B; R, note_pk):    owns  <=>  note_pk == [hash([a] R)] G + B

Built from jubjub_oracle.py (affine complete addition, double-and-add) and hades_oracle.Hash.digest_truncated -- formulas
independent of the kernels' (fixed-base table walk, extended coordinates, projective comparison).  The formulas are
phoenix-core's PublicKey::gen_stealth_address / ViewKey::owns as recalled, not checked against that crate (it is not
vendored): the library's contract is the formulas above."""
import hades_oracle as ho
import jubjub_oracle as jo


def hash_point(pt):
    """hash(P) of the model: the truncated digest of (u, v), a canonical JubJub scalar < 2^250"""
    return ho.Hash.digest_truncated(ho.Domain.Other, [pt[0], pt[1]])[0]


def stealth_address(r, A, B, G=jo.GENERATOR):
    """(R, note_pk), or None where the batch call reports ok = 0 (r >= r_J, A or B not a curve point)"""
    if not (0 <= r < jo.R_J) or not jo.on_curve(A) or not jo.on_curve(B):
        return None
    return jo.mul(r, G), jo.add(jo.mul(hash_point(jo.mul(r, A)), G), B)


def note_key(a, B, R, G=jo.GENERATOR):
    """[hash([a] R)] G + B: the note_pk view key a and spend key B own"""
    return jo.add(jo.mul(hash_point(jo.mul(a, R)), G), B)


def owns(a, B, R, note_pk, G=jo.GENERATOR):
    """1 owned, 0 not owned, None invalid (a >= r_J, R not a curve point, a note_pk coordinate >= p).  B and G are the
    call's host-checked points."""
    if not (0 <= a < jo.R_J) or not jo.on_curve(R) or not all(0 <= c < jo.P for c in note_pk):
        return None
    return int(note_key(a, B, R, G) == tuple(note_pk))


def keys(a, b, G=jo.GENERATOR):
    """the receiver's public key (A, B) = ([a] G, [b] G)"""
    return jo.mul(a, G), jo.mul(b, G)
