"""Pure-Python model of JubJub ElGamal and the encrypted sender of a Phoenix note (p252_elgamal_{encrypt,decrypt}_batch,
p252_note_sender_{encrypt,decrypt}_batch).

    encrypt(PK, M; r)   = (c1, c2) = ([r] G, M + [r] PK)
    decrypt(sk; c1, c2) = c2 - [sk] c1
    sender_encrypt(note_pk; (A, B); (r_A, r_B)) = [encrypt(note_pk, A; r_A), encrypt(note_pk, B; r_B)]
    sender_decrypt(a, b; R, note_pk, enc): note_sk = (hash([a] R) + b) mod r_J; owned iff [note_sk] G == note_pk, then
                                           (c2_A - [note_sk] c1_A, c2_B - [note_sk] c1_B)

Built from jubjub_oracle.py (affine complete addition, double-and-add) and nullifier_oracle.note_sk -- formulas
independent of the kernels'.  The formulas are phoenix-core's elgamal::encrypt / decrypt and Sender::Encryption as
recalled, not checked against that crate (it is not vendored): the library's contract is the formulas above.  Each
function returns None where the batch call reports ok = 0."""
import jubjub_oracle as jo
import nullifier_oracle as nuo

G = jo.GENERATOR


def _point(pt):
    return all(0 <= c < jo.P for c in pt) and jo.on_curve(pt)


def _scalar(s):
    return 0 <= s < jo.R_J


def sub(p1, p2):
    return jo.add(p1, jo.neg(p2))


def encrypt(PK, M, r, base=G):
    """(c1, c2), or None for r >= r_J or PK / M not a curve point with u, v < p"""
    if not (_scalar(r) and _point(PK) and _point(M)):
        return None
    return jo.mul(r, base), jo.add(M, jo.mul(r, PK))


def decrypt(sk, c1, c2):
    """M = c2 - [sk] c1, or None for sk >= r_J or a ciphertext point not a curve point with u, v < p.  Not
    authenticated: a wrong key gives another point."""
    if not (_scalar(sk) and _point(c1) and _point(c2)):
        return None
    return sub(c2, jo.mul(sk, c1))


def sender_encrypt(note_pk, A, B, r_A, r_B, base=G):
    """[(c1_A, c2_A), (c1_B, c2_B)], or None for an invalid item (any of the five operands)"""
    ea, eb = encrypt(note_pk, A, r_A, base), encrypt(note_pk, B, r_B, base)
    if ea is None or eb is None:
        return None
    return [ea, eb]


def sender_decrypt(a, b, R, note_pk, enc, base=G):
    """(A, B), or None where the call reports ok = 0: a or b >= r_J, R or a ciphertext point not a curve point with
    u, v < p, or the note not owned ([note_sk] G != note_pk)"""
    sk = nuo.note_sk(a, b, R)
    if sk is None or not all(_point(p) for pair in enc for p in pair):
        return None
    if jo.mul(sk, base) != tuple(note_pk):
        return None
    return tuple(sub(c2, jo.mul(sk, c1)) for c1, c2 in enc)
