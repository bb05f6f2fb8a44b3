"""JubJub ElGamal and the encrypted sender of a Phoenix note over the GPU engine.

    encrypt(PK, M; r)   = (c1, c2) = ([r] G, M + [r] PK)
    decrypt(sk; c1, c2) = c2 - [sk] c1                                              (NOT authenticated)
    sender_encrypt(note_pk; (A, B); (r_A, r_B)) = [encrypt(note_pk, A; r_A), encrypt(note_pk, B; r_B)]
    sender_decrypt(a, b; R, note_pk, enc):  note_sk = (hash([a] R) + b) mod r_J; only where [note_sk] G == note_pk,
                                            A = c2_A - [note_sk] c1_A,  B = c2_B - [note_sk] c1_B

hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0], as in the stealth calls; G is passed by the caller.
These are phoenix-core's elgamal::encrypt / decrypt and Sender::Encryption as recalled.  Decryption under a wrong key
gives another curve point; the sender call checks ownership first, so a note the key does not own reports ok == 0 instead
of a wrong sender.  r, the blinders, [a] R, its hash and note_sk never leave the device."""
import numpy as np

from .encryption import _jscalar_row
from .engine import _engine_for
from .errors import DecryptionFailed, InvalidPoint


def _pt(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)


def elgamal_encrypt(pk, msg, r, base, engine=None):
    """NEW: one ElGamal encryption.  pk, msg, base: (2, 4) BlsScalar.0 limbs; r: a canonical int < r_J or one
    p252_jscalar row -> (c1 (2, 4), c2 (2, 4)).  Raises InvalidPoint for r >= r_J, pk or msg off the curve, or a base off
    the curve."""
    eng = _engine_for(engine)
    c1, c2, ok = eng.elgamal_encrypt_batch(_pt(pk), _pt(msg), _jscalar_row(r), base)
    if not ok[0]:
        raise InvalidPoint()
    return c1[0], c2[0]


def elgamal_encrypt_batch(pk, msg, r, base, engine=None, async_=False):
    """NEW: n ElGamal encryptions.  pk (1 or n, 2, 4), msg (n, 2, 4), r (n, 4) p252_jscalar rows (one per message, never
    reused), base (2, 4) -> (c1 (n, 2, 4), c2 (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are
    zeroed."""
    eng = _engine_for(engine, r)
    return eng.elgamal_encrypt_batch(pk, msg, r, base, async_=async_)


def elgamal_decrypt(sk, c1, c2, engine=None):
    """NEW: one ElGamal decryption c2 - [sk] c1 -> (2, 4).  Not authenticated: a wrong key gives another point.  Raises
    InvalidPoint for sk >= r_J or c1 or c2 off the curve."""
    eng = _engine_for(engine)
    msg, ok = eng.elgamal_decrypt_batch(_jscalar_row(sk), _pt(c1), _pt(c2))
    if not ok[0]:
        raise InvalidPoint()
    return msg[0]


def elgamal_decrypt_batch(sk, c1, c2, engine=None, async_=False):
    """NEW: n ElGamal decryptions.  sk (1 or n, 4) p252_jscalar rows, c1 and c2 (n, 2, 4) -> (msg (n, 2, 4), ok (n,)
    uint8); ok == 0 marks an invalid item, whose row is zeroed."""
    eng = _engine_for(engine, c1)
    return eng.elgamal_decrypt_batch(sk, c1, c2, async_=async_)


def note_sender_encrypt_batch(note_pk, sender_A, sender_B, blinder, base, engine=None, async_=False):
    """NEW: the encrypted sender of n notes.  note_pk (n, 2, 4), sender_A and sender_B (1 or n, 2, 4), blinder (n, 2, 4)
    p252_jscalar rows [r_A, r_B], base (2, 4) -> (enc (n, 4, 2, 4) = [c1_A, c2_A, c1_B, c2_B], ok (n,) uint8)."""
    eng = _engine_for(engine, note_pk)
    return eng.note_sender_encrypt_batch(note_pk, sender_A, sender_B, blinder, base, async_=async_)


def note_sender_decrypt(a, b, R, note_pk, enc, base, engine=None):
    """NEW: the sender (A (2, 4), B (2, 4)) of one note under the secret key (a, b).  a, b: canonical ints < r_J or one
    p252_jscalar row each; R, note_pk, base: (2, 4); enc (4, 2, 4).  Raises DecryptionFailed for a note the key does not
    own or an invalid item."""
    eng = _engine_for(engine)
    A, B, ok = eng.note_sender_decrypt_batch(_jscalar_row(a), _jscalar_row(b), _pt(R), _pt(note_pk),
                                             np.ascontiguousarray(enc, dtype=np.uint64).reshape(1, 4, 2, 4), base)
    if not ok[0]:
        raise DecryptionFailed()
    return A[0], B[0]


def note_sender_decrypt_batch(a, b, R, note_pk, enc, base, engine=None, async_=False):
    """NEW: the senders of n notes.  a and b (1 or n, 4) p252_jscalar rows, R and note_pk (n, 2, 4), enc (n, 4, 2, 4),
    base (2, 4) -> (A (n, 2, 4), B (n, 2, 4), ok (n,) uint8); ok == 0 (rows zeroed) for a note the key does not own and
    for an invalid item."""
    eng = _engine_for(engine, R)
    return eng.note_sender_decrypt_batch(a, b, R, note_pk, enc, base, async_=async_)
