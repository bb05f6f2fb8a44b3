"""Phoenix note values over the GPU engine: Pedersen value commitments, creating obfuscated notes and opening them.

    commit(v, blinder) = C = [v] G + [blinder] G'                          (v < 2^64, blinder < r_J)
    create (r, v, blinder, nonce; A, B):  R = [r] G,  S = [r] A,  note_pk = [hash(S)] G + B,  C = commit(v, blinder),
                                          cipher = encrypt([Fr(v), Fr(blinder)], S, nonce)
    open  (a; R, nonce, cipher, C):       (m0, m1) = decrypt(cipher, [a] R, nonce); the note opens iff the authentication
                                          passes, m0 < 2^64, m1 < r_J and commit(m0, m1) == C

hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0], as in the stealth calls.  G and G' (GENERATOR_NUMS) are
passed by the caller, (A, B) is the receiver's public key and a its view key.  A note whose encrypted opening does not
match its commitment cannot be spent, so a wallet counts only the value of notes that open.  S and hash(S) never leave
the device; note_open returns v and the blinder, the spend proof's witnesses."""
import numpy as np

from .encryption import _jscalar_row
from .engine import _engine_for
from .errors import DecryptionFailed, InvalidPoint

# r_J, the order of JubJub's prime subgroup
_R_J = 0x0e7db4ea6533afa906673b0101343b00a6682093ccc81082d0970e5ed6f72cb7


def _pt(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)


def _fr(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 4)


def _value(v):
    return np.array([int(v)], dtype=np.uint64)


def value_commit(value, blinder, base, base_p, engine=None):
    """NEW: one value commitment [value] G + [blinder] G'.  value: an int in [0, 2^64); blinder: a canonical int < r_J or
    one p252_jscalar row; base (G), base_p (G'): (2, 4) BlsScalar.0 limbs -> (2, 4).  Raises InvalidPoint for
    blinder >= r_J or a base off the curve."""
    eng = _engine_for(engine)
    C, ok = eng.value_commit_batch(_value(value), _jscalar_row(blinder), base, base_p)
    if not ok[0]:
        raise InvalidPoint()
    return C[0]


def value_commit_batch(value, blinder, base, base_p, engine=None, async_=False):
    """NEW: n value commitments.  value (n,) uint64 (a CUDA int64 tensor for device buffers), blinder (n, 4) p252_jscalar
    rows, base and base_p (2, 4) -> (commitment (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose row is
    zeroed."""
    eng = _engine_for(engine, blinder)
    return eng.value_commit_batch(value, blinder, base, base_p, async_=async_)


def note_create(r, value, blinder, nonce, base, base_p, A, B, engine=None):
    """NEW: one obfuscated note for the receiver (A, B).  r, blinder: canonical ints < r_J or one p252_jscalar row each;
    value: an int in [0, 2^64); nonce: (4,) BlsScalar.0 limbs; base, base_p, A, B: (2, 4) -> (R (2, 4), note_pk (2, 4),
    commitment (2, 4), cipher (3, 4)).  Raises InvalidPoint for r or blinder >= r_J, A or B off the curve, or a base off
    the curve."""
    eng = _engine_for(engine)
    R, pk, C, cipher, ok = eng.note_create_batch(_jscalar_row(r), _value(value), _jscalar_row(blinder), _fr(nonce), base,
                                                 base_p, _pt(A), _pt(B))
    if not ok[0]:
        raise InvalidPoint()
    return R[0], pk[0], C[0], cipher[0]


def note_create_batch(r, value, blinder, nonce, base, base_p, A, B, engine=None, async_=False):
    """NEW: n obfuscated notes.  r and blinder (n, 4) p252_jscalar rows, value (n,) uint64 (a CUDA int64 tensor for device
    buffers), nonce (n, 4), base and base_p (2, 4), A and B (1 or n, 2, 4) -> (R (n, 2, 4), note_pk (n, 2, 4),
    commitment (n, 2, 4), cipher (n, 3, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are zeroed."""
    eng = _engine_for(engine, r)
    return eng.note_create_batch(r, value, blinder, nonce, base, base_p, A, B, async_=async_)


def note_open(a, R, nonce, cipher, commitment, base, base_p, engine=None):
    """NEW: the checked opening of one note under the view key a -> (value int, blinder (4,) p252_jscalar row).  a: a
    canonical int < r_J or one p252_jscalar row; R, commitment, base, base_p: (2, 4) BlsScalar.0 limbs; nonce (4,);
    cipher (3, 4).  Raises InvalidPoint for a >= r_J, R off the curve or a base off the curve, and DecryptionFailed for a
    note that does not open (another key, a tampered cipher or nonce, or an opening that is out of range or does not
    match the commitment)."""
    eng = _engine_for(engine)
    a_row, R_row = _jscalar_row(a), _pt(R)
    value, blinder, ok = eng.note_open_batch(a_row, R_row, _fr(nonce),
                                             np.ascontiguousarray(cipher, dtype=np.uint64).reshape(1, 3, 4),
                                             _pt(commitment), base, base_p)
    if not ok[0]:
        a_int = sum(int(a_row[0, k]) << (64 * k) for k in range(4))
        if a_int >= _R_J or not eng.points_to_bytes(R_row)[1][0]:
            raise InvalidPoint()
        raise DecryptionFailed()
    return int(value[0]), blinder[0]


def note_open_batch(a, R, nonce, cipher, commitment, base, base_p, engine=None, async_=False):
    """NEW: n checked openings.  a (1 or n, 4) p252_jscalar rows, R (n, 2, 4), nonce (n, 4), cipher (n, 3, 4),
    commitment (n, 2, 4), base and base_p (2, 4) -> (value (n,), blinder (n, 4), ok (n,) uint8); ok == 0 (value and
    blinder zeroed) marks a note that did not open or an invalid item.  A wallet's balance is the sum of value where ok."""
    eng = _engine_for(engine, R)
    return eng.note_open_batch(a, R, nonce, cipher, commitment, base, base_p, async_=async_)
