"""Double-key Schnorr signatures over JubJub -- jubjub-schnorr's SecretKey::sign_double / SignatureDouble::verify -- and
the spend signature of a Phoenix note, over the GPU engine:

    challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0]
    sign_double   (sk, r; m):             R = [r] G,  R' = [r] G',  u = (r - challenge2(R, R', m) sk) mod r_J
    verify_double ((PK, PK'); (u, R, R'), m):  [u] G + [c] PK == R  and  [u] G' + [c] PK' == R'
    note_sk(a, b, R_note) = (hash([a] R_note) + b) mod r_J            (the stealth and nullifier calls' hash)

G and G' (GENERATOR_NUMS) are passed by the caller.  A note is spent under (note_pk, pk') = ([note_sk] G, [note_sk] G');
note_sign_double_batch returns pk', the spend proof's witness, which links the spend to the note and must stay private.
note_sk never leaves the device.  The nonce r must be secret, uniformly random and used once."""
import numpy as np

from .encryption import _jscalar_row
from .engine import _engine_for
from .errors import InvalidPoint


def _pt(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)


def _fr(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 4)


def schnorr_sign_double(sk, r, msg, base, base_p, engine=None):
    """NEW: one double-key signature (u, R, R') of msg with secret key sk and nonce r.  sk, r: canonical ints < r_J or
    one p252_jscalar row; msg: (4,) BlsScalar.0 limbs; base (G), base_p (G'): (2, 4) -> (u (4,), R (2, 4), R' (2, 4)).
    Raises InvalidPoint for sk or r >= r_J, msg >= p, or a base off the curve."""
    eng = _engine_for(engine)
    u, R, Rp, ok = eng.schnorr_sign_double_batch(_jscalar_row(sk), _jscalar_row(r), _fr(msg), base, base_p)
    if not ok[0]:
        raise InvalidPoint()
    return u[0], R[0], Rp[0]


def schnorr_sign_double_batch(sk, r, msg, base, base_p, engine=None, async_=False):
    """NEW: n double-key signatures.  sk (1 or n, 4) and r (n, 4) p252_jscalar rows, msg (n, 4), base and base_p (2, 4)
    -> (u (n, 4), R (n, 2, 4), R' (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are zeroed."""
    eng = _engine_for(engine, r)
    return eng.schnorr_sign_double_batch(sk, r, msg, base, base_p, async_=async_)


def schnorr_verify_double(pk, pk_p, u, R, R_p, msg, base, base_p, engine=None):
    """NEW: SignatureDouble::verify for one signature (u, R, R') of msg under (PK, PK') -> bool.  pk, pk_p, R, R_p, base,
    base_p: (2, 4) BlsScalar.0 limbs; u: a canonical int < r_J or one p252_jscalar row; msg: (4,).  Raises InvalidPoint
    for u >= r_J, msg >= p, a coordinate of R or R' >= p, PK or PK' not a curve point, or a base off the curve."""
    eng = _engine_for(engine)
    verified = eng.schnorr_verify_double_batch(_pt(pk), _pt(pk_p), _jscalar_row(u), _pt(R), _pt(R_p), _fr(msg), base,
                                               base_p)
    if eng.last_schnorr_double_invalid():
        raise InvalidPoint()
    return bool(verified[0])


def schnorr_verify_double_batch(pk, pk_p, u, R, R_p, msg, base, base_p, engine=None, async_=False):
    """NEW: n verifications.  pk and pk_p (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R and R_p (n, 2, 4), msg (n, 4),
    base and base_p (2, 4) -> verified (n,) uint8 (0 also for an invalid item)."""
    eng = _engine_for(engine, u)
    return eng.schnorr_verify_double_batch(pk, pk_p, u, R, R_p, msg, base, base_p, async_=async_)


def note_sign_double_batch(a, b, note_R, r, msg, base, base_p, engine=None, async_=False):
    """NEW: n spend signatures of notes under their note secret keys (hash([a] note_R) + b) mod r_J.  a and b (1 or n, 4)
    p252_jscalar rows, note_R (n, 2, 4), r (n, 4), msg (n, 4), base and base_p (2, 4) -> (u (n, 4), R (n, 2, 4),
    R' (n, 2, 4), pk' (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are zeroed."""
    eng = _engine_for(engine, r)
    return eng.note_sign_double_batch(a, b, note_R, r, msg, base, base_p, async_=async_)
