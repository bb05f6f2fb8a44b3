"""Schnorr signatures over JubJub -- jubjub-schnorr's SecretKey::sign / PublicKey::verify over the GPU engine:

    challenge(R, m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0]
    sign   (sk, r; m):        R = [r] G,  u = (r - challenge(R, m) sk) mod r_J,  signature = (u, R)
    verify (PK; (u, R), m):   [u] G + [challenge(R, m)] PK == R

Scalars are p252_jscalar rows (canonical ints < r_J as 4 little-endian u64), points and messages BlsScalar.0 limbs.  The
nonce r must be secret, uniformly random and used once: two signatures with one sk and one r reveal sk."""
import numpy as np

from .encryption import _jscalar_row
from .engine import _engine_for
from .errors import InvalidPoint


def _pt(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)


def _fr(x):
    return np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 4)


def schnorr_sign(sk, r, msg, base, engine=None):
    """NEW: one signature (u, R) of msg with secret key sk and nonce r.  sk, r: canonical ints < r_J or one p252_jscalar
    row; msg: (4,) BlsScalar.0 limbs; base: (2, 4) -> (u (4,) p252_jscalar, R (2, 4)).  Raises InvalidPoint for sk or
    r >= r_J or msg >= p."""
    eng = _engine_for(engine)
    u, R, ok = eng.schnorr_sign_batch(_jscalar_row(sk), _jscalar_row(r), _fr(msg), base)
    if not ok[0]:
        raise InvalidPoint()
    return u[0], R[0]


def schnorr_sign_batch(sk, r, msg, base, engine=None, async_=False):
    """NEW: n signatures.  sk (1 or n, 4) and r (n, 4) p252_jscalar rows, msg (n, 4), base (2, 4)
    -> (u (n, 4), R (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are zeroed."""
    eng = _engine_for(engine, r)
    return eng.schnorr_sign_batch(sk, r, msg, base, async_=async_)


def schnorr_verify(pk, u, R, msg, base, engine=None):
    """NEW: PublicKey::verify for one signature (u, R) of msg -> bool.  pk, R, base: (2, 4) BlsScalar.0 limbs; u: a
    canonical int < r_J or one p252_jscalar row; msg: (4,).  Raises InvalidPoint for u >= r_J, msg >= p, an R coordinate
    >= p, PK not a curve point, or a base off the curve."""
    eng = _engine_for(engine)
    verified = eng.schnorr_verify_batch(_pt(pk), _jscalar_row(u), _pt(R), _fr(msg), base)
    if eng.last_schnorr_invalid():
        raise InvalidPoint()
    return bool(verified[0])


def schnorr_verify_batch(pk, u, R, msg, base, engine=None, async_=False):
    """NEW: n verifications.  pk (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R (n, 2, 4), msg (n, 4), base (2, 4)
    -> verified (n,) uint8 (0 also for an invalid item)."""
    eng = _engine_for(engine, u)
    return eng.schnorr_verify_batch(pk, u, R, msg, base, async_=async_)
