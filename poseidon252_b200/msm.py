"""JubJub multi-scalar multiplication and all-or-nothing Schnorr batch verification over the GPU engine:

    jubjub_msm(s, P)           = sum [s_i] P_i                     (the bucket method; the identity (0, 1) for n == 0)
    schnorr_verify_all(...)    = [8] ([sum z u] G + sum [z c] PK - sum [z] R) == O,  c = challenge(R, msg)
    schnorr_verify_double_all(...) = [8] ([sum z u] G + [sum z' u] G' + sum [z c] PK + sum [z' c] PK'
                                         - sum [z] R - sum [z'] R') == O,            c = challenge2(R, R', msg)

Both are VARIABLE TIME: scalar bits become bucket indexes on the device, so they take public data only.  The weights z
of schnorr_verify_all and schnorr_verify_double_all must be random and unpredictable to the signers; by default the
engine draws 128-bit weights from `secrets`, and for double-key signatures one independent array per equation.  The check is cofactored: a signature whose R carries a small-order component passes it, while
schnorr_verify_batch rejects it."""
from .engine import _engine_for


def jubjub_msm(scalars, points, engine=None, async_=False):
    """NEW: sum [scalars[i]] points[i].  scalars (n, 4) p252_jscalar rows, points (n, 2, 4) BlsScalar.0 limbs -> (2, 4).
    Invalid items (scalar >= r_J, a coordinate >= p, off the curve) are skipped; Engine.last_msm_invalid() counts them."""
    eng = _engine_for(engine, scalars)
    return eng.jubjub_msm(scalars, points, async_=async_)


def schnorr_verify_all(pk, u, R, msg, base, weights=None, engine=None):
    """NEW: one answer for n signatures -> bool.  pk (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R (n, 2, 4), msg (n, 4),
    base (2, 4); weights (n, 4) p252_jscalar rows or None (fresh 128-bit weights)."""
    eng = _engine_for(engine, u)
    return eng.schnorr_verify_all(pk, u, R, msg, base, weights=weights)


def schnorr_verify_double_all(pk, pk_p, u, R, R_p, msg, base, base_p, weights=None, weights_p=None, engine=None):
    """NEW: one answer for n double-key signatures -> bool.  pk and pk_p (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R and
    R_p (n, 2, 4), msg (n, 4), base (G) and base_p (G') (2, 4); weights and weights_p (n, 4) p252_jscalar rows or None
    (fresh, independent 128-bit weights)."""
    eng = _engine_for(engine, u)
    return eng.schnorr_verify_double_all(pk, pk_p, u, R, R_p, msg, base, base_p, weights=weights, weights_p=weights_p)
