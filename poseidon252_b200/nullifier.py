"""Phoenix note nullifiers over the GPU engine: which of a wallet's notes are spent.

    hash(P)   = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]            (the stealth calls' hash)
    note_sk   = (hash([a] R) + b) mod r_J                                        (SecretKey::gen_note_sk)
    nullifier = Hash::digest(Domain::Other, [pk'.u, pk'.v, pos])[0],  pk' = [note_sk] G'   (Note::gen_nullifier)

(a, b) is the wallet's secret key, R a note's ephemeral key, pos its position in the note tree and G' the second
generator (GENERATOR_NUMS), passed by the caller.  note_sk and pk' never leave the device."""
import numpy as np

from .encryption import _jscalar_row
from .engine import _engine_for
from .errors import InvalidPoint


def nullifier(a, b, base, R, pos, engine=None):
    """NEW: the nullifier of one note.  a, b: canonical ints < r_J or one p252_jscalar row each; base (G') and R: (2, 4)
    BlsScalar.0 limbs; pos: an int in [0, 2^64) -> (4,) BlsScalar.0 limbs.  Raises InvalidPoint for a or b >= r_J, R off
    the curve, or a base off the curve."""
    eng = _engine_for(engine)
    res, ok = eng.nullifier_batch(_jscalar_row(a), _jscalar_row(b), base,
                                  np.ascontiguousarray(R, dtype=np.uint64).reshape(1, 2, 4), np.array([pos], dtype=np.uint64))
    if not ok[0]:
        raise InvalidPoint()
    return res[0]


def nullifier_batch(a, b, base, R, pos, engine=None, async_=False):
    """NEW: n nullifiers.  a and b (1 or n, 4) p252_jscalar rows, base (2, 4), R (n, 2, 4), pos (n,) uint64 (a CUDA int64
    tensor for device buffers) -> (nullifier (n, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose row is zeroed."""
    eng = _engine_for(engine, R)
    return eng.nullifier_batch(a, b, base, R, pos, async_=async_)
