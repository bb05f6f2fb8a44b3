"""JubJub point compression -- dusk-jubjub's JubJubAffine::to_bytes / from_bytes over the GPU engine:

    to_bytes(u, v):   the 32 little-endian bytes of canonical v, bit 255 (bytes[31] >> 7) = the low bit of canonical u
    from_bytes(b):    v = b without bit 255 (rejected if >= p), u^2 = (v^2 - 1) / (1 + d v^2) (rejected if not a square),
                      u the root whose canonical low bit is bit 255

A set sign bit with u = 0 is accepted and decodes to the same point (pre-ZIP-216 behaviour); 32 zero bytes decode to the
order-4 point (sqrt(-1), 0).  There is no subgroup check.  Points are (2, 4) BlsScalar.0 limbs, encodings 32 bytes."""
import numpy as np

from .engine import _engine_for
from .errors import InvalidPoint


def point_from_bytes(data, engine=None):
    """NEW: JubJubAffine::from_bytes for one encoding: 32 bytes (bytes or uint8 array) -> (2, 4) point.  Raises
    InvalidPoint for v >= p or a u^2 that is not a square."""
    eng = _engine_for(engine)
    row = np.frombuffer(bytes(data), dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data
    pts, ok = eng.points_from_bytes(np.ascontiguousarray(row, dtype=np.uint8).reshape(1, 32))
    if not ok[0]:
        raise InvalidPoint()
    return pts[0]


def point_to_bytes(point, engine=None):
    """NEW: JubJubAffine::to_bytes for one point (2, 4) -> 32 bytes.  Raises InvalidPoint for a coordinate >= p or a
    point off the curve."""
    eng = _engine_for(engine)
    out, ok = eng.points_to_bytes(np.ascontiguousarray(point, dtype=np.uint64).reshape(1, 2, 4))
    if not ok[0]:
        raise InvalidPoint()
    return out[0].tobytes()


def points_from_bytes_batch(data, engine=None, async_=False):
    """NEW: n decodings.  data (n, 32) uint8 (host) or an (n, 4) 64-bit CUDA tensor of the same bytes
    -> (points (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid encoding, whose row is (0, 0)."""
    eng = _engine_for(engine, data)
    return eng.points_from_bytes(data, async_=async_)


def points_to_bytes_batch(points, engine=None, async_=False):
    """NEW: n encodings.  points (n, 2, 4) -> (bytes (n, 32) uint8 on the host or (n, 4) on the device, ok (n,) uint8);
    ok == 0 marks an invalid point, whose encoding is 32 bytes of 0xff."""
    eng = _engine_for(engine, points)
    return eng.points_to_bytes(points, async_=async_)
