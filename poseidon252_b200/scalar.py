"""BlsScalar at the boundary: numpy uint64 arrays of shape (..., 4) holding `BlsScalar.0`
(little-endian u64 limbs of x*R mod p, R = 2^256 mod p) -- exactly what the reference keeps in
memory (dusk_bls12_381::Scalar([u64; 4])).  These helpers only convert representations for
callers/tests; no hashing or permutation happens here."""
import numpy as np

P = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
R = (1 << 256) % P
R_INV = pow(R, -1, P)
_M64 = (1 << 64) - 1


def to_mont(values):
    """canonical integers (iterable or nested) -> uint64 array (..., 4) of Montgomery limbs."""
    a = np.asarray(values, dtype=object)
    out = np.empty(a.shape + (4,), dtype=np.uint64)
    flat = out.reshape(-1, 4)
    for i, v in enumerate(a.reshape(-1)):
        m = (int(v) % P) * R % P
        for k in range(4):
            flat[i, k] = (m >> (64 * k)) & _M64
    return out


def from_mont(limbs):
    """uint64 array (..., 4) -> object array (...) of canonical Python integers."""
    a = np.ascontiguousarray(limbs, dtype=np.uint64)
    flat = a.reshape(-1, 4)
    out = np.empty(flat.shape[0], dtype=object)
    for i in range(flat.shape[0]):
        v = sum(int(flat[i, k]) << (64 * k) for k in range(4))
        out[i] = v * R_INV % P
    return out.reshape(a.shape[:-1])


def random_scalars(rng, shape):
    """Uniform scalars in [0, p) as Montgomery limbs: 64 PRNG bytes reduced mod p
    (the `ff::Field::random` recipe the reference's tests use, e.g. README.md:31-38)."""
    shape = (shape,) if isinstance(shape, int) else tuple(shape)
    n = int(np.prod(shape)) if shape else 1
    raw = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
    vals = [int.from_bytes(raw[i].tobytes(), "little") % P for i in range(n)]
    return to_mont(vals).reshape(shape + (4,))


def random_limbs_fast(rng, shape):
    """Fast uniform-ish field elements for large synthetic batches: 255 random bits with the top
    limb clamped below p's top limb (so the value is < p).  Any value < p is a valid BlsScalar.0."""
    shape = (shape,) if isinstance(shape, int) else tuple(shape)
    a = rng.integers(0, 1 << 63, size=shape + (4,), dtype=np.uint64) * np.uint64(2) + \
        rng.integers(0, 2, size=shape + (4,), dtype=np.uint64)
    a[..., 3] %= np.uint64(0x73EDA753299D7D48)
    return a


def jubjub_limbs(values):
    """canonical integers -> (n, 4) uint64 rows of p252_jscalar: the little-endian u64 limbs of each value, i.e. the 32
    bytes of JubJubScalar::to_bytes().  NOT a Montgomery image; values >= r_J are passed through (the device marks such an
    item invalid)."""
    vals = [int(v) for v in values]
    out = np.empty((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        if not 0 <= v < 1 << 256:
            raise ValueError("a JubJub scalar must be in [0, 2^256), got %d" % v)
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & _M64
    return out
