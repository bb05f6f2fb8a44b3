"""Pure-Python model of the JubJub key exchange (dhke) and of encrypt / decrypt with a derived shared secret.

The curve is JubJub, a u^2 + v^2 = 1 + d u^2 v^2 over BLS12-381 Fr with a = -1 and d = -10240/10241.  The model adds
points with the AFFINE complete addition law and multiplies MSB-first by double-and-add -- deliberately different formulas
from the kernel's (extended coordinates, 4-bit window, one inversion at the end), so that agreement is an independent
check.  [s]P is unique and affine coordinates are canonical, so any correct algorithm is bit-exact.

Pinned: the curve constants below (re-checked by tests/test_jubjub_cpu.py).  Recollection, not checked against the crate
(dusk-jubjub is not vendored): that `dhke(&JubJubScalar, &JubJubExtended) -> JubJubAffine` is the reference's signature
and that GENERATOR below equals dusk-jubjub's GENERATOR.  No test depends on either."""
import hades_oracle as ho

P = ho.P
A = P - 1                                   # a = -1
D = (-10240 * pow(10241, -1, P)) % P
D_HEX = 0x2a9318e74bfa2b48f5fd9207e6bd7fd4292d7f6d37579d2601065fd6d6343eb1
R_J = 0x0e7db4ea6533afa906673b0101343b00a6682093ccc81082d0970e5ed6f72cb7
COFACTOR = 8
IDENTITY = (0, 1)
GENERATOR = (0x3fd2814c43ac65a6f1fbf02d0fd6cce62e3ebb21fd6c54ed4df7b7ffec7beaca, 18)
SQRT_M1 = pow(5, (P - 1) // 4, P)           # 5 is a non-residue mod p, so 5^((p-1)/4) squares to -1


def on_curve(pt):
    """u, v < p and a u^2 + v^2 == 1 + d u^2 v^2"""
    u, v = pt
    if not (0 <= u < P and 0 <= v < P):
        return False
    uu, vv = u * u % P, v * v % P
    return (A * uu + vv) % P == (1 + D * uu % P * vv) % P


def add(p1, p2):
    """Complete affine addition (d non-square, a square): no exceptional inputs."""
    u1, v1 = p1
    u2, v2 = p2
    t = D * u1 % P * u2 % P * v1 % P * v2 % P
    u3 = (u1 * v2 + v1 * u2) * pow((1 + t) % P, -1, P) % P
    v3 = (v1 * v2 - A * u1 * u2) * pow((1 - t) % P, -1, P) % P
    return (u3, v3)


def neg(pt):
    return ((-pt[0]) % P, pt[1])


def mul(k, pt):
    """[k] pt, MSB-first double-and-add (k >= 0)"""
    acc = IDENTITY
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc


def dhke(secret, public):
    """[secret] public in affine coordinates; None where the batch calls report ok = 0 (and the single-item front end
    raises InvalidPoint): secret >= r_J or public not a curve point."""
    if not (0 <= secret < R_J) or not on_curve(public):
        return None
    return mul(secret, public)


def sqrt(x):
    """a square root mod p (Tonelli-Shanks), or None"""
    x %= P
    if x == 0:
        return 0
    if pow(x, (P - 1) // 2, P) != 1:
        return None
    q, s = P - 1, 0
    while q % 2 == 0:
        q, s = q // 2, s + 1
    z = 5
    m, c, t, r = s, pow(z, q, P), pow(x, q, P), pow(x, (q + 1) // 2, P)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % P, i + 1
        b = pow(c, 1 << (m - i - 1), P)
        m, c, t, r = i, b * b % P, t * b * b % P, r * b % P
    return r


def point_from_v(v):
    """a curve point with this v (solving the curve equation for u), or None: u^2 = (1 - v^2) / (a - d v^2)"""
    vv = v * v % P
    den = (A - D * vv) % P
    if den == 0:
        return None
    u = sqrt((1 - vv) * pow(den, -1, P) % P)
    return None if u is None else (u, v % P)


def random_point(rng):
    """a uniformly chosen point of the full group (order dividing 8 r_J, usually 8 r_J)"""
    while True:
        pt = point_from_v(int(rng.integers(0, 1 << 62)) << 190 | int(rng.integers(0, 1 << 62)))
        if pt is not None:
            return pt if rng.integers(0, 2) else neg(pt)


def random_subgroup_point(rng):
    """[k] G for a random k < r_J"""
    return mul(random_secret(rng), GENERATOR)


def random_secret(rng):
    return int.from_bytes(rng.integers(0, 256, 32, dtype="uint8").tobytes(), "little") % R_J


def order8_point(rng):
    """a point of order exactly 8: [r_J] P for a random P of full order"""
    while True:
        q = mul(R_J, random_point(rng))
        if mul(4, q) != IDENTITY:
            return q


def small_order_points(rng):
    """the identity, (0, -1) of order 2, (+-sqrt(-1), 0) of order 4, a point of order 8"""
    return [IDENTITY, (0, P - 1), (SQRT_M1, 0), (P - SQRT_M1, 0), order8_point(rng)]


def off_curve_point(rng):
    while True:
        pt = (int(rng.integers(0, 1 << 62)) << 190, int(rng.integers(0, 1 << 62)))
        if not on_curve(pt):
            return pt


def encrypt(message, secret, public, nonce):
    """encrypt(message, dhke(secret, public), nonce) on canonical ints (hades_oracle)"""
    return ho.encrypt(message, list(dhke(secret, public)), nonce)


def decrypt(cipher, secret, public, nonce):
    return ho.decrypt(cipher, list(dhke(secret, public)), nonce)


# ---- boundary representations -----------------------------------------------------------------------------------
def jscalar_limbs(values):
    """canonical ints -> p252_jscalar rows (n, 4) uint64 (JubJubScalar::to_bytes as little-endian u64 limbs)"""
    import numpy as np
    out = np.zeros((len(values), 4), dtype=np.uint64)
    for i, v in enumerate(values):
        for k in range(4):
            out[i, k] = (int(v) >> (64 * k)) & ((1 << 64) - 1)
    return out


def points_mont(points):
    """affine points (u, v) of ints (< 2^256, not reduced) -> (n, 2, 4) uint64 Montgomery limbs; a coordinate >= p is
    passed through as the raw limbs of that value, so that the device sees it unreduced"""
    import numpy as np
    out = np.zeros((len(points), 2, 4), dtype=np.uint64)
    for i, pt in enumerate(points):
        for j, c in enumerate(pt):
            m = c * ho.R % P if c < P else c
            for k in range(4):
                out[i, j, k] = (m >> (64 * k)) & ((1 << 64) - 1)
    return out


def points_from_mont(arr):
    """(n, 2, 4) Montgomery limbs -> list of (u, v) ints"""
    res = []
    for row in arr:
        u, v = (sum(int(row[j, k]) << (64 * k) for k in range(4)) * pow(ho.R, -1, P) % P for j in range(2))
        res.append((u, v))
    return res
