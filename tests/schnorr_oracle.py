"""Pure-Python model of the Schnorr signatures of p252_schnorr_sign_batch / p252_schnorr_verify_batch.

    challenge(R, m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0]      (R affine; c < 2^250 < r_J)
    sign   (sk, r; m):        R = [r] G,   c = challenge(R, m),   u = (r - c sk) mod r_J,   signature = (u, R)
    verify (PK; (u, R), m):   ok  <=>  [u] G + [c] PK == R

Built from jubjub_oracle.py (affine complete addition, double-and-add) and hades_oracle.Hash.digest_truncated -- formulas
independent of the kernels' (table walks, extended coordinates, projective comparison).  The formulas are
jubjub-schnorr's SecretKey::sign / PublicKey::verify as recalled, not checked against that crate (it is not vendored):
the library's contract is the formulas above.

The second half models the kernel's arithmetic modulo r_J limb by limb (jubjub_device.cuh: order_mont, order_mul,
order_sub), so that its carries and corrections can be checked against big integers on the CPU."""
import hades_oracle as ho
import jubjub_oracle as jo

G = jo.GENERATOR


def challenge(R, m):
    """c of the model: the truncated digest of (R.u, R.v, m), a canonical JubJub scalar < 2^250"""
    return ho.Hash.digest_truncated(ho.Domain.Other, [R[0], R[1], m])[0]


def public_key(sk, base=G):
    return jo.mul(sk, base)


def sign(sk, r, m, base=G):
    """(u, R), or None where the batch call reports ok = 0 (sk or r >= r_J, m >= p)"""
    if not (0 <= sk < jo.R_J) or not (0 <= r < jo.R_J) or not (0 <= m < jo.P):
        return None
    R = jo.mul(r, base)
    return (r - challenge(R, m) * sk) % jo.R_J, R


def verify(pk, u, R, m, base=G):
    """1 verified, 0 not verified, None invalid (u >= r_J, m >= p, an R coordinate >= p, PK not a curve point)"""
    if not (0 <= u < jo.R_J) or not (0 <= m < jo.P) or not all(0 <= x < jo.P for x in R) or not jo.on_curve(pk):
        return None
    return int(jo.add(jo.mul(u, base), jo.mul(challenge(R, m), pk)) == tuple(R))


# ---- the kernel's arithmetic modulo r_J, on 8 x 32-bit limbs --------------------------------------------------------
W = 32
MASK = (1 << W) - 1
N = jo.R_J
RR = 1 << 256                                   # the Montgomery radix
ORDER_INV = (-pow(N, -1, 1 << W)) % (1 << W)    # kOrderInv
ORDER_R2 = RR * RR % N                           # P252_JJ_ORDER_R2


def limbs(x):
    return [(x >> (W * k)) & MASK for k in range(8)]


def value(ls):
    return sum(v << (W * k) for k, v in enumerate(ls))


def order_mont(a, b, trace=None):
    """order_mont of the kernel: a b / 2^256 mod r_J for a, b < r_J, row by row as the kernel does it; every word
    stays 32 bits and every carry fits 64.  trace (a list) receives True when the final subtraction of r_J is taken."""
    al, bl, n = limbs(a), limbs(b), limbs(N)
    t = [0] * 8
    for i in range(8):
        c = 0
        for j in range(8):
            c += al[j] * bl[i] + t[j]
            assert c < 1 << 64
            t[j], c = c & MASK, c >> W
        hi = c
        m = (t[0] * ORDER_INV) & MASK
        c = (m * n[0] + t[0])
        assert c & MASK == 0
        c >>= W
        for j in range(1, 8):
            c += m * n[j] + t[j]
            assert c < 1 << 64
            t[j - 1], c = c & MASK, c >> W
        assert c + hi <= MASK                   # the row's top word: t < a + r_J < 2^256
        t[7] = c + hi
    tv = value(t)
    assert tv < 2 * N
    taken = tv >= N
    if trace is not None:
        trace.append(taken)
    return tv - N if taken else tv


def order_mul(a, b, trace=None):
    """a b mod r_J: two Montgomery products, the second by R^2 mod r_J"""
    return order_mont(order_mont(a, b, trace), ORDER_R2, trace)


def order_sub(a, b, trace=None):
    """a - b mod r_J for a, b < r_J: trace receives True when r_J is added back (a < b)"""
    d = (a - b) % RR
    borrow = a < b
    if trace is not None:
        trace.append(borrow)
    return (d + N) % RR if borrow else d


def sign_u(sk, r, c):
    """u as the sign kernel computes it"""
    return order_sub(r, order_mul(c, sk))
