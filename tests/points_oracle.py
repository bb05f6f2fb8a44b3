"""Pure-Python model of JubJub point compression (dusk-jubjub's JubJubAffine::to_bytes / from_bytes) on big integers, and a
restatement of the kernel's square root (RFC 9380 Appendix F.2.1.1 sqrt_ratio, jubjub_device.cuh) step by step.

    encode(u, v):  the 32 little-endian bytes of canonical v, bit 255 = the low bit of u
    decode(b):     sign = bit 255, cleared; v = the rest (None if >= p); u^2 = (v^2 - 1) / (1 + d v^2) (None if not a
                   square); u = the root with low bit sign (p - root otherwise; for u = 0 a set sign is accepted)

decode solves with jubjub_oracle.sqrt (Tonelli-Shanks), not with sqrt_ratio, so that agreement between the kernel and this
model is an independent check.  Pinned: the formulas above follow from the curve equation.  Recollection, not checked
against the crate (dusk-jubjub is not vendored): that dusk-jubjub accepts a set sign bit with u = 0 (pre-ZIP-216)."""
import jubjub_oracle as jo

P = jo.P
Z = 5                                       # a non-residue mod p (jubjub_oracle.SQRT_M1 is Z^((p-1)/4))
C1 = 32                                     # p - 1 = 2^C1 T, T odd
T = (P - 1) >> C1
C3 = (T - 1) // 2
C6 = pow(Z, T, P)
C7 = pow(Z, (T + 1) // 2, P)
FF = b"\xff" * 32                           # the encoding of an invalid to_bytes item


def encode(pt):
    """JubJubAffine::to_bytes of a curve point (u, v) of canonical ints; None for a coordinate >= p or off the curve"""
    if not jo.on_curve(pt):
        return None
    u, v = pt
    return (v | (u & 1) << 255).to_bytes(32, "little")


def decode(b):
    """JubJubAffine::from_bytes of 32 bytes -> (u, v), or None"""
    x = int.from_bytes(bytes(b), "little")
    sign, v = x >> 255, x & ((1 << 255) - 1)
    if v >= P:
        return None
    vv = v * v % P
    u = jo.sqrt((vv - 1) * pow((1 + jo.D * vv) % P, -1, P) % P)
    if u is None:
        return None
    if (u & 1) != sign:
        u = (P - u) % P
    return (u, v)


def sqrt_ratio(num, den, trace=None):
    """The kernel's sqrt_ratio on ints mod p, step for step (RFC numbering) -> (is_square, y): y^2 = num / den if
    is_square, else y^2 = Z num / den.  num = 0 counts as a square (the RFC's own is_square is false there).  trace: a
    list that receives (k, e1) for every loop round k = 32..2, the conditional moves of steps 25-26."""
    tv1 = C6                                            # 1.
    tv2 = den
    k = 1
    while k < C1:                                       # 2. den^(2^32 - 1): x^(2^2k - 1) = (x^(2^k - 1))^(2^k) x^(2^k - 1)
        tv2 = pow(tv2, 1 << k, P) * tv2 % P
        k *= 2
    tv3 = tv2 * tv2 % P                                 # 3.
    tv3 = tv3 * den % P                                 # 4.
    tv5 = num * tv3 % P                                 # 5.
    tv5 = pow(tv5, C3, P)                               # 6.
    tv5 = tv5 * tv2 % P                                 # 7.
    tv2 = tv5 * den % P                                 # 8.
    tv3 = tv5 * num % P                                 # 9.
    tv4 = tv3 * tv2 % P                                 # 10.
    tv5 = pow(tv4, 1 << (C1 - 1), P)                    # 11.
    is_qr = tv5 == 1                                    # 12.
    tv2 = tv3 * C7 % P                                  # 13.
    tv5 = tv4 * tv1 % P                                 # 14.
    tv3 = tv3 if is_qr else tv2                         # 15.
    tv4 = tv4 if is_qr else tv5                         # 16.
    for k in range(C1, 1, -1):                          # 17.
        tv5 = pow(tv4, 1 << (k - 2), P)                 # 18.-20.
        e1 = tv5 == 1                                   # 21.
        tv2 = tv3 * tv1 % P                             # 22.
        tv1 = tv1 * tv1 % P                             # 23.
        tv5 = tv4 * tv1 % P                             # 24.
        tv3 = tv3 if e1 else tv2                        # 25.
        tv4 = tv4 if e1 else tv5                        # 26.
        if trace is not None:
            trace.append((k, e1))
    return (is_qr or num % P == 0), tv3


def decode_kernel(b):
    """decode with the kernel's steps (sqrt_ratio, no inversion) -> (u, v) or None"""
    x = int.from_bytes(bytes(b), "little")
    sign, v = x >> 255, x & ((1 << 255) - 1)
    if v >= P:
        return None
    vv = v * v % P
    square, r = sqrt_ratio((vv - 1) % P, (1 + jo.D * vv) % P)
    if not square:
        return None
    return (r if (r & 1) == sign else (P - r) % P, v)


# ---- boundary representations -----------------------------------------------------------------------------------
def bytes_rows(encodings):
    """list of 32-byte strings -> (n, 32) uint8"""
    import numpy as np
    return np.frombuffer(b"".join(encodings), dtype=np.uint8).reshape(len(encodings), 32).copy()
