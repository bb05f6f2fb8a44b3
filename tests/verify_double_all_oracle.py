"""Model of p252_schnorr_verify_double_all, composed from schnorr_double_oracle.challenge2 and msm_oracle.msm:

    verify_double_all(...) = [8] ( [sum z u] G + [sum z' u] G' + sum [z c] PK + sum [z' c] PK' - sum [z] R - sum [z'] R' )
                             == O,    c = challenge2(R, R', m)

and the per-item equations the batch answer stands for, both cofactored:

    [8] ([u] G + [c] PK - R) == O   and   [8] ([u] G' + [c] PK' - R') == O

The sum runs through msm_oracle.msm (affine complete addition, double-and-add), so it shares no code with the kernels
(bucket MSM, fixed-base tables, extended coordinates)."""
import jubjub_oracle as jo
import msm_oracle as mo
import schnorr_double_oracle as sdo

N, P, G = jo.R_J, jo.P, jo.GENERATOR


def item_valid(pk, pkp, u, R, Rp, m, z, zp):
    """the validity of p252_schnorr_verify_double_batch plus z, z' < r_J"""
    canon = all(0 <= x < P for x in tuple(R) + tuple(Rp))
    return (0 <= u < N and 0 <= m < P and canon and jo.on_curve(pk) and jo.on_curve(pkp) and 0 <= z < N
            and 0 <= zp < N)


def verify_double_all(pks, pkps, us, Rs, Rps, ms, ws, wps, Gp, base=G, cofactor=8):
    """True iff every item is valid, every R and R' is on the curve and the cofactored weighted sum is the identity.
    pks / pkps hold 1 or n points."""
    n = len(us)
    sc, pts = [], []
    zu = zpu = 0
    for i in range(n):
        pk, pkp = (pks[0], pkps[0]) if len(pks) == 1 else (pks[i], pkps[i])
        u, R, Rp, m, z, zp = us[i], tuple(Rs[i]), tuple(Rps[i]), ms[i], ws[i], wps[i]
        if not item_valid(pk, pkp, u, R, Rp, m, z, zp):
            return False
        if not (jo.on_curve(R) and jo.on_curve(Rp)):
            return False
        c = sdo.challenge2(R, Rp, m)
        zu, zpu = (zu + z * u) % N, (zpu + zp * u) % N
        sc += [z * c % N, zp * c % N, z, zp]
        pts += [pk, pkp, jo.neg(R), jo.neg(Rp)]
    acc = mo.msm([zu, zpu] + sc, [base, Gp] + pts)
    return jo.mul(cofactor, acc) == jo.IDENTITY


def cofactored_items(pk, pkp, u, R, Rp, m, Gp, base=G):
    """both per-item equations, cofactored"""
    c = sdo.challenge2(R, Rp, m)
    one = jo.add(jo.add(jo.mul(u, base), jo.mul(c, pk)), jo.neg(R))
    two = jo.add(jo.add(jo.mul(u, Gp), jo.mul(c, pkp)), jo.neg(Rp))
    return jo.mul(8, one) == jo.IDENTITY and jo.mul(8, two) == jo.IDENTITY


def cancelling_signature(sk, r, m, D, Gp, base=G):
    """(u, R, R') with R = [r] G + D and R' = [r] G' - D, signed as usual: each equation is off by -D and +D, so the
    per-item check fails (for D of order r_J) and the sum of the two equations holds"""
    R = jo.add(jo.mul(r, base), D)
    Rp = jo.add(jo.mul(r, Gp), jo.neg(D))
    return (r - sdo.challenge2(R, Rp, m) * sk) % N, R, Rp


__all__ = ["item_valid", "verify_double_all", "cofactored_items", "cancelling_signature"]
