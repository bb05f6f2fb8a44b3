"""Models of p252_jubjub_msm and p252_schnorr_verify_all.

    msm(s, P)            = sum [s_i] P_i                        (jubjub_oracle: affine complete addition, double-and-add)
    verify_all(...)      = [8] ([sum z u] G + sum [z c] PK - sum [z] R) == O,   c = schnorr_oracle.challenge(R, m)

The second half models the kernels' algorithm (jubjub_device.cuh / kernels.cu) over the additive group Z/r_J, a point being
its discrete log: c-bit signed recoding, the (window, bucket) keys and their sentinel, the passes of k_msm_bucket over
pieces of sorted entries with their carries, the running sums of k_msm_window with the offset correction, and the
window combination of k_msm_final.  Group sums there are additions of integers, so the model runs at 2^16 items and
checks the indexing, not the curve arithmetic."""
import jubjub_edges as je
import jubjub_oracle as jo
import schnorr_oracle as so

N = jo.R_J
G = jo.GENERATOR
MIN_BITS, MAX_BITS = 4, 13          # kMsmMinBits, kMsmMaxBits
PIECE = 32                          # kMsmPiece
THREADS = 128                       # kMsmThreads
PRODUCTS_PER_DIGIT, PRODUCTS_PER_BUCKET = 7, 18


def msm(scalars, points):
    """sum [s_i] P_i over the valid items (s < r_J, P on the curve with canonical coordinates)"""
    acc = jo.IDENTITY
    for s, pt in zip(scalars, points):
        if 0 <= s < N and all(0 <= x < jo.P for x in pt) and jo.on_curve(pt):
            acc = jo.add(acc, jo.mul(s, pt))
    return acc


def edge_points(limit=48):
    """curve points whose coordinates and Niels entries sit at the field's edges (jubjub_edges.py)"""
    seen = []
    for e in je.all_edges():
        if e.pt not in seen:
            seen.append(e.pt)
        if len(seen) == limit:
            break
    return seen


def edge_scalars():
    """0, 1, r_J - 1, powers of two, every 13-bit digit at -2^12 (and the 4-bit one at -8), the top-window carry"""
    out = [0, 1, 2, N - 1, N - 2, 1 << 251, (1 << 251) - 1]
    out += [1 << k for k in (12, 13, 64, 128, 200, 247)]
    for c in (4, 13):
        out.append(all_low_digits_negative(c))                            # digit -2^(c-1) in every window below the top
        out.append(((1 << (c * (windows(c) - 1))) - 1) % N)               # all low windows carry into the top one
    return out


def all_low_digits_negative(c):
    """the scalar whose digits below the top window are all -2^(c-1): window 0 holds 2^(c-1), the others 2^(c-1) - 1
    (plus the carry 1), and the top window takes the last carry"""
    half = 1 << (c - 1)
    return half + sum((half - 1) << (c * w) for w in range(1, windows(c) - 1))


def verify_all(pks, us, Rs, ms, ws, base=G, cofactor=8):
    """True iff every item is valid, every R on the curve and [cofactor] ([sum z u] G + sum [z c] PK - sum [z] R) == O"""
    n = len(us)
    acc = jo.IDENTITY
    zu = 0
    for i in range(n):
        pk = pks[0] if len(pks) == 1 else pks[i]
        u, R, m, z = us[i], Rs[i], ms[i], ws[i]
        if not (0 <= u < N and 0 <= z < N and 0 <= m < jo.P and all(0 <= x < jo.P for x in R) and jo.on_curve(pk)):
            return False
        if not jo.on_curve(R):
            return False
        c = so.challenge(R, m)
        zu = (zu + z * u) % N
        acc = jo.add(acc, jo.add(jo.mul(z * c % N, pk), jo.neg(jo.mul(z, R))))
    return jo.mul(cofactor, jo.add(acc, jo.mul(zu, base))) == jo.IDENTITY


def cofactored_item(pk, u, R, m, base=G):
    """the per-item equation the batch answer stands for: [8] ([u] G + [c] PK - R) == O"""
    c = so.challenge(R, m)
    return jo.mul(8, jo.add(jo.add(jo.mul(u, base), jo.mul(c, pk)), jo.neg(R))) == jo.IDENTITY


# ---- the kernels' algorithm over Z/r_J --------------------------------------------------------------------------------
def windows(c):
    """W(c) = ceil(253 / c): the top window holds at most c - 1 bits of s < 2^252, so it takes no carry out"""
    return -(-253 // c)


def recode(s, c):
    """recode_window over all windows: digits e_w in [-2^(c-1), 2^(c-1)), the top one in [0, 2^(c-1)]"""
    W = windows(c)
    out, carry = [], 0
    for w in range(W):
        x = (s & ((1 << c) - 1)) + carry
        s >>= c
        if w == W - 1:
            out.append(x)
            carry = 0
        else:
            carry = (x + (1 << (c - 1))) >> c
            out.append(x - (carry << c))
    assert s == 0 and carry == 0
    return out


def bits_for(rows):
    """msm_bits: the window width with the fewest products for chunks of `rows` rows"""
    cost = lambda c: rows * windows(c) * PRODUCTS_PER_DIGIT + windows(c) * (1 << (c - 1)) * PRODUCTS_PER_BUCKET
    return min(range(MIN_BITS, MAX_BITS + 1), key=lambda c: (cost(c), c))


def keys(scalars, c):
    """k_msm_prep: window-major (key, value) entries; value = (row, negative), sentinel W B for a zero digit"""
    W, B = windows(c), 1 << (c - 1)
    m = len(scalars)
    digits = [recode(s, c) for s in scalars]
    return [((w * B + abs(digits[i][w]) - 1) if digits[i][w] else W * B, (i, digits[i][w] < 0))
            for w in range(W) for i in range(m)]


def bucket_pass(entries, nb, buckets, value, piece=PIECE):
    """one k_msm_bucket pass over key-sorted entries (key, payload); payload None is an empty slot.  Whole runs go to
    buckets (each key written once), runs crossing a piece boundary to the returned list (None for one piece)."""
    n = len(entries)
    pieces = -(-n // piece)
    out = [None] * (2 * pieces) if pieces > 1 else None
    work = 0
    for t in range(pieces):
        lo, hi = t * piece, min(n, t * piece + piece)
        prevk = entries[lo - 1][0] if lo > 0 else None
        nextk = entries[hi][0] if hi < n else None
        head = tail = False
        i = lo
        while i < hi:
            k = entries[i][0]
            acc, any_, j = 0, False, i
            while j < hi and entries[j][0] == k:
                if k < nb and entries[j][1] is not None:
                    acc = (acc + value(entries[j][1])) % N
                    any_ = True
                    work += 1
                j += 1
            first = i == lo
            if (first and prevk == k) or (j == hi and nextk == k):
                out[2 * t + (0 if first else 1)] = (k, acc if any_ else None)
                head, tail = head or first, tail or not first
            elif any_:
                assert k not in buckets
                buckets[k] = acc
            i = j
        if out is not None:
            if not head:
                out[2 * t] = (entries[lo][0], None)
            if not tail:
                out[2 * t + 1] = (entries[hi - 1][0], None)
    return out, work


def window_parts(c):
    B = 1 << (c - 1)
    return min(THREADS, B // 32) if B >= 32 else 1


def window_sum(buckets, w, c):
    """k_msm_window: per part, running sums from the top (r = sum B, t = sum (j + 1) B), then t + lo r"""
    B = 1 << (c - 1)
    P = window_parts(c)
    L = B // P
    total = 0
    for p in range(P):
        lo = p * L
        r = t = 0
        for j in reversed(range(L)):
            r = (r + buckets.get(w * B + lo + j, 0)) % N
            t = (t + r) % N
        total = (total + t + lo * r) % N
    return total


def msm_model(scalars, logs, c=None, chunk=None, piece=PIECE, stats=None):
    """sum s_i log_i mod r_J the way the kernels compute it (chunks, keys, sorted passes, windows, Horner)"""
    n = len(scalars)
    chunk = chunk or max(n, 1)
    c = c or bits_for(chunk)
    W, B = windows(c), 1 << (c - 1)
    nb = W * B
    S = [0] * W
    for off in range(0, n, chunk):
        sc, lg = scalars[off:off + chunk], logs[off:off + chunk]
        ent = sorted(keys(sc, c), key=lambda e: e[0])         # the radix sort (stable, as CUB's)
        buckets = {}
        value = lambda v: -lg[v[0]] if v[1] else lg[v[0]]
        lst, work = bucket_pass(ent, nb, buckets, value, piece)
        passes, most = 1, work
        while lst is not None:
            lst, work = bucket_pass(lst, nb, buckets, lambda v: v, piece)
            passes += 1
        if stats is not None:
            stats.append(passes)
        for w in range(W):
            S[w] = (S[w] + window_sum(buckets, w, c)) % N
    acc = S[W - 1]
    for w in reversed(range(W - 1)):
        acc = ((acc << c) + S[w]) % N
    return acc


def plain_sum(scalars, logs):
    return sum(s * g for s, g in zip(scalars, logs)) % N


__all__ = ["msm", "verify_all", "cofactored_item", "windows", "recode", "keys", "bucket_pass", "window_sum", "msm_model",
           "plain_sum", "bits_for", "edge_points", "edge_scalars"]
