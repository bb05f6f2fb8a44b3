"""Pure-Python model of the Phoenix note values of p252_value_commit_batch / p252_note_create_batch /
p252_note_open_batch.

    commit(v, blinder) = C = [v] G + [blinder] G'                              (v < 2^64, blinder < r_J)
    create (r, v, blinder, nonce; A, B):  R = [r] G,  S = [r] A,  note_pk = [hash(S)] G + B,  C = commit(v, blinder),
                                          cipher = encrypt([v, blinder], S, nonce)                     (3 scalars)
    open  (a; R, nonce, cipher, C):       (m0, m1) = decrypt(cipher, [a] R, nonce); the note opens iff the
                                          authentication passes, m0 < 2^64, m1 < r_J and commit(m0, m1) == C

Built from jubjub_oracle.py (affine complete addition, double-and-add, encrypt / decrypt over the Python Hades) and
stealth_oracle.py (stealth_address, hash_point) -- formulas independent of the kernels' (table walks with signed digits,
extended coordinates, projective comparison).  The formulas are phoenix-core's Note::new (obfuscated) and Note::value /
value_blinder as recalled, not checked against that crate (it is not vendored): the library's contract is the formulas
above.  The range checks of open are the library's own rule."""
import hades_oracle as ho
import jubjub_oracle as jo
import stealth_oracle as so

G = jo.GENERATOR
V_MAX = 1 << 64


def commit(v, blinder, Gp, base=G):
    """C, or None where the batch call reports ok = 0 (blinder >= r_J); v must be a u64"""
    assert 0 <= v < V_MAX
    if not (0 <= blinder < jo.R_J):
        return None
    return jo.add(jo.mul(v, base), jo.mul(blinder, Gp))


def create(r, v, blinder, nonce, A, B, Gp, base=G):
    """(R, note_pk, C, cipher), or None where the batch call reports ok = 0 (r or blinder >= r_J, A or B not a curve
    point)"""
    note = so.stealth_address(r, A, B, base)
    C = commit(v, blinder, Gp, base)
    if note is None or C is None:
        return None
    S = jo.mul(r, A)
    return note[0], note[1], C, ho.encrypt([v, blinder], list(S), nonce)


def valid_opening(a, R):
    """the item checks of open: a < r_J and R a curve point"""
    return 0 <= a < jo.R_J and jo.on_curve(R)


def decrypt_rows(a, R, nonce, cipher):
    """the plaintext (m0, m1) the device decrypts, or None where the authentication fails"""
    try:
        return tuple(ho.decrypt(list(cipher), list(jo.mul(a, R)), nonce))
    except ho.DecryptionFailed:
        return None


def open_note(a, R, nonce, cipher, C, Gp, base=G):
    """(v, blinder) if the note opens, None otherwise (invalid item included)"""
    if not valid_opening(a, R) or not all(0 <= c < jo.P for c in C):
        return None
    m = decrypt_rows(a, R, nonce, cipher)
    if m is None or not (0 <= m[0] < V_MAX and 0 <= m[1] < jo.R_J):
        return None
    return m if jo.add(jo.mul(m[0], base), jo.mul(m[1], Gp)) == tuple(C) else None


def recode_u64(v):
    """the kernel's recoding of a u64 for the 17-window walk: 16 signed digits in [-8, 8), least significant first, and
    the final carry digit in {0, 1}; v = sum e_w 16^w"""
    digits, carry = [], 0
    for _ in range(16):
        x = (v & 15) + carry
        v >>= 4
        carry = (x + 8) >> 4
        digits.append(x - 16 * carry)
    return digits + [carry]


def walk_u64(v, base, acc=jo.IDENTITY):
    """acc + [v] base by the walk of recode_u64: one addition of e_w (16^w base) per window, as the fixed-base table
    holds it"""
    for w, e in enumerate(recode_u64(v)):
        entry = jo.mul(abs(e) * 16 ** w, base)
        acc = jo.add(acc, entry if e >= 0 else jo.neg(entry))
    return acc
