"""`encrypt` / `decrypt` -- mirror of src/encryption.rs over the GPU engine.
The shared secret is the (u, v) coordinate pair of the JubJubAffine point
(src/encryption.rs:71,92): a (2, 4) uint64 array."""
import numpy as np

from .engine import _engine_for, varlen_out_offsets
from .errors import DecryptionFailed, EncryptionFailed, Error, InvalidPoint
from .hash import pack_varlen
from .scalar import jubjub_limbs


def encrypt(message, shared_secret, nonce, engine=None):
    """src/encryption.rs:62-74 -> cipher with len(message)+1 scalars."""
    msg = np.ascontiguousarray(message, dtype=np.uint64).reshape(1, -1, 4)
    sec = np.ascontiguousarray(shared_secret, dtype=np.uint64).reshape(1, 2, 4)
    non = np.ascontiguousarray(nonce, dtype=np.uint64).reshape(1, 4)
    eng = _engine_for(engine)
    try:
        return eng.encrypt_batch(msg, sec, non)[0]
    except Error as e:                      # dusk-safe wraps pattern errors of encrypt
        raise EncryptionFailed() from e


def decrypt(cipher, shared_secret, nonce, engine=None):
    """src/encryption.rs:83-95; raises DecryptionFailed like the reference returns
    Err(Error::DecryptionFailed) (tests/encryption.rs:48-115)."""
    cip = np.ascontiguousarray(cipher, dtype=np.uint64).reshape(1, -1, 4)
    if cip.shape[1] < 2:
        raise DecryptionFailed()
    sec = np.ascontiguousarray(shared_secret, dtype=np.uint64).reshape(1, 2, 4)
    non = np.ascontiguousarray(nonce, dtype=np.uint64).reshape(1, 4)
    eng = _engine_for(engine)
    msg, ok = eng.decrypt_batch(cip, sec, non)
    if not ok[0]:
        raise DecryptionFailed()
    return msg[0]


def encrypt_batch(messages, secrets_uv, nonces, engine=None, out=None, async_=False):
    """NEW: n independent encrypt() calls.  (n, L, 4), (n, 2, 4), (n, 4) -> (n, L+1, 4)."""
    eng = _engine_for(engine, messages)
    return eng.encrypt_batch(messages, secrets_uv, nonces, out=out, async_=async_)


def decrypt_batch(ciphers, secrets_uv, nonces, engine=None, async_=False):
    """NEW: n independent decrypt() calls -> (messages (n, L, 4), ok (n,)); ok[i] == 0 marks the
    items for which the reference returns Error::DecryptionFailed (their message is zeroed)."""
    eng = _engine_for(engine, ciphers)
    return eng.decrypt_batch(ciphers, secrets_uv, nonces, async_=async_)


def _jscalar_row(secret):
    if isinstance(secret, (int, np.integer)):
        return jubjub_limbs([secret])
    return np.ascontiguousarray(secret, dtype=np.uint64).reshape(1, 4)


def dhke(secret, public, engine=None):
    """dhke(secret, public) = [secret] public, the shared secret encrypt / decrypt take (src/encryption.rs:11-43).
    secret: a canonical int < r_J or one p252_jscalar row (4,) uint64; public: the point's (u, v) as a (2, 4) array of
    BlsScalar.0 limbs -> (2, 4) uint64.  Raises InvalidPoint for a secret >= r_J or a point off the curve."""
    sec = _jscalar_row(secret)
    pub = np.ascontiguousarray(public, dtype=np.uint64).reshape(1, 2, 4)
    eng = _engine_for(engine)
    shared, ok = eng.dhke_batch(sec, pub)
    if not ok[0]:
        raise InvalidPoint()
    return shared[0]


def dhke_batch(secrets, publics, engine=None, out=None, async_=False):
    """NEW: n x dhke(secret, public).  secrets (1 or n, 4) p252_jscalar rows (scalar.jubjub_limbs), publics (1 or n, 2, 4)
    -> (shared (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose output is (0, 0)."""
    eng = _engine_for(engine, publics)
    return eng.dhke_batch(secrets, publics, out=out, async_=async_)


def encrypt_batch_dhke(messages, secrets, publics, nonces, engine=None, out=None, async_=False):
    """NEW: n x encrypt(messages[i], dhke(secret, public), nonces[i]), the shared secret derived on the device
    -> (ciphers (n, L+1, 4), ok (n,) uint8)."""
    eng = _engine_for(engine, messages)
    return eng.encrypt_batch_dhke(messages, secrets, publics, nonces, out=out, async_=async_)


def decrypt_batch_dhke(ciphers, secrets, publics, nonces, engine=None, out=None, async_=False):
    """NEW: n x decrypt(ciphers[i], dhke(secret, public), nonces[i]) -> (messages (n, L, 4), ok (n,) uint8); ok == 0 for
    an authentication failure or an invalid key-exchange item (message zeroed).  A wallet scan passes one view key."""
    eng = _engine_for(engine, ciphers)
    return eng.decrypt_batch_dhke(ciphers, secrets, publics, nonces, out=out, async_=async_)


def fixed_base(secret, base, engine=None):
    """[secret] base for one item: a public key GENERATOR_EXTENDED * secret when base is the generator's (u, v).
    secret: a canonical int < r_J or one p252_jscalar row (4,) uint64; base: (2, 4) BlsScalar.0 limbs -> (2, 4) uint64.
    Raises InvalidPoint for a secret >= r_J or a base off the curve.  There is no built-in generator: pass it."""
    sec = _jscalar_row(secret)
    eng = _engine_for(engine)
    out, ok = eng.fixed_base_batch(sec, base)
    if not ok[0]:
        raise InvalidPoint()
    return out[0]


def fixed_base_batch(secrets, base, engine=None, out=None, async_=False):
    """NEW: n x [secret] base for one base point.  secrets (n, 4) p252_jscalar rows (scalar.jubjub_limbs), base (2, 4)
    -> (points (n, 2, 4), ok (n,) uint8); ok == 0 marks a secret >= r_J, whose output is (0, 0)."""
    eng = _engine_for(engine, secrets)
    return eng.fixed_base_batch(secrets, base, out=out, async_=async_)


def encrypt_batch_ephemeral(messages, r, base, publics, nonces, engine=None, out=None, async_=False):
    """NEW: the sender (src/encryption.rs:22-42) as a batch: R_i = [r_i] base and
    cipher_i = encrypt(messages[i], dhke(r_i, publics[i]), nonces[i]), the shared secret derived on the device
    -> (ciphers (n, L+1, 4), R (n, 2, 4), ok (n,) uint8).  publics holds 1 or n receiver keys."""
    eng = _engine_for(engine, messages)
    return eng.encrypt_batch_ephemeral(messages, r, base, publics, nonces, out=out, async_=async_)


def stealth_address(r, base, A, B, engine=None):
    """NEW: one stealth address, the sender's PublicKey::gen_stealth_address: R = [r] base and
    note_pk = [hash([r] A)] base + B, hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0].  r: a canonical int
    < r_J or one p252_jscalar row; base, A, B: (2, 4) BlsScalar.0 limbs -> (R (2, 4), note_pk (2, 4)).  Raises
    InvalidPoint for r >= r_J or a point off the curve."""
    eng = _engine_for(engine)
    pt = lambda x: np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)   # noqa: E731
    R, pk, ok = eng.stealth_address_batch(_jscalar_row(r), base, pt(A), pt(B))
    if not ok[0]:
        raise InvalidPoint()
    return R[0], pk[0]


def stealth_address_batch(r, base, publics_A, publics_B, engine=None, async_=False):
    """NEW: n stealth addresses.  r (n, 4) p252_jscalar rows, base (2, 4), publics_A / publics_B (1 or n, 2, 4)
    -> (R (n, 2, 4), note_pk (n, 2, 4), ok (n,) uint8); ok == 0 marks an invalid item, whose rows are zeroed."""
    eng = _engine_for(engine, r)
    return eng.stealth_address_batch(r, base, publics_A, publics_B, async_=async_)


def owns(view_a, spend_B, base, R, note_pk, engine=None):
    """NEW: ViewKey::owns for one note: note_pk == [hash([view_a] R)] base + spend_B -> bool.  view_a: a canonical int
    < r_J or one p252_jscalar row; spend_B, base, R, note_pk: (2, 4) BlsScalar.0 limbs.  Raises InvalidPoint for
    view_a >= r_J, R off the curve, a note_pk coordinate >= p, or spend_B or base off the curve."""
    eng = _engine_for(engine)
    pt = lambda x: np.ascontiguousarray(x, dtype=np.uint64).reshape(1, 2, 4)   # noqa: E731
    owned = eng.stealth_owns_batch(_jscalar_row(view_a), spend_B, base, pt(R), pt(note_pk))
    if eng.last_stealth_invalid():
        raise InvalidPoint()
    return bool(owned[0])


def stealth_owns_batch(view_a, spend_B, base, R, note_pk, engine=None, async_=False):
    """NEW: a wallet's scan with one view key: owned[i] = note_pk[i] == [hash([view_a] R[i])] base + spend_B.
    view_a (1, 4), R and note_pk (n, 2, 4), spend_B and base (2, 4) -> owned (n,) uint8 (0 also for an invalid item)."""
    eng = _engine_for(engine, R)
    return eng.stealth_owns_batch(view_a, spend_B, base, R, note_pk, async_=async_)


def cipher_offsets(offsets):
    """Offsets of the ciphers of messages at `offsets` (each one scalar longer, packed from 0): offsets - offsets[0] + i.
    Works on numpy arrays and CUDA tensors (no host sync)."""
    return varlen_out_offsets(offsets, 1)


def message_offsets(offsets):
    """Offsets of the messages of ciphers at `offsets` (each one scalar shorter, packed from 0): offsets - offsets[0] - i."""
    return varlen_out_offsets(offsets, -1)


def _split(flat, offsets):
    return [flat[int(offsets[i]):int(offsets[i + 1])] for i in range(len(offsets) - 1)]


def encrypt_batch_varlen(messages, secrets_uv, nonces, engine=None, max_len=None, out=None, async_=False):
    """NEW: n independent encrypt() calls over messages of different lengths, one device call.
    messages: a list of (k_i, 4) host arrays (packed by `pack_varlen`) -> a list of (k_i + 1, 4) ciphers; or a
    `(data, offsets)` pair as taken by `Engine.encrypt_batch_varlen` (numpy or CUDA tensors) -> (cipher, cipher_offsets)."""
    if isinstance(messages, tuple):
        data, offsets = messages
        eng = _engine_for(engine, data)
        return eng.encrypt_batch_varlen(data, offsets, secrets_uv, nonces, max_len=max_len, out=out, async_=async_)
    data, offsets, longest = pack_varlen(messages)
    eng = _engine_for(engine)
    cipher, coff = eng.encrypt_batch_varlen(data, offsets, secrets_uv, nonces,
                                            max_len=max(longest, 1) if max_len is None else max_len, out=out)
    return _split(cipher, coff)


def decrypt_batch_varlen(ciphers, secrets_uv, nonces, engine=None, max_len=None, async_=False):
    """NEW: n independent decrypt() calls over ciphers of different lengths, one device call.
    ciphers: a list of (k_i + 1, 4) host arrays -> (list of (k_i, 4) messages, ok (n,) uint8); or a `(data, offsets)`
    pair as taken by `Engine.decrypt_batch_varlen` -> (msg, msg_offsets, ok).  ok[i] == 0 marks the items for which the
    reference returns Error::DecryptionFailed (their message is zeroed)."""
    if isinstance(ciphers, tuple):
        data, offsets = ciphers
        eng = _engine_for(engine, data)
        return eng.decrypt_batch_varlen(data, offsets, secrets_uv, nonces, max_len=max_len, async_=async_)
    data, offsets, longest = pack_varlen(ciphers)
    eng = _engine_for(engine)
    msg, moff, ok = eng.decrypt_batch_varlen(data, offsets, secrets_uv, nonces,
                                             max_len=max(longest - 1, 1) if max_len is None else max_len)
    return _split(msg, moff), ok
