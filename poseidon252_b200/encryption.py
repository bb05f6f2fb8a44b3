"""`encrypt` / `decrypt` -- mirror of src/encryption.rs over the GPU engine.
The shared secret is the (u, v) coordinate pair of the JubJubAffine point
(src/encryption.rs:71,92): a (2, 4) uint64 array."""
import numpy as np

from .engine import default_engine
from .errors import DecryptionFailed, EncryptionFailed, Error


def encrypt(message, shared_secret, nonce, engine=None):
    """src/encryption.rs:62-74 -> cipher with len(message)+1 scalars."""
    msg = np.ascontiguousarray(message, dtype=np.uint64).reshape(1, -1, 4)
    sec = np.ascontiguousarray(shared_secret, dtype=np.uint64).reshape(1, 2, 4)
    non = np.ascontiguousarray(nonce, dtype=np.uint64).reshape(1, 4)
    eng = engine or default_engine()
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
    eng = engine or default_engine()
    msg, ok = eng.decrypt_batch(cip, sec, non)
    if not ok[0]:
        raise DecryptionFailed()
    return msg[0]


def encrypt_batch(messages, secrets_uv, nonces, engine=None, out=None, async_=False):
    """NEW: n independent encrypt() calls.  (n, L, 4), (n, 2, 4), (n, 4) -> (n, L+1, 4)."""
    eng = engine or default_engine(messages.device.index if hasattr(messages, "is_cuda") else 0)
    return eng.encrypt_batch(messages, secrets_uv, nonces, out=out, async_=async_)


def decrypt_batch(ciphers, secrets_uv, nonces, engine=None, async_=False):
    """NEW: n independent decrypt() calls -> (messages (n, L, 4), ok (n,)); ok[i] == 0 marks the
    items for which the reference returns Error::DecryptionFailed (their message is zeroed)."""
    eng = engine or default_engine(ciphers.device.index if hasattr(ciphers, "is_cuda") else 0)
    return eng.decrypt_batch(ciphers, secrets_uv, nonces, async_=async_)
