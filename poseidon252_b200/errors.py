"""Error variants of the batch engine -- mirror of dusk_poseidon::Error
(src/error.rs:11-32) plus engine failures."""


class Error(Exception):
    """Base of all dusk_poseidon::Error variants."""
    code = None


class IOPatternViolation(Error):
    """src/error.rs:14 -- a call that does not fit the io-pattern (e.g. Merkle4 with != 4 inputs,
    src/hash.rs:71-76)."""
    code = 1


class InvalidIOPattern(Error):
    """src/error.rs:17"""
    code = 2


class TooFewInputElements(Error):
    """src/error.rs:20"""
    code = 3


class EncryptionFailed(Error):
    """src/error.rs:24"""
    code = 4


class DecryptionFailed(Error):
    """src/error.rs:28 -- wrong secret / nonce or tampered cipher (tests/encryption.rs:48-115)."""
    code = 5


class InvalidPoint(Error):
    """src/error.rs:31"""
    code = 6


class EngineError(RuntimeError):
    """CUDA / NCCL / argument failures of the engine (negative p252_status codes)."""

    def __init__(self, code, message):
        super().__init__("p252 status %d: %s" % (code, message))
        self.code = code


_BY_CODE = {c.code: c for c in (IOPatternViolation, InvalidIOPattern, TooFewInputElements, EncryptionFailed,
                                DecryptionFailed, InvalidPoint)}


def raise_for_status(code, lib=None, ctx=None):
    if code == 0:
        return
    if code in _BY_CODE:
        raise _BY_CODE[code]()
    msg = lib.p252_strerror(code).decode() if lib is not None else "engine error"
    if lib is not None and ctx:
        detail = lib.p252_last_error(ctx).decode()
        if detail:
            msg += " (" + detail + ")"
    raise EngineError(code, msg)
