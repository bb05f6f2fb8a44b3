"""Phoenix wallet scans over the GPU engine: which of several keys owns each note, and for the owned notes their
nullifier, checked opening and per-key totals, in one call.

    keys (a_j, b_j):  B_j = [b_j] G
    owner(i)        = the smallest j with note_pk_i == [hash([a_j] R_i)] G + B_j   (stealth_owns), -1 if none
    nullifier(i)    = nullifier(a_j, b_j; R_i, pos_i)                                (nullifier_batch, under G')
    opening(i)      = note_open(a_j; R_i, nonce_i, cipher_i, C_i)                     (note_open_batch: value, blinder)
    totals(j)       = (value_lo, value_hi, n_owned, n_opened) over the notes key j owns

hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0], as in the stealth calls.  [a_j] R_i is computed once per
(note, key) pair, and the nullifier and opening only for owned notes.  The keys, the shared points and the plaintexts
never leave the device; the call returns value and blinder, the spend proof's witnesses."""
from .engine import _engine_for


def wallet_scan_batch(a, b, R, note_pk, pos, nonce, cipher, commitment, base, base_p, engine=None, async_=False):
    """NEW: scan n notes with k keys.  a and b (k, 4) p252_jscalar rows (1 <= k <= 256), R and note_pk (n, 2, 4), pos (n,)
    uint64 (a CUDA int64 tensor for device buffers), nonce (n, 4), cipher (n, 3, 4), commitment (n, 2, 4), base (G) and
    base_p (G') (2, 4) -> (owner (n,) int32, nullifier (n, 4), value (n,), blinder (n, 4), opened (n,) uint8,
    key_totals (k, 4)).  owner == -1 marks a note no key owns (and an invalid note); its rows are zeroed.  An owned note
    with opened == 0 cannot be spent and is not in the totals.  A wallet's balance under key j is
    key_totals[j, 0] + 2^64 key_totals[j, 1]."""
    eng = _engine_for(engine, R)
    return eng.wallet_scan_batch(a, b, R, note_pk, pos, nonce, cipher, commitment, base, base_p, async_=async_)
