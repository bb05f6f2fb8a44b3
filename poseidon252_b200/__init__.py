"""poseidon252_b200 -- H100-native batched Poseidon/Hades engine with the dusk_poseidon API.

Public surface mirrors src/lib.rs:13-31:
    Hash, Domain, Error, HADES_WIDTH, encrypt, decrypt
plus the batch entry points this engine adds:
    Hash.digest_batch, Hash.digest_batch_varlen (inputs of different lengths in one call), finalize_batch /
    digest_batch_mixed (Hash.finalize_batch / Hash.digest_batch_mixed: items of different domains, input and output lengths,
    finalized or truncated, in one call), hash_to_scalar_batch
    (BlsScalar::hash_to_scalar of byte strings of different lengths in one call), hades.permute_batch,
    encrypt_batch, decrypt_batch, encrypt_batch_varlen / decrypt_batch_varlen (messages of different lengths in one call),
    dhke / dhke_batch (JubJub key exchange), encrypt_batch_dhke / decrypt_batch_dhke (shared secret derived on the device),
    fixed_base / fixed_base_batch ([s] B for one base, e.g. public and ephemeral keys), encrypt_batch_ephemeral (the
    sender: ephemeral keys and ciphers in one call), stealth_address / stealth_address_batch and owns /
    stealth_owns_batch (stealth addresses: the sender's note keys and a view key's ownership scan), schnorr_sign /
    schnorr_sign_batch and schnorr_verify / schnorr_verify_batch (Schnorr signatures over JubJub), point_from_bytes /
    points_from_bytes_batch and point_to_bytes / points_to_bytes_batch (JubJub point compression), jubjub_msm
    (multi-scalar multiplication), schnorr_verify_all and schnorr_verify_double_all (all-or-nothing batch verification
    of single- and double-key signatures), nullifier /
    nullifier_batch (Phoenix note nullifiers: which owned notes are spent), schnorr_sign_double /
    schnorr_sign_double_batch, schnorr_verify_double / schnorr_verify_double_batch and note_sign_double_batch (double-key
    Schnorr signatures over G and G', and spending a note under its note secret key), value_commit /
    value_commit_batch, note_create / note_create_batch and note_open / note_open_batch (Phoenix note values: Pedersen
    commitments, creating obfuscated notes and their checked opening), wallet_scan_batch (which of several keys owns each
    note, with the owned notes' nullifiers, checked openings and per-key totals), elgamal_encrypt / elgamal_encrypt_batch,
    elgamal_decrypt / elgamal_decrypt_batch, note_sender_encrypt_batch and note_sender_decrypt /
    note_sender_decrypt_batch (JubJub ElGamal and the encrypted sender of a Phoenix note), merkle4_build, Tree (fixed-height Merkle tree with batched appends / overwrites), SparseTree (fixed-height Merkle tree
    with batched inserts / removals at any position).
All computation runs in hand-written sm_90a CUDA behind the C ABI in include/poseidon252_b200.h.
"""
from . import hades, merkle, scalar
from .encryption import (cipher_offsets, decrypt, decrypt_batch, decrypt_batch_dhke, decrypt_batch_varlen, dhke, dhke_batch,
                         encrypt, encrypt_batch, encrypt_batch_dhke, encrypt_batch_ephemeral, encrypt_batch_varlen,
                         fixed_base, fixed_base_batch, message_offsets, owns, stealth_address, stealth_address_batch,
                         stealth_owns_batch)
from .elgamal import (elgamal_decrypt, elgamal_decrypt_batch, elgamal_encrypt, elgamal_encrypt_batch,
                      note_sender_decrypt, note_sender_decrypt_batch, note_sender_encrypt_batch)
from .engine import Engine, default_engine
from .errors import (DecryptionFailed, EncryptionFailed, EngineError, Error, InvalidIOPattern, InvalidPoint,
                     IOPatternViolation, TooFewInputElements)
from .hash import Domain, Hash, digest_batch_mixed, finalize_batch, hash_to_scalar_batch, pack_bytes, pack_varlen
from .merkle import CompactTree, SparseTree, Tree, merkle4_build, merkle4_level
from .msm import jubjub_msm, schnorr_verify_all, schnorr_verify_double_all
from .notes import note_create, note_create_batch, note_open, note_open_batch, value_commit, value_commit_batch
from .nullifier import nullifier, nullifier_batch
from .points import point_from_bytes, point_to_bytes, points_from_bytes_batch, points_to_bytes_batch
from .schnorr import schnorr_sign, schnorr_sign_batch, schnorr_verify, schnorr_verify_batch
from .schnorr_double import (note_sign_double_batch, schnorr_sign_double, schnorr_sign_double_batch,
                             schnorr_verify_double, schnorr_verify_double_batch)
from .wallet import wallet_scan_batch

HADES_WIDTH = hades.WIDTH

__all__ = ["Hash", "Domain", "Error", "HADES_WIDTH", "encrypt", "decrypt", "encrypt_batch", "decrypt_batch", "pack_varlen",
           "hash_to_scalar_batch", "pack_bytes", "finalize_batch", "digest_batch_mixed",
           "encrypt_batch_varlen", "decrypt_batch_varlen", "cipher_offsets", "message_offsets",
           "dhke", "dhke_batch", "encrypt_batch_dhke", "decrypt_batch_dhke", "fixed_base", "fixed_base_batch",
           "encrypt_batch_ephemeral", "stealth_address", "stealth_address_batch", "owns", "stealth_owns_batch",
           "schnorr_sign", "schnorr_sign_batch", "schnorr_verify", "schnorr_verify_batch",
           "point_from_bytes", "point_to_bytes", "points_from_bytes_batch", "points_to_bytes_batch",
           "jubjub_msm", "schnorr_verify_all", "schnorr_verify_double_all", "nullifier", "nullifier_batch",
           "schnorr_sign_double", "schnorr_sign_double_batch", "schnorr_verify_double", "schnorr_verify_double_batch",
           "note_sign_double_batch", "value_commit", "value_commit_batch", "note_create", "note_create_batch",
           "note_open", "note_open_batch", "wallet_scan_batch", "elgamal_encrypt", "elgamal_encrypt_batch",
           "elgamal_decrypt", "elgamal_decrypt_batch", "note_sender_encrypt_batch", "note_sender_decrypt",
           "note_sender_decrypt_batch",
           "hades", "merkle", "scalar", "Engine", "default_engine", "merkle4_build", "merkle4_level", "Tree", "SparseTree",
           "CompactTree",
           "IOPatternViolation", "InvalidIOPattern", "TooFewInputElements", "EncryptionFailed",
           "DecryptionFailed", "InvalidPoint", "EngineError"]
