"""CPU ORACLE (test infrastructure, NOT product code) -- Python big-int restatement of the
dusk-poseidon hot path: Hades permutation + SAFE sponge + Hash / encrypt / decrypt.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
The product path (poseidon252_b200/) never imports it and has no CPU fallback.

Every function cites the reference file:line (relative to the reference repository's root) it restates.
All values here are *canonical* integers in [0, p); the reference's in-memory form
(`BlsScalar.0`, 4 x u64 little-endian limbs, Montgomery form x*R mod p) is produced by
`to_mont_limbs` / consumed by `from_mont_limbs`.

PINNING STATUS
  * pinned (absolute): field add/mul, constant interpretation, round schedule, sponge
    absorb/permute/squeeze schedule -- by the 6 known-answer vectors of src/hades.rs:128-162
    (tests/test_oracle.py reproduces all of them with this file).
  * parity unpinned: `hash_to_scalar` (dusk-bls12_381 0.14, BLAKE2b-512 -> from_bytes_wide) and
    the tag-input byte encoding + encrypt/decrypt internals of dusk-safe 0.3. Neither crate is
    vendored in the reference and no reference test fixes their absolute output; they are
    restated from the crates' published algorithm (SAFE paper, eprint 2023/522 sec. 2.3) and
    anchored on the reference's call sites and property tests (README doctest,
    tests/encryption.rs). The device never computes a tag: it is a per-batch input.
"""
from __future__ import annotations

import hashlib
from typing import Iterable, List, Sequence

# ----------------------------------------------------------------------------------------------
# Field: BLS12-381 scalar field (src/hades.rs:12, src/hades/permutation.rs:13-14)
# ----------------------------------------------------------------------------------------------
P = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
R = (1 << 256) % P          # Montgomery radix of dusk_bls12_381::BlsScalar (4 x u64 limbs)
R_INV = pow(R, -1, P)
MASK64 = (1 << 64) - 1

WIDTH = 5                   # src/hades.rs:34
FULL_ROUNDS = 8             # src/hades.rs:29
PARTIAL_ROUNDS = 60         # src/hades.rs:31
ROUNDS = FULL_ROUNDS + PARTIAL_ROUNDS   # src/hades/round_constants.rs:18
RATE = WIDTH - 1            # dusk-safe: capacity = 1 element (state[0] holds the tag)


def to_mont_limbs(x: int) -> List[int]:
    """canonical integer -> BlsScalar.0 (4 x u64 LE limbs of x*R mod p)."""
    v = (x % P) * R % P
    return [(v >> (64 * i)) & MASK64 for i in range(4)]


def from_mont_limbs(limbs: Sequence[int]) -> int:
    """BlsScalar.0 -> canonical integer."""
    v = sum(int(l) << (64 * i) for i, l in enumerate(limbs))
    return v * R_INV % P


def from_bytes_wide(b: bytes) -> int:
    """dusk_bls12_381::BlsScalar::from_bytes_wide: 64 LE bytes -> integer mod p
    (used at assets/HOWTO.md:36 and by hash_to_scalar, src/hades/permutation/scalar.rs:30)."""
    assert len(b) == 64
    return int.from_bytes(b, "little") % P


def from_le_hex(s: str) -> int:
    """dusk_bytes ParseHexStr on BlsScalar: 32 LE bytes, canonical (src/hades.rs:94-105,131)."""
    v = int.from_bytes(bytes.fromhex(s), "little")
    assert v < P
    return v


def debug_hex(x: int) -> str:
    """`{:?}` of BlsScalar: 0x + big-endian hex of the canonical value (src/hades.rs:134-136)."""
    return "0x%064x" % x


# ----------------------------------------------------------------------------------------------
# Constants, regenerated from the published recipe (assets/HOWTO.md) -- not copied from the .bin
# ----------------------------------------------------------------------------------------------
def gen_arc_file_ints() -> List[int]:
    """The 340 integers stored in assets/arc.bin.

    assets/HOWTO.md:23-41: h_0 = SHA512("poseidon-for-plonk"), h_k = SHA512(h_{k-1});
    c_k = from_bytes_wide(h_k) + c_{k-1}, c_{-1} = 1.  HOWTO.md:44-52 dumps `internal_repr()`,
    i.e. the Montgomery limbs c_k*R mod p.  src/hades/round_constants.rs:40-47 reads those limbs
    back with `BlsScalar::from_raw`, i.e. as a *canonical* integer.  So the effective round
    constant is the integer c_k*R mod p."""
    out = []
    prev = 1
    data = b"poseidon-for-plonk"
    for _ in range(ROUNDS * WIDTH):
        data = hashlib.sha512(data).digest()
        c = (from_bytes_wide(data) + prev) % P
        prev = c
        out.append(c * R % P)
    return out


def gen_mds_file_ints() -> List[List[int]]:
    """The 25 integers stored in assets/mds.bin (row-major).

    assets/HOWTO.md:70-97: Cauchy matrix 1/(x_i + y_j), x_i = i, y_j = j + 5, dumped with
    `internal_repr()` (HOWTO.md:100-108) and read with `from_raw` (src/hades/mds_matrix.rs:25-32):
    effective entry = R * (i + j + 5)^-1 mod p."""
    return [[pow(i + j + WIDTH, -1, P) * R % P for j in range(WIDTH)] for i in range(WIDTH)]


_ARC_FLAT = gen_arc_file_ints()
# ROUND_CONSTANTS[round][i], file index round*5+i  (src/hades/round_constants.rs:26-54)
ROUND_CONSTANTS = [_ARC_FLAT[r * WIDTH:(r + 1) * WIDTH] for r in range(ROUNDS)]
# MDS_MATRIX[i][j]  (src/hades/mds_matrix.rs:17-39)
MDS_MATRIX = gen_mds_file_ints()


def arc_bin_bytes() -> bytes:
    """Byte image of assets/arc.bin (used by tests to compare with the reference file)."""
    return b"".join(v.to_bytes(32, "little") for v in _ARC_FLAT)


def mds_bin_bytes() -> bytes:
    """Byte image of assets/mds.bin."""
    return b"".join(v.to_bytes(32, "little") for row in MDS_MATRIX for v in row)


# ----------------------------------------------------------------------------------------------
# Hades permutation (src/hades/permutation.rs + src/hades/permutation/scalar.rs)
# ----------------------------------------------------------------------------------------------
def add_round_constants(rnd: int, state: List[int]) -> None:
    """src/hades/permutation/scalar.rs:39-48"""
    for i in range(WIDTH):
        state[i] = (state[i] + ROUND_CONSTANTS[rnd][i]) % P


def quintic_s_box(v: int) -> int:
    """src/hades/permutation/scalar.rs:50-52: value.square().square() * value"""
    v2 = v * v % P
    v4 = v2 * v2 % P
    return v4 * v % P


def mul_matrix(state: List[int]) -> None:
    """src/hades/permutation/scalar.rs:54-64: result[k] += MDS[k][j] * state[j]"""
    result = [0] * WIDTH
    for j, value in enumerate(state):
        for k in range(WIDTH):
            result[k] = (result[k] + MDS_MATRIX[k][j] * value) % P
    state[:] = result


def apply_partial_round(rnd: int, state: List[int]) -> None:
    """src/hades/permutation.rs:63-72"""
    add_round_constants(rnd, state)
    state[WIDTH - 1] = quintic_s_box(state[WIDTH - 1])
    mul_matrix(state)


def apply_full_round(rnd: int, state: List[int]) -> None:
    """src/hades/permutation.rs:83-92"""
    add_round_constants(rnd, state)
    for i in range(WIDTH):
        state[i] = quintic_s_box(state[i])
    mul_matrix(state)


def perm(state: Sequence[int]) -> List[int]:
    """src/hades/permutation.rs:105-123 (returns a new list; the reference permutes in place)."""
    s = [x % P for x in state]
    assert len(s) == WIDTH
    for rnd in range(FULL_ROUNDS // 2):
        apply_full_round(rnd, s)
    for rnd in range(PARTIAL_ROUNDS):
        apply_partial_round(rnd + FULL_ROUNDS // 2, s)
    for rnd in range(FULL_ROUNDS // 2):
        apply_full_round(rnd + FULL_ROUNDS // 2 + PARTIAL_ROUNDS, s)
    return s


# ----------------------------------------------------------------------------------------------
# SAFE sponge (external crate dusk-safe 0.3, Cargo.toml:18; driven at src/hash.rs:128-155 and
# src/hades.rs:107-125).  Scheduling pinned by the KATs; tag encoding parity-unpinned.
# ----------------------------------------------------------------------------------------------
class Error(Exception):
    """src/error.rs:11-32 -- one subclass per variant."""


class IOPatternViolation(Error):
    pass


class InvalidIOPattern(Error):
    pass


class TooFewInputElements(Error):
    pass


class EncryptionFailed(Error):
    pass


class DecryptionFailed(Error):
    pass


ABSORB, SQUEEZE = "absorb", "squeeze"


def Absorb(n: int):
    return (ABSORB, n)


def Squeeze(n: int):
    return (SQUEEZE, n)


def validate_io_pattern(pattern: Sequence[tuple]) -> None:
    """dusk-safe: a pattern must start with an absorb, end with a squeeze and contain no
    zero-length call."""
    if not pattern or pattern[0][0] != ABSORB or pattern[-1][0] != SQUEEZE:
        raise InvalidIOPattern()
    if any(n == 0 for _, n in pattern):
        raise InvalidIOPattern()


def tag_input(pattern: Sequence[tuple], domain_sep: int) -> bytes:
    """dusk-safe tag input (SAFE paper 2.3): aggregate consecutive calls of the same kind, encode
    each as a big-endian u32 (absorb: MSB set), then append the u64 domain separator big-endian.
    PARITY UNPINNED (see module header); consistent with the README doctest (README.md:40-47):
    update(x[..3]); update(x[3..]) must give the digest of update(x)."""
    validate_io_pattern(pattern)
    words: List[int] = []
    prev_kind = None
    for kind, n in pattern:
        if kind == prev_kind:
            words[-1] += n
        else:
            words.append((0x80000000 + n) if kind == ABSORB else n)
        prev_kind = kind
    out = b"".join((w & 0xFFFFFFFF).to_bytes(4, "big") for w in words)
    return out + (domain_sep & MASK64).to_bytes(8, "big")


def hash_to_scalar(data: bytes) -> int:
    """dusk_bls12_381::BlsScalar::hash_to_scalar (called at src/hades/permutation/scalar.rs:30):
    BLAKE2b-512 of the bytes, digest read as a 512-bit LE integer and reduced mod p.
    PARITY UNPINNED (see module header)."""
    return from_bytes_wide(hashlib.blake2b(data, digest_size=64).digest())


class ScalarPermutation:
    """src/hades/permutation/scalar.rs:15-36,67-80 (Safe + Encryption impls)."""

    def permute(self, state: List[int]) -> None:
        state[:] = perm(state)

    def tag(self, data: bytes) -> int:
        return hash_to_scalar(data)

    def add(self, right: int, left: int) -> int:
        return (right + left) % P

    def subtract(self, minuend: int, subtrahend: int) -> int:
        return (minuend - subtrahend) % P

    def is_equal(self, lhs: int, rhs: int) -> bool:
        return lhs % P == rhs % P


class ZeroTagPermutation(ScalarPermutation):
    """The `Test` Safe impl of the KAT: tag == 0 (src/hades.rs:67-92)."""

    def tag(self, data: bytes) -> int:
        return 0


class Sponge:
    """dusk_safe::Sponge<S, BlsScalar, 5>: state[0] = tag (capacity), state[1..5] = rate."""

    def __init__(self, safe, pattern: Sequence[tuple], domain_sep: int):
        pattern = list(pattern)
        validate_io_pattern(pattern)
        self.safe = safe
        self.pattern = pattern
        self.state = [0] * WIDTH
        self.state[0] = safe.tag(tag_input(pattern, domain_sep))
        self.pos_absorb = 0
        self.pos_squeeze = 0
        self.io_count = 0
        self.output: List[int] = []

    def absorb(self, n: int, data: Sequence[int]) -> None:
        if len(data) < n:
            raise TooFewInputElements()
        if self.io_count >= len(self.pattern) or self.pattern[self.io_count] != (ABSORB, n):
            raise IOPatternViolation()
        for e in list(data)[:n]:
            if self.pos_absorb == RATE:
                self.safe.permute(self.state)
                self.pos_absorb = 0
            pos = self.pos_absorb + 1
            self.state[pos] = self.safe.add(self.state[pos], e)
            self.pos_absorb += 1
        self.pos_squeeze = RATE          # force a permutation before the next squeeze
        self.io_count += 1

    def squeeze(self, n: int) -> None:
        if self.io_count >= len(self.pattern) or self.pattern[self.io_count] != (SQUEEZE, n):
            raise IOPatternViolation()
        for _ in range(n):
            if self.pos_squeeze == RATE:
                self.safe.permute(self.state)
                self.pos_squeeze = 0
                self.pos_absorb = 0
            self.output.append(self.state[self.pos_squeeze + 1])
            self.pos_squeeze += 1
        self.io_count += 1

    def finish(self) -> List[int]:
        if self.io_count != len(self.pattern):
            raise IOPatternViolation()
        return list(self.output)


# ----------------------------------------------------------------------------------------------
# Hash / Domain (src/hash.rs)
# ----------------------------------------------------------------------------------------------
class Domain:
    """src/hash.rs:21-56 -- value = u64::from(domain)."""
    Merkle4 = 0x0000_0000_0000_000F
    Merkle2 = 0x0000_0000_0000_0003
    Encryption = 0x0000_0001_0000_0000
    Other = 0x0000_0000_0000_0000


def io_pattern(domain: int, chunks: Sequence[Sequence[int]], output_len: int) -> List[tuple]:
    """src/hash.rs:62-85"""
    input_len = sum(len(c) for c in chunks)
    if domain == Domain.Merkle2 and (input_len != 2 or output_len != 1):
        raise IOPatternViolation()
    if domain == Domain.Merkle4 and (input_len != 4 or output_len != 1):
        raise IOPatternViolation()
    pat = [Absorb(len(c)) for c in chunks]
    pat.append(Squeeze(output_len))
    return pat


class Hash:
    """src/hash.rs:92-210"""

    def __init__(self, domain: int):
        self.domain = domain
        self.input: List[Sequence[int]] = []
        self._output_len = 1

    def output_len(self, n: int) -> None:
        """src/hash.rs:111-115"""
        if self.domain == Domain.Other and n > 0:
            self._output_len = n

    def update(self, chunk: Sequence[int]) -> None:
        """src/hash.rs:118-120"""
        self.input.append(list(chunk))

    def finalize(self) -> List[int]:
        """src/hash.rs:128-155 (the reference panics where this raises)."""
        sponge = Sponge(ScalarPermutation(), io_pattern(self.domain, self.input, self._output_len),
                        self.domain)
        for chunk in self.input:
            sponge.absorb(len(chunk), chunk)
        sponge.squeeze(self._output_len)
        return sponge.finish()

    def finalize_truncated(self) -> List[int]:
        """src/hash.rs:164-183: canonical value & (2^250 - 1) -> JubJubScalar."""
        return [v & ((1 << 250) - 1) for v in self.finalize()]

    @staticmethod
    def digest(domain: int, data: Sequence[int]) -> List[int]:
        """src/hash.rs:191-195"""
        h = Hash(domain)
        h.update(data)
        return h.finalize()

    @staticmethod
    def digest_truncated(domain: int, data: Sequence[int]) -> List[int]:
        """src/hash.rs:203-210"""
        h = Hash(domain)
        h.update(data)
        return h.finalize_truncated()


def kat_poseidon_hash(inputs: Sequence[int]) -> int:
    """create_poseidon_hash of the reference KAT: tag 0, pattern [Absorb(n), Absorb(1),
    Squeeze(1)], padding BlsScalar::one() (src/hades.rs:107-125)."""
    sponge = Sponge(ZeroTagPermutation(), [Absorb(len(inputs)), Absorb(1), Squeeze(1)], 0)
    sponge.absorb(len(inputs), inputs)
    sponge.absorb(1, [1])
    sponge.squeeze(1)
    return sponge.finish()[0]


# ----------------------------------------------------------------------------------------------
# Encryption (src/encryption.rs -> dusk_safe::{encrypt, decrypt}; parity-unpinned internals)
# ----------------------------------------------------------------------------------------------
def _prepare_sponge(message_len: int, shared_secret: Sequence[int], nonce: int) -> Sponge:
    pat = [Absorb(2), Absorb(1), Squeeze(message_len), Absorb(message_len), Squeeze(1)]
    sponge = Sponge(ScalarPermutation(), pat, Domain.Encryption)
    sponge.absorb(2, list(shared_secret))
    sponge.absorb(1, [nonce])
    sponge.squeeze(message_len)
    return sponge


def encrypt(message: Sequence[int], shared_secret: Sequence[int], nonce: int) -> List[int]:
    """src/encryption.rs:62-74.  shared_secret = (u, v) coordinates of the JubJubAffine point
    (src/encryption.rs:71); cipher has len(message)+1 elements (src/encryption.rs:61)."""
    message = list(message)
    L = len(message)
    try:
        sponge = _prepare_sponge(L, shared_secret, nonce)
        sponge.absorb(L, message)
        sponge.squeeze(1)
        out = sponge.finish()
    except Error as e:
        raise EncryptionFailed() from e
    safe = sponge.safe
    return [safe.add(message[i], out[i]) for i in range(L)] + [out[L]]


def decrypt(cipher: Sequence[int], shared_secret: Sequence[int], nonce: int) -> List[int]:
    """src/encryption.rs:83-95; wrong secret / nonce / tampering -> DecryptionFailed
    (tests/encryption.rs:48-115)."""
    cipher = list(cipher)
    L = len(cipher) - 1
    try:
        sponge = _prepare_sponge(L, shared_secret, nonce)
        safe = sponge.safe
        message = [safe.subtract(cipher[i], sponge.output[i]) for i in range(L)]
        sponge.absorb(L, message)
        sponge.squeeze(1)
        out = sponge.finish()
    except Error as e:
        raise DecryptionFailed() from e
    if not safe.is_equal(out[L], cipher[L]):
        raise DecryptionFailed()
    return message


# ----------------------------------------------------------------------------------------------
# Reference known-answer vectors (src/hades.rs:94-105 inputs, :134-162 outputs)
# ----------------------------------------------------------------------------------------------
KAT_INPUTS_LE_HEX = [
    "bb67ed265bf1db490ded2e1ede55c0d14c55521509dc73f9c354e98ab76c9625",
    "7e74220084d75e10c89e9435d47bb5b8075991b2e29be3b84421dac3b1ee6007",
    "5ce5481a4d78cca03498f72761da1b9f1d2aa8fb300be39f0e4fe2534f9d4308",
    "b1e710e3c4a8c35154b0ce4e4f4af6f498ebd79f8e7cdf3150372c7501be250b",
    "33c9e2025f86b5d82149f1ab8e20a168fc3d99d09b48cbce0286db8752cc3306",
    "e98206bfdce791e4e5144079b997d4fc25006194b35655f0e48490b26e24ea35",
    "86d2a95cc552de8d5bb20bd4a407fee5ffdc314e93dfe6b2dc792bc71fd8cc2d",
    "4edd8307ce28a8c70963d20a7bc28df1e1720bbbc93878a18bd07fad7d51fa15",
    "eabc7a296704a68aa01f95adc85f6dd758b175745336d8fc795a17984024b21e",
    "cfc108673c93df305e31c283b9c767b7097ae4e174a223e0c24b15a67b701a3a",
]
KAT_EXPECTED = {
    3: "0x26abf2d0476f154e69bf19740092fe36265680c294462b8e759ad73a99567dd5",
    4: "0x1cc40219c7ec92919d6db7a41cd41953333a2ed544606daca182e4eaa6c7db2d",
    5: "0x707c98a0e9a6e4832ac33ee08811bce122017a58dbbbf66a2f6fcdc69d45462d",
    6: "0x26905a794d3d2fb0c3ed2276abc696c27a5bfdea7f106e596cbeedd86891c461",
    8: "0x1b98a2c5f1fe54d21b5ce9bf0dcc99ea8784a64f3c544fa06d3f73569741006e",
    10: "0x211b7ea21c9afca93dabdfbda8b2d5275b2dd802fed87bb431e98557c61667d2",
}


def kat_inputs() -> List[int]:
    return [from_le_hex(s) for s in KAT_INPUTS_LE_HEX]


def self_check() -> None:
    ins = kat_inputs()
    for n, want in KAT_EXPECTED.items():
        got = debug_hex(kat_poseidon_hash(ins[:n]))
        assert got == want, (n, got, want)


if __name__ == "__main__":
    self_check()
    print("oracle: all 6 reference KATs (src/hades.rs:134-162) reproduced")
