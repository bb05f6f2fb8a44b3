"""`Hash` / `Domain` -- host-side mirror of src/hash.rs over the GPU engine.

Same names, argument meaning and error behaviour as the reference; every digest is computed by the
CUDA sponge kernel (a single `Hash::digest` is a batch of one).  New: `Hash.digest_batch` and the other batch entries
below; `Hash.finalize_batch` / `Hash.digest_batch_mixed` take items of any domains, lengths and truncation in one call."""
import ctypes
import enum

import numpy as np

from . import _native
from .engine import _engine_for
from .errors import raise_for_status
from .scalar import P, from_mont


class Domain(enum.IntEnum):
    """src/hash.rs:21-36.  The enum value is the C ABI's p252_domain; `u64(domain)` below is
    `u64::from(Domain)` (src/hash.rs:38-56)."""
    Merkle4 = 0
    Merkle2 = 1
    Encryption = 2
    Other = 3


def domain_separator(domain):
    """u64::from(domain), src/hash.rs:43-55"""
    out = ctypes.c_uint64(0)
    raise_for_status(_native.lib().p252_domain_separator(int(domain), ctypes.byref(out)))
    return int(out.value)


def _calls(pattern):
    """[('absorb'|'squeeze', len), ...] -> u32 call words of the C ABI."""
    return np.array([(0x80000000 | n) if kind == "absorb" else n for kind, n in pattern], dtype=np.uint32)


def tag_input(pattern, domain_sep):
    """dusk-safe tag input bytes for an io-pattern."""
    calls = _calls(pattern)
    buf = (ctypes.c_uint8 * (4 * len(calls) + 16))()
    n = ctypes.c_size_t(len(buf))
    raise_for_status(_native.lib().p252_tag_input(calls.ctypes.data, len(calls), domain_sep, buf, ctypes.byref(n)))
    return bytes(buf[:n.value])


def tag(pattern, domain_sep):
    """Safe::tag of an io-pattern -> (4,) uint64 Montgomery limbs."""
    calls = _calls(pattern)
    out = np.zeros(4, dtype=np.uint64)
    raise_for_status(_native.lib().p252_tag(calls.ctypes.data, len(calls), domain_sep, out.ctypes.data))
    return out


def hash_to_scalar(data: bytes):
    """BlsScalar::hash_to_scalar (src/hades/permutation/scalar.rs:29-31)."""
    out = np.zeros(4, dtype=np.uint64)
    buf = (ctypes.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    raise_for_status(_native.lib().p252_hash_to_scalar(buf, len(data), out.ctypes.data))
    return out


def pack_bytes(messages):
    """A list of byte strings -> (data (sum len_i,) uint8, offsets (n + 1,) uint64, longest len_i), the layout of
    `Engine.hash_to_scalar_batch`.  Pure host work."""
    lens = np.fromiter((len(m) for m in messages), dtype=np.uint64, count=len(messages))
    offsets = np.zeros(len(messages) + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    data = np.frombuffer(b"".join(bytes(m) for m in messages), dtype=np.uint8)
    return data, offsets, int(lens.max()) if len(messages) else 0


def hash_to_scalar_batch(messages, engine=None, max_len=None, out=None, async_=False):
    """NEW batch entry: n x `hash_to_scalar(messages[i])` on the device, one call for byte strings of any lengths.
    messages: a list of `bytes` (packed on the host by `pack_bytes`), or a `(data, offsets)` pair as taken by
    `Engine.hash_to_scalar_batch` (numpy arrays, or CUDA tensors).  Returns (n, 4) Montgomery limbs in input order."""
    if isinstance(messages, tuple):
        data, offsets = messages
    else:
        data, offsets, longest = pack_bytes(messages)
        max_len = longest if max_len is None else max_len
    eng = _engine_for(engine, data)
    return eng.hash_to_scalar_batch(data, offsets, max_len=max_len, out=out, async_=async_)


def io_pattern(domain, chunk_lens, output_len):
    """src/hash.rs:62-85: one Absorb per update() chunk + Squeeze(output_len); Merkle arity check."""
    from .errors import IOPatternViolation
    total = sum(chunk_lens)
    if domain == Domain.Merkle2 and (total != 2 or output_len != 1):
        raise IOPatternViolation()
    if domain == Domain.Merkle4 and (total != 4 or output_len != 1):
        raise IOPatternViolation()
    return [("absorb", n) for n in chunk_lens] + [("squeeze", output_len)]


def pack_varlen(inputs):
    """A list of (k_i, 4) scalar arrays -> (data (sum k_i, 4) uint64, offsets (n + 1,) uint64, longest k_i), the
    layout of `Engine.hash_batch_varlen`.  Pure host work."""
    arrs = [np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4) for a in inputs]
    lens = np.array([a.shape[0] for a in arrs], dtype=np.uint64)
    offsets = np.zeros(len(arrs) + 1, dtype=np.uint64)
    np.cumsum(lens, out=offsets[1:])
    data = np.concatenate(arrs, axis=0) if arrs else np.zeros((0, 4), dtype=np.uint64)
    return data, offsets, int(lens.max()) if len(arrs) else 0


class Hash:
    """src/hash.rs:92-210.  Scalars are (k, 4) uint64 arrays of BlsScalar.0 limbs."""

    def __init__(self, domain, engine=None):
        self.domain = Domain(domain)
        self.input = []
        self._output_len = 1
        self._engine = engine

    def output_len(self, output_len):
        """src/hash.rs:111-115: only honoured for Domain::Other and > 0."""
        if self.domain == Domain.Other and output_len > 0:
            self._output_len = int(output_len)

    def update(self, chunk):
        """src/hash.rs:118-120"""
        self.input.append(np.ascontiguousarray(chunk, dtype=np.uint64).reshape(-1, 4))

    def finalize(self):
        """src/hash.rs:128-155.  Raises IOPatternViolation / InvalidIOPattern where the reference
        panics ("io-pattern should be valid", src/hash.rs:133-137)."""
        lens = [int(c.shape[0]) for c in self.input]
        pattern = io_pattern(self.domain, lens, self._output_len)
        t = tag(pattern, domain_separator(self.domain))
        eng = _engine_for(self._engine)
        data = np.concatenate(self.input, axis=0) if self.input else np.zeros((0, 4), dtype=np.uint64)
        out = eng.digest_batch_with_tag(t, data.reshape(1, -1, 4), self._output_len)
        return out[0]

    def finalize_truncated(self):
        """src/hash.rs:164-183: canonical value & (2^250 - 1); returns the (out_len, 4) raw u64 limbs that the
        reference hands to JubJubScalar::from_raw (computed on the device, see digest_truncated_batch)."""
        lens = [int(c.shape[0]) for c in self.input]
        if len(lens) != 1:
            # chunked updates only change the tag; use the generic path + host post-step
            mask = (1 << 250) - 1
            vals = [int(v) & mask for v in from_mont(self.finalize())]
            return np.array([[(v >> (64 * k)) & ((1 << 64) - 1) for k in range(4)] for v in vals], dtype=np.uint64)
        io_pattern(self.domain, lens, self._output_len)
        eng = _engine_for(self._engine)
        return eng.hash_batch_truncated(self.domain, self.input[0].reshape(1, -1, 4), self._output_len)[0]

    @staticmethod
    def finalize_batch(hashes, truncated=False, engine=None):
        """NEW batch entry: [h.finalize() or h.finalize_truncated() for h in hashes] in one device call
        (Engine.hash_batch_mixed), whatever their domains, update() chunks and output lengths (inputs and outputs of up to
        VARLEN_MAX_LEN scalars each).  truncated: one bool for all, or one per hash.  Raises what Hash.finalize would raise for the lowest-index invalid hash (a Merkle arity
        violation, no input or a zero-length update() chunk) before any engine is touched.  engine: None takes the first
        hash's engine, then the default one."""
        from .errors import InvalidIOPattern
        hashes = list(hashes)
        if isinstance(truncated, (bool, np.bool_)):
            truncated = [truncated] * len(hashes)
        trunc = [bool(t) for t in truncated]
        if len(trunc) != len(hashes):
            raise ValueError("truncated must be one bool or one per hash")
        for h in hashes:
            lens = [int(c.shape[0]) for c in h.input]
            io_pattern(h.domain, lens, h._output_len)
            if not lens or 0 in lens:
                raise InvalidIOPattern()
        if not hashes:
            return []
        mode = np.array([int(h.domain) | (_native.MIXED_TRUNCATED if t else 0) for h, t in zip(hashes, trunc)],
                        dtype=np.uint8)
        lens = np.array([sum(int(c.shape[0]) for c in h.input) for h in hashes], dtype=np.uint64)
        out_lens = np.array([h._output_len for h in hashes], dtype=np.uint64)
        offsets = np.zeros(len(hashes) + 1, dtype=np.uint64)
        out_offsets = np.zeros(len(hashes) + 1, dtype=np.uint64)
        np.cumsum(lens, out=offsets[1:])
        np.cumsum(out_lens, out=out_offsets[1:])
        data = np.concatenate([c for h in hashes for c in h.input], axis=0)
        eng = _engine_for(engine if engine is not None else hashes[0]._engine)
        out = eng.hash_batch_mixed(mode, data, offsets, out_offsets, int(lens.max()), int(out_lens.max()))
        return [out[out_offsets[i]:out_offsets[i + 1]] for i in range(len(hashes))]

    @staticmethod
    def digest_batch_mixed(mode, data, offsets, out_offsets, engine=None, max_len=None, max_out_len=None, out=None,
                           async_=False):
        """NEW batch entry: Engine.hash_batch_mixed over CSR arrays (numpy, or CUDA tensors): item i is
        Hash::new(mode[i] & 3) over data[offsets[i]:offsets[i+1]] with out_offsets[i+1] - out_offsets[i] outputs, truncated where mode[i] &
        MIXED_TRUNCATED.  Output lengths are taken as given, for every domain.  Returns the (n_out, 4) output rows."""
        eng = _engine_for(engine, data)
        return eng.hash_batch_mixed(mode, data, offsets, out_offsets, max_len=max_len, max_out_len=max_out_len, out=out,
                                    async_=async_)

    @staticmethod
    def digest(domain, data, engine=None):
        """src/hash.rs:191-195"""
        h = Hash(domain, engine)
        h.update(data)
        return h.finalize()

    @staticmethod
    def digest_truncated(domain, data, engine=None):
        """src/hash.rs:203-210"""
        h = Hash(domain, engine)
        h.update(data)
        return h.finalize_truncated()

    @staticmethod
    def digest_truncated_batch(domain, inputs, output_len=1, engine=None, out=None, async_=False):
        """NEW batch entry: n x Hash::digest_truncated -> (n, out_len, 4) raw limbs (< 2^250)."""
        domain = Domain(domain)
        ol = int(output_len) if (domain == Domain.Other and output_len > 0) else 1
        eng = _engine_for(engine, inputs)
        return eng.hash_batch_truncated(domain, inputs, ol, out=out, async_=async_)

    @staticmethod
    def digest_batch_varlen(domain, inputs, output_len=1, engine=None, max_len=None, out=None, async_=False):
        """NEW batch entry: n independent `Hash::digest(domain, inputs[i])` over inputs of different lengths, one call.
        inputs: a list of (k_i, 4) host arrays (packed by `pack_varlen`), or a `(data, offsets)` pair as taken by
        `Engine.hash_batch_varlen` (numpy or CUDA tensors).  Returns (n, out_len, 4) in input order."""
        domain = Domain(domain)
        ol = int(output_len) if (domain == Domain.Other and output_len > 0) else 1
        if isinstance(inputs, tuple):
            data, offsets = inputs
        else:
            data, offsets, longest = pack_varlen(inputs)
            max_len = max(longest, 1) if max_len is None else max_len
        eng = _engine_for(engine, data)
        return eng.hash_batch_varlen(domain, data, offsets, ol, max_len=max_len, out=out, async_=async_)

    @staticmethod
    def digest_batch(domain, inputs, output_len=1, engine=None, out=None, async_=False):
        """NEW batch entry: n independent `Hash::digest(domain, inputs[i])` (with
        `output_len(output_len)` applied under the reference's rule).  inputs: (n, in_len, 4) numpy
        array (host) or torch CUDA tensor (device).  Returns (n, out_len, 4)."""
        domain = Domain(domain)
        ol = int(output_len) if (domain == Domain.Other and output_len > 0) else 1
        eng = _engine_for(engine, inputs)
        return eng.hash_batch(domain, inputs, ol, out=out, async_=async_)


finalize_batch = Hash.finalize_batch
digest_batch_mixed = Hash.digest_batch_mixed
