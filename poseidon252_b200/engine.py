"""Engine: one CUDA device + stream behind the C ABI (include/poseidon252_b200.h).

Buffers are either numpy uint64 arrays (HOST: the library stages H2D/D2H in overlapped chunks) or
torch CUDA tensors of dtype int64/uint64 (DEVICE: zero-copy, enqueued on the engine's stream).
There is no CPU fallback: constructing an Engine without an H100 (sm_90) GPU raises EngineError."""
import ctypes

import numpy as np

from . import _native
from .errors import EngineError, raise_for_status

_DEFAULT = {}


def _is_torch(x):
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _random_weights(n, like):
    """n fresh nonzero 128-bit weights from `secrets` as (n, 4) p252_jscalar rows, in the memory space of `like`."""
    import secrets
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, :2] = np.frombuffer(secrets.token_bytes(16 * n), dtype=np.uint64).reshape(n, 2)
    for i in np.flatnonzero((w[:, 0] == 0) & (w[:, 1] == 0)):
        w[i, 0] = 1 + secrets.randbelow((1 << 64) - 1)
    if _is_torch(like):
        import torch
        return torch.from_numpy(w.view(np.int64)).to(like.device)
    return w


class Engine:
    def __init__(self, device=0, stream=None):
        """stream: None -> the engine creates its own non-blocking stream; an int -> an existing
        cudaStream_t handle (e.g. torch.cuda.current_stream().cuda_stream; 0 means the legacy
        default stream)."""
        self._lib = _native.lib()
        self._ctx = ctypes.c_void_p()
        self.device = int(device)
        if stream is None:
            rc = self._lib.p252_create(self.device, ctypes.byref(self._ctx))
        else:
            handle = int(stream) or 1          # 0 -> cudaStreamLegacy
            rc = self._lib.p252_create_on_stream(self.device, ctypes.c_void_p(handle), ctypes.byref(self._ctx))
        if rc != 0:
            self._ctx = ctypes.c_void_p()
            raise EngineError(rc, self._lib.p252_strerror(rc).decode())
        self._dist = False
        self._stream_handle = None if stream is None else int(stream)
        # name -> the c_size_t the last call that publishes that count was given (read by the last_*() methods)
        self._counters = {}
        # what an async device call left for the stream to use after it returned: a host function writes through its
        # counters, the device reads the temporaries made for it; all of it stays alive until sync() or close()
        self._kept_until_sync = []

    def _fence_torch(self):
        """Device tensors are produced on torch's current stream; unless the engine was bound to that
        very stream, wait for it before enqueueing on ours (cross-stream ordering)."""
        import torch
        cur = torch.cuda.current_stream(self.device)
        if self._stream_handle is None or int(cur.cuda_stream) != self._stream_handle:
            cur.synchronize()

    # -- lifetime ---------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self._lib.p252_destroy(self._ctx)          # drains the stream: pending counter writes are done
            self._ctx = ctypes.c_void_p()
        self._kept_until_sync = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def sync(self):
        self._check(self._lib.p252_sync(self._ctx))
        self._kept_until_sync = []

    def _keep_until_sync(self, obj):
        """Keep `obj` alive until sync() or close(): the stream still reads or writes it after the call returned."""
        self._kept_until_sync.append(obj)

    def _counter(self, name, flags):
        """A fresh c_size_t for the count the library publishes as `name`, installed before the call so that a call
        that raises leaves 0 behind; kept alive until sync() when the call is asynchronous."""
        c = self._counters[name] = ctypes.c_size_t(0)
        if flags & _native.ASYNC:
            self._keep_until_sync(c)
        return c

    def _last(self, name):
        """The count `name` of the last call that publishes it; 0 before any such call."""
        return int(self._counters[name].value) if name in self._counters else 0

    @property
    def launch_count(self):
        return int(self._lib.p252_launch_count(self._ctx))

    def _check(self, rc):
        raise_for_status(rc, self._lib, self._ctx)

    # -- buffer plumbing --------------------------------------------------------------------------
    def _in(self, x, shape_tail):
        """-> (pointer, leading-shape, flags, keepalive)"""
        if _is_torch(x):
            if not x.is_cuda or x.device.index != self.device:
                raise EngineError(-1, "tensor is not on cuda:%d" % self.device)
            if str(x.dtype) not in ("torch.int64", "torch.uint64") or not x.is_contiguous():
                raise EngineError(-1, "device buffers must be contiguous int64/uint64 tensors")
            if tuple(x.shape[-len(shape_tail):]) != tuple(shape_tail):
                raise EngineError(-1, "expected trailing shape %s, got %s" % (shape_tail, tuple(x.shape)))
            self._fence_torch()
            return x.data_ptr(), tuple(x.shape[:-len(shape_tail)]), _native.MEM_DEVICE, x
        a = np.ascontiguousarray(x, dtype=np.uint64)
        if tuple(a.shape[-len(shape_tail):]) != tuple(shape_tail):
            raise EngineError(-1, "expected trailing shape %s, got %s" % (shape_tail, a.shape))
        return a.ctypes.data, tuple(a.shape[:-len(shape_tail)]), _native.MEM_HOST, a

    @staticmethod
    def _flags(flags, async_):
        """The flags of a call on buffers of memory space `flags`: ASYNC only when asked for and only for DEVICE buffers
        (MEM_HOST is 0); a HOST call is always synchronous."""
        return flags | (_native.ASYNC if async_ and flags else 0)

    @staticmethod
    def _same_space(*flags):
        if len(set(flags)) > 1:
            raise EngineError(-1, "all buffers must live in the same memory space")

    def _check_out(self, out, shape, like, itemsize=8):
        """A caller-supplied result buffer goes to native code as a raw pointer: refuse anything whose shape,
        element type, contiguity or memory space differs from what the call will write."""
        shape = tuple(int(v) for v in shape)
        if _is_torch(like):
            if not _is_torch(out) or not out.is_cuda or out.device != like.device:
                raise EngineError(-1, "out must be a CUDA tensor on %s" % like.device)
            ok_dtype = str(out.dtype) in (("torch.int64", "torch.uint64") if itemsize == 8 else ("torch.uint8",))
            if tuple(out.shape) != shape or not ok_dtype or not out.is_contiguous():
                raise EngineError(-1, "out must be a contiguous %d-byte integer tensor of shape %s" % (itemsize, shape))
        else:
            want = np.uint64 if itemsize == 8 else np.uint8
            if not isinstance(out, np.ndarray) or out.dtype != want or tuple(out.shape) != shape or \
                    not out.flags.c_contiguous or not out.flags.writeable:
                raise EngineError(-1, "out must be a writable C-contiguous %s array of shape %s" % (np.dtype(want).name, shape))
        return out

    @staticmethod
    def _same_lead(name, lead, n):
        if tuple(lead) != (n,):
            raise EngineError(-1, "%s must have %d rows, got leading shape %s" % (name, n, tuple(lead)))

    def _out_like(self, like, shape, itemsize=8):
        """An uninitialised result buffer in the memory space of `like`: 64-bit words (a tensor takes the dtype of
        `like`) or, with itemsize 1, bytes."""
        if _is_torch(like):
            import torch
            return torch.empty(shape, dtype=like.dtype if itemsize == 8 else torch.uint8, device=like.device)
        return np.empty(shape, dtype=np.uint64 if itemsize == 8 else np.uint8)

    def _ok_like(self, like, n):
        return self._out_like(like, (n,), itemsize=1)

    def _result(self, out, shape, like, itemsize=8):
        """The buffer a call writes its result to: a new one like `like`, or the caller's `out` once it is validated."""
        return self._out_like(like, shape, itemsize) if out is None else self._check_out(out, shape, like, itemsize)

    def _rows_like(self, like, rows):
        """A new (rows, 4) result buffer whose pointer is never NULL, even for zero rows."""
        return self._out_like(like, (max(rows, 1), 4))[:rows]

    @staticmethod
    def _ptr(x):
        return x.data_ptr() if _is_torch(x) else x.ctypes.data

    @staticmethod
    def _host_limbs(x, shape, what):
        """A public value the library reads on the host for every memory space, as a host uint64 array of `shape`: a CUDA
        tensor is copied there, and int64 (a tensor's dtype) is reinterpreted, not converted."""
        a = np.ascontiguousarray(x.detach().cpu().numpy() if _is_torch(x) else x)
        b = a.view(np.uint64) if a.dtype == np.int64 else np.ascontiguousarray(a, dtype=np.uint64)
        if b.size != int(np.prod(shape)):
            raise EngineError(-1, "%s of shape %s, got %s" % (what, shape, b.shape))
        return b.reshape(shape)

    # -- hades::permute_batch ---------------------------------------------------------------------
    def permute_batch(self, states, dense=False, out=None, async_=False):
        """n x Safe::permute (src/hades/permutation/scalar.rs:25-27).  states: (n, 5, 4)."""
        ptr, lead, flags, keep = self._in(states, (5, 4))
        n = int(np.prod(lead)) if lead else 1
        if _is_torch(keep):
            if out is None:
                res = keep.clone()
            else:
                res = self._check_out(out, keep.shape, keep)
                if out is not keep:
                    out.copy_(keep)
            self._fence_torch()                   # that copy was enqueued on torch's stream
        elif out is not None:
            res = self._check_out(out, keep.shape, keep)
            if res is not states:
                np.copyto(res, keep)              # the caller's `states` stays untouched
        else:
            res = keep.copy() if keep is states else keep   # `keep` is already a private copy otherwise
        fn = self._lib.p252_permute_batch_dense if dense else self._lib.p252_permute_batch
        self._check(fn(self._ctx, self._ptr(res), n, self._flags(flags, async_)))
        return res

    def permute_batch_inplace(self, states, async_=False):
        ptr, lead, flags, keep = self._in(states, (5, 4))
        n = int(np.prod(lead)) if lead else 1
        if not _is_torch(keep) and keep is not states:
            raise EngineError(-1, "in-place permute needs a contiguous uint64 array")
        self._check(self._lib.p252_permute_batch(self._ctx, ptr, n, self._flags(flags, async_)))
        return states

    # -- sponges ------------------------------------------------------------------------------------
    def _sponge_batch(self, fn, first, inputs, out_len, out, async_):
        """The fixed-length digest calls: fn(ctx, first, inputs, n, in_len, out, out_len, flags); `first` is the tag
        pointer or the domain."""
        if inputs.ndim != 3:
            raise EngineError(-1, "inputs must have shape (n, in_len, 4)")
        in_len = int(inputs.shape[1])
        ptr, lead, flags, keep = self._in(inputs, (in_len, 4))
        n = lead[0]
        res = self._result(out, (n, int(out_len), 4), keep)
        self._check(fn(self._ctx, first, ptr, n, in_len, self._ptr(res), int(out_len), self._flags(flags, async_)))
        return res

    def digest_batch_with_tag(self, tag, inputs, out_len=1, out=None, async_=False):
        """start(tag) -> absorb(in_len) -> squeeze(out_len) for every item.  inputs: (n, in_len, 4)."""
        tag = np.ascontiguousarray(tag, dtype=np.uint64).reshape(4)
        return self._sponge_batch(self._lib.p252_digest_batch, tag.ctypes.data, inputs, out_len, out, async_)

    def hash_batch(self, domain, inputs, out_len=1, out=None, async_=False):
        """n x Hash::digest(domain, inputs[i]) with output_len(out_len)."""
        return self._sponge_batch(self._lib.p252_hash_batch, int(domain), inputs, out_len, out, async_)

    def hash_batch_truncated(self, domain, inputs, out_len=1, out=None, async_=False):
        """n x Hash::digest_truncated: raw (canonical, 250-bit masked) limbs for JubJubScalar::from_raw."""
        return self._sponge_batch(self._lib.p252_hash_batch_truncated, int(domain), inputs, out_len, out, async_)

    @staticmethod
    def _longest_item(offsets, n, extra=0):
        """max_len of a varlen call that was given none: the longest of the n items at `offsets`, less the `extra`
        scalars an item carries beyond its message, at least 1.  CUDA offsets cost one device-to-host read."""
        if n == 0:
            return 1
        if _is_torch(offsets):
            import torch
            o = offsets.view(torch.int64)
            longest = int((o[1:] - o[:-1]).max().item())
        else:
            longest = int((offsets[1:].astype(np.int64) - offsets[:-1].astype(np.int64)).max())
        return max(longest - extra, 1)

    def hash_batch_varlen(self, domain, data, offsets, out_len=1, max_len=None, out=None, async_=False):
        """n x Hash::digest(domain, data[offsets[i]:offsets[i+1]]) with output_len(out_len), inputs of any lengths in one
        call.  data (n_scalars, 4) and offsets (n + 1,) live in the same memory space (numpy, or CUDA tensors); offsets[0]
        need not be 0.  Returns (n, out_len, 4) in input order.  max_len bounds the item lengths (at most
        VARLEN_MAX_LEN); None takes the longest item, which for CUDA tensors costs a device-to-host sync.  Host batches
        raise on an invalid item and write nothing; device batches give invalid items a zero row and count them
        (last_varlen_rejected())."""
        dp, dlead, flags, dk = self._in(data, (4,))
        op, n1, ok_ = self._idx(offsets, dk, "offsets")
        if n1 < 1:
            raise EngineError(-1, "offsets must have n + 1 >= 1 entries")
        n = n1 - 1
        if max_len is None:
            max_len = self._longest_item(ok_, n)
        res = self._result(out, (n, int(out_len), 4), dk)
        flags = self._flags(flags, async_)
        rejected = self._counter("varlen_rejected", flags)
        self._check(self._lib.p252_hash_batch_varlen(self._ctx, int(domain), dp, int(dlead[0]), op, n, int(max_len),
                                                     self._ptr(res), int(out_len), ctypes.byref(rejected), flags))
        return res

    def last_varlen_rejected(self):
        """Items of the last hash_batch_varlen skipped as invalid (device buffers; sync() first after async_)."""
        return self._last("varlen_rejected")

    def hash_batch_mixed(self, mode, data, offsets, out_offsets, max_len=None, max_out_len=None, out=None, async_=False):
        """Every Hash the reference can build, in one call: item i is Hash::new(mode[i] & 3), update(data[offsets[i]:
        offsets[i+1]]), output_len(out_offsets[i+1] - out_offsets[i]), then finalize(), or finalize_truncated() where
        mode[i] & MIXED_TRUNCATED (raw limbs masked to 250 bits).  mode (n,) uint8, data (n_scalars, 4), offsets and
        out_offsets (n + 1,) live in one memory space (numpy, or CUDA tensors on one device); offsets[0] and out_offsets[0]
        need not be 0.  Returns (n_out, 4) with n_out = out_offsets[-1]: item i's rows are out[out_offsets[i]:
        out_offsets[i+1]]; a caller's `out` of (n_out, 4) may hold more rows.  max_len / max_out_len bound the input /
        output lengths (at most VARLEN_MAX_LEN); None takes the longest item, which for CUDA tensors costs a
        device-to-host sync.  Host batches raise for the lowest-index
        invalid item and write nothing; device batches give invalid items zero rows and count them
        (last_mixed_rejected())."""
        dp, dlead, flags, dk = self._in(data, (4,))
        op, n1, ok_ = self._idx(offsets, dk, "offsets")
        oop, no1, ook = self._idx(out_offsets, dk, "out_offsets")
        if n1 < 1 or no1 != n1:
            raise EngineError(-1, "offsets and out_offsets must both have n + 1 >= 1 entries")
        n = n1 - 1
        mp, mk = self._bytes(mode, dk, "mode", n)
        if max_len is None:
            max_len = self._longest_item(ok_, n)
        if max_out_len is None:
            max_out_len = self._longest_item(ook, n)
        if out is None:
            if _is_torch(ook):
                import torch
                n_out = int(ook.view(torch.int64)[-1].item())
            else:
                n_out = int(ook[-1])
            res = self._rows_like(dk, n_out)
        else:
            n_out = int(out.shape[0]) if getattr(out, "ndim", 0) == 2 else -1
            res = self._check_out(out, (n_out, 4), dk)
        flags = self._flags(flags, async_)
        rejected = self._counter("mixed_rejected", flags)
        self._check(self._lib.p252_hash_batch_mixed(self._ctx, mp, dp, int(dlead[0]), op, n, int(max_len), self._ptr(res),
                                                    n_out, oop, int(max_out_len), ctypes.byref(rejected), flags))
        return res

    def last_mixed_rejected(self):
        """Items of the last hash_batch_mixed skipped as invalid (device buffers; sync() first after async_)."""
        return self._last("mixed_rejected")

    def scalars_from_bytes(self, data, async_=False):
        """(n, 32) uint8 canonical little-endian (host) or (n, 4) 64-bit device tensor of the same bytes
        -> (scalars (n, 4), ok (n,) uint8); ok == 0 where the value is >= p."""
        if _is_torch(data):
            ptr, lead, flags, keep = self._in(data, (4,))
            n = lead[0]
        else:
            keep = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1, 32)
            ptr, n, flags = keep.ctypes.data, keep.shape[0], _native.MEM_HOST
        out = self._out_like(keep, (n, 4))
        ok = self._ok_like(keep, n)
        self._check(self._lib.p252_scalars_from_bytes(self._ctx, ptr, n, self._ptr(out), self._ptr(ok),
                                                      self._flags(flags, async_)))
        return out, ok

    def scalars_from_bytes_wide(self, data, async_=False):
        """BlsScalar::from_bytes_wide: (n, 64) uint8 rows (host) or an (n, 8) 64-bit device tensor of the same bytes
        -> (n, 4) scalars, (lo + hi 2^256) mod p in Montgomery form.  Every row is valid."""
        if _is_torch(data):
            ptr, lead, flags, keep = self._in(data, (8,))
            n = lead[0]
        else:
            keep = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1, 64)
            ptr, n, flags = keep.ctypes.data, keep.shape[0], _native.MEM_HOST
        out = self._out_like(keep, (n, 4)) if _is_torch(keep) else np.empty((n, 4), dtype=np.uint64)
        self._check(self._lib.p252_scalars_from_bytes_wide(self._ctx, ptr, n, self._ptr(out), self._flags(flags, async_)))
        return out

    def hash_to_scalar_batch(self, data, offsets, max_len=None, out=None, async_=False):
        """n x BlsScalar::hash_to_scalar(data[offsets[i]:offsets[i+1]]) in one call, byte strings of any lengths (0 included).
        data: a 1-D uint8 numpy array (or bytes) with (n + 1,) uint64 offsets, or a contiguous 1-D uint8 CUDA tensor with
        int64 / uint64 CUDA offsets; offsets[0] need not be 0.  Returns (n, 4) scalars in Montgomery form, in input order,
        in the memory space of the inputs: the rows are ready as the msg of the Schnorr calls.  max_len bounds the item
        lengths in bytes (at most HASH_TO_SCALAR_MAX_LEN); None takes the longest item, which for CUDA tensors costs a
        device-to-host sync.  Host batches raise on an invalid item and write nothing; device batches give invalid items a
        zero row and count them (last_hash_to_scalar_rejected())."""
        if _is_torch(data):
            if not data.is_cuda or data.device.index != self.device or str(data.dtype) != "torch.uint8" or \
                    not data.is_contiguous() or data.dim() != 1:
                raise EngineError(-1, "data must be a contiguous 1-D uint8 tensor on cuda:%d" % self.device)
            self._fence_torch()
            dp, nb, flags, dk = data.data_ptr(), int(data.shape[0]), _native.MEM_DEVICE, data
        else:
            if isinstance(data, (bytes, bytearray, memoryview)):
                data = np.frombuffer(data, dtype=np.uint8)
            dk = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
            dp, nb, flags = dk.ctypes.data, int(dk.shape[0]), _native.MEM_HOST
        op, n1, ok_ = self._idx(offsets, dk, "offsets")
        if n1 < 1:
            raise EngineError(-1, "offsets must have n + 1 >= 1 entries")
        n = n1 - 1
        if max_len is None:
            max_len = self._longest_item(ok_, n)
        res = self._result(out, (n, 4), ok_)
        flags = self._flags(flags, async_)
        rejected = self._counter("hash_to_scalar_rejected", flags)
        self._check(self._lib.p252_hash_to_scalar_batch(self._ctx, dp, nb, op, n, int(max_len), self._ptr(res),
                                                        ctypes.byref(rejected), flags))
        return res

    def last_hash_to_scalar_rejected(self):
        """Items of the last hash_to_scalar_batch skipped as invalid (device buffers; sync() first after async_)."""
        return self._last("hash_to_scalar_rejected")

    def scalars_to_bytes(self, scalars, async_=False):
        """(n, 4) scalars -> canonical little-endian bytes: (n, 32) uint8 (host) or (n, 4) device tensor."""
        ptr, lead, flags, keep = self._in(scalars, (4,))
        n = lead[0]
        out = self._out_like(keep, (n, 4)) if _is_torch(keep) else np.empty((n, 32), dtype=np.uint8)
        self._check(self._lib.p252_scalars_to_bytes(self._ctx, ptr, n, self._ptr(out), self._flags(flags, async_)))
        return out

    def encrypt_batch(self, messages, secrets_uv, nonces, out=None, async_=False):
        """messages (n, L, 4), secrets_uv (n, 2, 4), nonces (n, 4) -> ciphers (n, L+1, 4)."""
        L = int(messages.shape[1])
        mp, lead, flags, mk = self._in(messages, (L, 4))
        n = lead[0]
        sp, l2, f2, sk = self._in(secrets_uv, (2, 4))
        np_, l3, f3, nk = self._in(nonces, (4,))
        self._same_space(flags, f2, f3)
        self._same_lead("secrets_uv", l2, n)
        self._same_lead("nonces", l3, n)
        res = self._result(out, (n, L + 1, 4), mk)
        self._check(self._lib.p252_encrypt_batch(self._ctx, mp, n, L, sp, np_, self._ptr(res), self._flags(flags, async_)))
        return res

    def decrypt_batch(self, ciphers, secrets_uv, nonces, async_=False):
        """ciphers (n, L+1, 4) -> (messages (n, L, 4), ok (n,) uint8)."""
        L = int(ciphers.shape[1]) - 1
        cp, lead, flags, ck = self._in(ciphers, (L + 1, 4))
        n = lead[0]
        sp, l2, f2, sk = self._in(secrets_uv, (2, 4))
        np_, l3, f3, nk = self._in(nonces, (4,))
        self._same_space(flags, f2, f3)
        self._same_lead("secrets_uv", l2, n)
        self._same_lead("nonces", l3, n)
        if L < 1:
            raise EngineError(-1, "ciphers must hold at least one message scalar plus the authentication scalar")
        msg = self._out_like(ck, (n, L, 4))
        ok = self._ok_like(ck, n)
        flags = self._flags(flags, async_)
        failed = self._counter("decrypt_failures", flags)
        self._check(self._lib.p252_decrypt_batch(self._ctx, cp, n, L, sp, np_, self._ptr(msg), self._ptr(ok),
                                                 ctypes.byref(failed), flags))
        return msg, ok

    def last_decrypt_failures(self):
        """Items of the last decrypt_batch or decrypt_batch_varlen whose authentication failed (counted on the device for
        device buffers; after an async_ call, sync() first)."""
        return self._last("decrypt_failures")

    # -- JubJub key exchange ----------------------------------------------------------------------
    def _dhke_args(self, secrets, publics, n=None):
        """Shared validation of the dhke calls -> (secret ptr, n_secret, public ptr, n_public, n, flags, keepalives).
        secrets (n_secret, 4) p252_jscalar rows (scalar.jubjub_limbs), publics (n_public, 2, 4); each leading dimension
        is 1 (broadcast) or n.  n: the batch size the other buffers fix, or None to take it from these two."""
        sp, sl, fs, sk = self._in(secrets, (4,))
        pp, pl, fp, pk = self._in(publics, (2, 4))
        self._same_space(fs, fp)
        if len(sl) != 1 or len(pl) != 1:
            raise EngineError(-1, "secrets must have shape (n_secret, 4) and publics (n_public, 2, 4)")
        ns, npub = int(sl[0]), int(pl[0])
        if n is None:
            n = npub if ns == 1 else ns
        for name, k in (("secrets", ns), ("publics", npub)):
            if k not in (1, n):
                raise EngineError(-1, "%s must have 1 or %d rows, got %d" % (name, n, k))
        return sp, ns, pp, npub, n, fs, (sk, pk)

    def dhke_batch(self, secrets, publics, out=None, async_=False):
        """n x dhke(secret, public) = [secret] public as (u, v): secrets (n_secret, 4) canonical p252_jscalar rows,
        publics (n_public, 2, 4); n_secret and n_public are each 1 or n -> (shared (n, 2, 4), ok (n,) uint8).  ok[i] == 0
        marks an invalid item (secret >= r_J, or the point not on the curve with u, v < p); its output is (0, 0) and it is
        counted in last_dhke_invalid()."""
        sp, ns, pp, npub, n, flags, keep = self._dhke_args(secrets, publics)
        like = keep[1]
        res = self._result(out, (n, 2, 4), like)
        ok = self._ok_like(like, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("dhke_invalid", flags)
        self._check(self._lib.p252_dhke_batch(self._ctx, sp, ns, pp, npub, n, self._ptr(res), self._ptr(ok),
                                              ctypes.byref(invalid), flags))
        return res, ok

    def last_dhke_invalid(self):
        """Invalid items of the last dhke_batch or encrypt_batch_dhke (sync() first after async_)."""
        return self._last("dhke_invalid")

    def _crypt_dhke(self, decrypt, data, secrets, publics, nonces, out, async_):
        L = int(data.shape[1]) - (1 if decrypt else 0)
        if L < 1:
            raise EngineError(-1, "ciphers must hold at least one message scalar plus the authentication scalar" if decrypt
                              else "messages must hold at least one scalar")
        dp, lead, flags, dk = self._in(data, (int(data.shape[1]), 4))
        if len(lead) != 1:
            raise EngineError(-1, "expected shape (n, %s, 4)" % ("L + 1" if decrypt else "L"))
        n = lead[0]
        sp, ns, pp, npub, _, f2, keep = self._dhke_args(secrets, publics, n)
        np_, l3, f3, nk = self._in(nonces, (4,))
        self._same_space(flags, f2, f3)
        self._same_lead("nonces", l3, n)
        res = self._result(out, (n, L if decrypt else L + 1, 4), dk)
        ok = self._ok_like(dk, n)
        flags = self._flags(flags, async_)
        cnt = self._counter("decrypt_failures" if decrypt else "dhke_invalid", flags)
        fn = self._lib.p252_decrypt_batch_dhke if decrypt else self._lib.p252_encrypt_batch_dhke
        self._check(fn(self._ctx, dp, n, L, sp, ns, pp, npub, np_, self._ptr(res), self._ptr(ok), ctypes.byref(cnt), flags))
        return res, ok

    def encrypt_batch_dhke(self, messages, secrets, publics, nonces, out=None, async_=False):
        """n x encrypt(messages[i], dhke(secret, public), nonces[i]) with the shared secret derived on the device and never
        returned: messages (n, L, 4), secrets (1 or n, 4) p252_jscalar rows, publics (1 or n, 2, 4), nonces (n, 4) ->
        (ciphers (n, L+1, 4), ok (n,) uint8).  An invalid key-exchange item has ok == 0 and a zeroed cipher row (count:
        last_dhke_invalid())."""
        return self._crypt_dhke(False, messages, secrets, publics, nonces, out, async_)

    def decrypt_batch_dhke(self, ciphers, secrets, publics, nonces, out=None, async_=False):
        """n x decrypt(ciphers[i], dhke(secret, public), nonces[i]) -> (messages (n, L, 4), ok (n,) uint8).  ok == 0 for an
        authentication failure or an invalid key-exchange item (message zeroed); their count: last_decrypt_failures().
        The wallet-scan shape is one view key (secrets of 1 row) against every note's public key."""
        return self._crypt_dhke(True, ciphers, secrets, publics, nonces, out, async_)

    # -- fixed-base JubJub scalar multiplication --------------------------------------------------
    @classmethod
    def _base(cls, base):
        """The base point (u, v) as a host (2, 4) uint64 array: the library reads it on the host for every memory space
        (a CUDA tensor is copied; the base is public)."""
        return cls._host_limbs(base, (2, 4), "base must be one point (u, v)")

    def fixed_base_batch(self, secrets, base, out=None, async_=False):
        """n x [secret] base for one base point: secrets (n, 4) canonical p252_jscalar rows (scalar.jubjub_limbs), base
        (2, 4) -- e.g. the generator, for public keys or ephemeral keys R = [r] G -> (points (n, 2, 4), ok (n,) uint8).
        ok[i] == 0 marks a secret >= r_J; its output is (0, 0) and it is counted in last_dhke_invalid().  The base is
        read on the host (a CUDA tensor is copied there); a base off the curve raises InvalidPoint.  The engine keeps
        the table of its last base, so repeated calls with one base build it once."""
        sp, sl, flags, sk = self._in(secrets, (4,))
        if len(sl) != 1:
            raise EngineError(-1, "secrets must have shape (n, 4)")
        n = int(sl[0])
        b = self._base(base)
        res = self._result(out, (n, 2, 4), sk)
        ok = self._ok_like(sk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("dhke_invalid", flags)
        self._check(self._lib.p252_fixed_base_batch(self._ctx, b.ctypes.data, sp, n, self._ptr(res), self._ptr(ok),
                                                    ctypes.byref(invalid), flags))
        return res, ok

    def encrypt_batch_ephemeral(self, messages, r, base, publics, nonces, out=None, R_out=None, async_=False):
        """The sender's side of the reference's key exchange as one call: R_i = [r_i] base and
        cipher_i = encrypt(messages[i], dhke(r_i, publics[i]), nonces[i]) with the shared secret derived on the device and
        never returned.  messages (n, L, 4), r (n, 4) p252_jscalar rows, base (2, 4) (host-read, as in fixed_base_batch),
        publics (1 or n, 2, 4), nonces (n, 4) -> (ciphers (n, L+1, 4), R (n, 2, 4), ok (n,) uint8).  An item with
        r >= r_J or a public key off the curve has ok == 0 and zeroed cipher and R rows (count: last_dhke_invalid())."""
        L = int(messages.shape[1])
        if L < 1:
            raise EngineError(-1, "messages must hold at least one scalar")
        dp, lead, flags, dk = self._in(messages, (L, 4))
        if len(lead) != 1:
            raise EngineError(-1, "expected shape (n, L, 4)")
        n = lead[0]
        sp, ns, pp, npub, _, f2, keep = self._dhke_args(r, publics, n)
        if ns != n:
            raise EngineError(-1, "r must have %d rows, got %d" % (n, ns))
        np_, l3, f3, nk = self._in(nonces, (4,))
        self._same_space(flags, f2, f3)
        self._same_lead("nonces", l3, n)
        b = self._base(base)
        res = self._result(out, (n, L + 1, 4), dk)
        R = self._result(R_out, (n, 2, 4), dk)
        ok = self._ok_like(dk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("dhke_invalid", flags)
        self._check(self._lib.p252_encrypt_batch_ephemeral(self._ctx, dp, n, L, sp, b.ctypes.data, pp, npub, np_,
                                                           self._ptr(res), self._ptr(R), self._ptr(ok),
                                                           ctypes.byref(invalid), flags))
        return res, R, ok

    # -- stealth addresses ------------------------------------------------------------------------
    def stealth_address_batch(self, r, base, publics_A, publics_B, R_out=None, out=None, async_=False):
        """The sender's stealth addresses: R_i = [r_i] base and note_pk_i = [hash([r_i] A_i)] base + B_i, where
        hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0].  r (n, 4) p252_jscalar rows, base (2, 4)
        (host-read, as in fixed_base_batch), publics_A and publics_B (1 or n, 2, 4) with the same number of rows: the
        receiver's public key (A, B) -> (R (n, 2, 4), note_pk (n, 2, 4), ok (n,) uint8).  An item with r >= r_J or A or B
        not a curve point has ok == 0 and zeroed R and note_pk rows (count: last_stealth_invalid())."""
        if len(tuple(r.shape)) != 2:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(r.shape[0])
        sp, _, ap, na, _, flags, keep = self._dhke_args(r, publics_A, n)
        bp, bl, fb, bk = self._in(publics_B, (2, 4))
        self._same_space(flags, fb)
        if tuple(bl) != (na,):
            raise EngineError(-1, "publics_B must have %d rows like publics_A, got leading shape %s" % (na, tuple(bl)))
        b = self._base(base)
        like = keep[0]
        R = self._result(R_out, (n, 2, 4), like)
        pk = self._result(out, (n, 2, 4), like)
        ok = self._ok_like(like, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("stealth_invalid", flags)
        self._check(self._lib.p252_stealth_address_batch(self._ctx, sp, n, b.ctypes.data, ap, bp, na, self._ptr(R),
                                                         self._ptr(pk), self._ptr(ok), ctypes.byref(invalid), flags))
        return R, pk, ok

    def stealth_owns_batch(self, view_a, spend_B, base, R, note_pk, out=None, async_=False):
        """The receiver's scan, ViewKey::owns over a batch of notes: owned[i] = note_pk[i] == [hash([view_a] R[i])] base +
        spend_B.  view_a: one p252_jscalar row (1, 4) in the memory space of R and note_pk (n, 2, 4); spend_B and base
        (2, 4) are host-read, as the base of fixed_base_batch -> owned (n,) uint8.  An item with view_a >= r_J, R not a
        curve point or a note_pk coordinate >= p is invalid: owned == 0, counted in last_stealth_invalid(), not in
        last_stealth_owned().  A spend_B or base off the curve raises InvalidPoint."""
        rp, rl, flags, rk = self._in(R, (2, 4))
        if len(rl) != 1:
            raise EngineError(-1, "R must have shape (n, 2, 4)")
        n = rl[0]
        pp, pl, fp, pk = self._in(note_pk, (2, 4))
        vp, vl, fv, vk = self._in(view_a, (4,))
        self._same_space(flags, fp, fv)
        self._same_lead("note_pk", pl, n)
        if tuple(vl) not in ((), (1,)):
            raise EngineError(-1, "view_a must be one p252_jscalar row, got leading shape %s" % (tuple(vl),))
        b, g = self._base(spend_B), self._base(base)
        owned = self._result(out, (n,), rk, itemsize=1)
        flags = self._flags(flags, async_)
        n_owned, invalid = self._counter("stealth_owned", flags), self._counter("stealth_invalid", flags)
        self._check(self._lib.p252_stealth_owns_batch(self._ctx, vp, b.ctypes.data, g.ctypes.data, rp, pp, n,
                                                      self._ptr(owned), ctypes.byref(n_owned), ctypes.byref(invalid),
                                                      flags))
        return owned

    def last_stealth_owned(self):
        """Owned notes of the last stealth_owns_batch (sync() first after async_)."""
        return self._last("stealth_owned")

    def last_stealth_invalid(self):
        """Invalid items of the last stealth_address_batch or stealth_owns_batch (sync() first after async_)."""
        return self._last("stealth_invalid")

    # -- Schnorr signatures -----------------------------------------------------------------------
    def schnorr_sign_batch(self, sk, r, msg, base, u_out=None, R_out=None, async_=False):
        """jubjub-schnorr's SecretKey::sign over a batch: R_i = [r_i] base, c_i = challenge(R_i, msg_i) =
        Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0] and u_i = (r_i - c_i sk_i) mod r_J.  sk (1 or n, 4) and
        r (n, 4) p252_jscalar rows (one nonce per message, never reused), msg (n, 4) BlsScalar.0 limbs, base (2, 4)
        (host-read, as in fixed_base_batch) -> (u (n, 4), R (n, 2, 4), ok (n,) uint8).  An item with sk or r >= r_J or
        msg >= p has ok == 0 and zeroed u and R rows (count: last_schnorr_invalid())."""
        rp, rl, flags, rk = self._in(r, (4,))
        if len(rl) != 1:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(rl[0])
        sp, sl, fs, skk = self._in(sk, (4,))
        mp, ml, fm, mk = self._in(msg, (4,))
        self._same_space(flags, fs, fm)
        if len(sl) != 1 or int(sl[0]) not in (1, n):
            raise EngineError(-1, "sk must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(sl)))
        self._same_lead("msg", ml, n)
        b = self._base(base)
        u = self._result(u_out, (n, 4), rk)
        R = self._result(R_out, (n, 2, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("schnorr_invalid", flags)
        self._check(self._lib.p252_schnorr_sign_batch(self._ctx, sp, int(sl[0]), rp, mp, n, b.ctypes.data, self._ptr(u),
                                                      self._ptr(R), self._ptr(ok), ctypes.byref(invalid), flags))
        return u, R, ok

    def schnorr_verify_batch(self, pk, u, R, msg, base, out=None, async_=False):
        """jubjub-schnorr's PublicKey::verify over a batch: verified[i] = [u_i] base + [c_i] PK_i == R_i with
        c_i = challenge(R_i, msg_i).  pk (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R (n, 2, 4), msg (n, 4), base (2, 4)
        (host-read) -> verified (n,) uint8.  An item with u >= r_J, msg >= p, an R coordinate >= p or PK not a curve point
        is invalid: verified == 0, counted in last_schnorr_invalid(), not in last_schnorr_verified().  A base off the
        curve raises InvalidPoint."""
        up, ul, flags, uk = self._in(u, (4,))
        if len(ul) != 1:
            raise EngineError(-1, "u must have shape (n, 4)")
        n = int(ul[0])
        pp, pl, fp, pkk = self._in(pk, (2, 4))
        Rp, Rl, fR, Rk = self._in(R, (2, 4))
        mp, ml, fm, mk = self._in(msg, (4,))
        self._same_space(flags, fp, fR, fm)
        if len(pl) != 1 or int(pl[0]) not in (1, n):
            raise EngineError(-1, "pk must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(pl)))
        self._same_lead("R", Rl, n)
        self._same_lead("msg", ml, n)
        b = self._base(base)
        verified = self._result(out, (n,), uk, itemsize=1)
        flags = self._flags(flags, async_)
        n_verified, invalid = self._counter("schnorr_verified", flags), self._counter("schnorr_invalid", flags)
        self._check(self._lib.p252_schnorr_verify_batch(self._ctx, pp, int(pl[0]), up, Rp, mp, n, b.ctypes.data,
                                                        self._ptr(verified), ctypes.byref(n_verified),
                                                        ctypes.byref(invalid), flags))
        return verified

    def last_schnorr_verified(self):
        """Verified signatures of the last schnorr_verify_batch (sync() first after async_)."""
        return self._last("schnorr_verified")

    def last_schnorr_invalid(self):
        """Invalid items of the last schnorr_sign_batch or schnorr_verify_batch (sync() first after async_)."""
        return self._last("schnorr_invalid")

    # -- note nullifiers --------------------------------------------------------------------------
    def nullifier_batch(self, a, b, base, R, pos, out=None, async_=False):
        """Phoenix note nullifiers: nullifier_i = Hash::digest(Domain::Other, [pk'.u, pk'.v, pos_i])[0] with
        pk' = [note_sk] base and note_sk = (hash([a] R_i) + b) mod r_J, hash(P) = Hash::digest_truncated(Domain::Other,
        [P.u, P.v])[0].  a and b (1 or n, 4) p252_jscalar rows with the same number of rows (the wallet's secret key),
        base (2, 4) (G', host-read, as in fixed_base_batch), R (n, 2, 4), pos (n,): a numpy uint64 array or a CUDA int64
        tensor -> (nullifier (n, 4), ok (n,) uint8).  An item with a or b >= r_J or R not a curve point has ok == 0 and a
        zeroed nullifier row (count: last_nullifier_invalid()).  A base off the curve raises InvalidPoint."""
        rp, rl, flags, rk = self._in(R, (2, 4))
        if len(rl) != 1:
            raise EngineError(-1, "R must have shape (n, 2, 4)")
        n = int(rl[0])
        ap, al, fa, ak = self._in(a, (4,))
        bp, bl, fb, bk = self._in(b, (4,))
        self._same_space(flags, fa, fb, _native.MEM_DEVICE if _is_torch(pos) else _native.MEM_HOST)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "a must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(al)))
        ns = int(al[0])
        if tuple(bl) != (ns,):
            raise EngineError(-1, "b must have %d rows like a, got leading shape %s" % (ns, tuple(bl)))
        pp, npos, pk = self._idx(pos, rk, "pos")
        if npos != n:
            raise EngineError(-1, "pos must have %d entries, got %d" % (n, npos))
        g = self._base(base)
        res = self._result(out, (n, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("nullifier_invalid", flags)
        self._check(self._lib.p252_nullifier_batch(self._ctx, ap, bp, ns, g.ctypes.data, rp, pp, n, self._ptr(res),
                                                   self._ptr(ok), ctypes.byref(invalid), flags))
        return res, ok

    def last_nullifier_invalid(self):
        """Invalid items of the last nullifier_batch (sync() first after async_)."""
        return self._last("nullifier_invalid")

    # -- double-key Schnorr signatures (SignatureDouble) and note signing ------------------------------
    def schnorr_sign_double_batch(self, sk, r, msg, base, base_p, async_=False):
        """jubjub-schnorr's SecretKey::sign_double over a batch: R_i = [r_i] base, R'_i = [r_i] base_p,
        c_i = challenge2(R_i, R'_i, msg_i) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0] and
        u_i = (r_i - c_i sk_i) mod r_J.  sk (1 or n, 4) and r (n, 4) p252_jscalar rows (one nonce per message, never
        reused), msg (n, 4), base (G) and base_p (G') (2, 4), host-read -> (u (n, 4), R (n, 2, 4), R' (n, 2, 4), ok (n,)
        uint8).  An item with sk or r >= r_J or msg >= p has ok == 0 and zeroed rows (count:
        last_schnorr_double_invalid()).  A base off the curve raises InvalidPoint."""
        rp, rl, flags, rk = self._in(r, (4,))
        if len(rl) != 1:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(rl[0])
        sp, sl, fs, skk = self._in(sk, (4,))
        mp, ml, fm, mk = self._in(msg, (4,))
        self._same_space(flags, fs, fm)
        if len(sl) != 1 or int(sl[0]) not in (1, n):
            raise EngineError(-1, "sk must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(sl)))
        self._same_lead("msg", ml, n)
        g, gp = self._base(base), self._base(base_p)
        u = self._result(None, (n, 4), rk)
        R = self._result(None, (n, 2, 4), rk)
        Rp = self._result(None, (n, 2, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("schnorr_double_invalid", flags)
        self._check(self._lib.p252_schnorr_sign_double_batch(self._ctx, sp, int(sl[0]), rp, mp, n, g.ctypes.data,
                                                             gp.ctypes.data, self._ptr(u), self._ptr(R), self._ptr(Rp),
                                                             self._ptr(ok), ctypes.byref(invalid), flags))
        return u, R, Rp, ok

    def schnorr_verify_double_batch(self, pk, pk_p, u, R, R_p, msg, base, base_p, async_=False):
        """jubjub-schnorr's SignatureDouble::verify over a batch: verified[i] = [u_i] base + [c_i] PK_i == R_i and
        [u_i] base_p + [c_i] PK'_i == R'_i with c_i = challenge2(R_i, R'_i, msg_i).  pk and pk_p (1 or n, 2, 4) with the
        same number of rows, u (n, 4) p252_jscalar rows, R and R_p (n, 2, 4), msg (n, 4), base and base_p (2, 4)
        (host-read) -> verified (n,) uint8.  An item with u >= r_J, msg >= p, a coordinate of R or R' >= p, or PK or PK'
        not a curve point is invalid: verified == 0, counted once in last_schnorr_double_invalid(), not in
        last_schnorr_double_verified().  A base off the curve raises InvalidPoint."""
        up, ul, flags, uk = self._in(u, (4,))
        if len(ul) != 1:
            raise EngineError(-1, "u must have shape (n, 4)")
        n = int(ul[0])
        pp, pl, fp, _ = self._in(pk, (2, 4))
        qp, ql, fq, _ = self._in(pk_p, (2, 4))
        Rp, Rl, fR, _ = self._in(R, (2, 4))
        Sp, Sl, fS, _ = self._in(R_p, (2, 4))
        mp, ml, fm, _ = self._in(msg, (4,))
        self._same_space(flags, fp, fq, fR, fS, fm)
        if len(pl) != 1 or int(pl[0]) not in (1, n):
            raise EngineError(-1, "pk must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(pl)))
        if tuple(ql) != tuple(pl):
            raise EngineError(-1, "pk_p must have %d rows like pk, got leading shape %s" % (int(pl[0]), tuple(ql)))
        self._same_lead("R", Rl, n)
        self._same_lead("R_p", Sl, n)
        self._same_lead("msg", ml, n)
        g, gp = self._base(base), self._base(base_p)
        verified = self._result(None, (n,), uk, itemsize=1)
        flags = self._flags(flags, async_)
        n_verified = self._counter("schnorr_double_verified", flags)
        invalid = self._counter("schnorr_double_invalid", flags)
        self._check(self._lib.p252_schnorr_verify_double_batch(self._ctx, pp, qp, int(pl[0]), up, Rp, Sp, mp, n,
                                                               g.ctypes.data, gp.ctypes.data, self._ptr(verified),
                                                               ctypes.byref(n_verified), ctypes.byref(invalid), flags))
        return verified

    def note_sign_double_batch(self, a, b, note_R, r, msg, base, base_p, async_=False):
        """Spend signatures of Phoenix notes: sign_double (as schnorr_sign_double_batch) under each note's secret key
        note_sk = (hash([a] note_R_i) + b) mod r_J, hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0].
        a and b (1 or n, 4) p252_jscalar rows with the same number of rows (the wallet's secret key), note_R (n, 2, 4)
        the notes' ephemeral keys, r (n, 4), msg (n, 4), base (G) and base_p (G') (2, 4), host-read -> (u (n, 4),
        R (n, 2, 4), R' (n, 2, 4), pk' (n, 2, 4), ok (n,) uint8) with pk' = [note_sk] base_p, the spend proof's witness:
        it links the spend to the note and must stay private.  An item with a, b or r >= r_J, note_R not a curve point
        or msg >= p has ok == 0 and zeroed rows (count: last_schnorr_double_invalid()).  note_sk never leaves the
        device."""
        rp, rl, flags, rk = self._in(r, (4,))
        if len(rl) != 1:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(rl[0])
        ap, al, fa, _ = self._in(a, (4,))
        bp, bl, fb, _ = self._in(b, (4,))
        np_, nl, fn, _ = self._in(note_R, (2, 4))
        mp, ml, fm, _ = self._in(msg, (4,))
        self._same_space(flags, fa, fb, fn, fm)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "a must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(al)))
        ns = int(al[0])
        if tuple(bl) != (ns,):
            raise EngineError(-1, "b must have %d rows like a, got leading shape %s" % (ns, tuple(bl)))
        self._same_lead("note_R", nl, n)
        self._same_lead("msg", ml, n)
        g, gp = self._base(base), self._base(base_p)
        u = self._result(None, (n, 4), rk)
        R = self._result(None, (n, 2, 4), rk)
        Rp = self._result(None, (n, 2, 4), rk)
        pkp = self._result(None, (n, 2, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("schnorr_double_invalid", flags)
        self._check(self._lib.p252_note_sign_double_batch(self._ctx, ap, bp, ns, np_, rp, mp, n, g.ctypes.data,
                                                          gp.ctypes.data, self._ptr(u), self._ptr(R), self._ptr(Rp),
                                                          self._ptr(pkp), self._ptr(ok), ctypes.byref(invalid), flags))
        return u, R, Rp, pkp, ok

    def last_schnorr_double_verified(self):
        """Verified signatures of the last schnorr_verify_double_batch (sync() first after async_)."""
        return self._last("schnorr_double_verified")

    def last_schnorr_double_invalid(self):
        """Invalid items of the last schnorr_sign_double_batch, schnorr_verify_double_batch or note_sign_double_batch
        (sync() first after async_)."""
        return self._last("schnorr_double_invalid")

    # -- note values: commitments, creating and opening notes ---------------------------------------------
    def _values(self, value, like, n):
        """value (n,): a numpy uint64 array, or a CUDA int64 tensor for device buffers"""
        vp, nv, vk = self._idx(value, like, "value")
        if nv != n:
            raise EngineError(-1, "value must have %d entries, got %d" % (n, nv))
        return vp, vk

    def value_commit_batch(self, value, blinder, base, base_p, async_=False):
        """Pedersen value commitments C_i = [value_i] base + [blinder_i] base_p.  value (n,) (a numpy uint64 array or a
        CUDA int64 tensor), blinder (n, 4) p252_jscalar rows, base (G) and base_p (G' = GENERATOR_NUMS) (2, 4),
        host-read -> (commitment (n, 2, 4), ok (n,) uint8).  An item with blinder >= r_J has ok == 0 and a zeroed row
        (count: last_note_invalid()).  A base off the curve raises InvalidPoint."""
        bp, bl, flags, bk = self._in(blinder, (4,))
        if len(bl) != 1:
            raise EngineError(-1, "blinder must have shape (n, 4)")
        n = int(bl[0])
        self._same_space(flags, _native.MEM_DEVICE if _is_torch(value) else _native.MEM_HOST)
        vp, vk = self._values(value, bk, n)
        g, gp = self._base(base), self._base(base_p)
        C = self._result(None, (n, 2, 4), bk)
        ok = self._ok_like(bk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("note_invalid", flags)
        self._check(self._lib.p252_value_commit_batch(self._ctx, vp, bp, n, g.ctypes.data, gp.ctypes.data, self._ptr(C),
                                                      self._ptr(ok), ctypes.byref(invalid), flags))
        return C, ok

    def note_create_batch(self, r, value, blinder, nonce, base, base_p, publics_A, publics_B, async_=False):
        """The sender's obfuscated notes: R_i = [r_i] base, S_i = [r_i] A_i, note_pk_i = [hash(S_i)] base + B_i,
        C_i = [value_i] base + [blinder_i] base_p and cipher_i = encrypt([Fr(value_i), Fr(blinder_i)], S_i, nonce_i), with
        hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0].  r and blinder (n, 4) p252_jscalar rows, value (n,)
        (a numpy uint64 array or a CUDA int64 tensor), nonce (n, 4), base (G) and base_p (G') (2, 4) host-read, publics_A
        and publics_B (1 or n, 2, 4) with the same number of rows: the receiver's public key -> (R (n, 2, 4), note_pk
        (n, 2, 4), commitment (n, 2, 4), cipher (n, 3, 4), ok (n,) uint8).  An item with r or blinder >= r_J or A or B not
        a curve point has ok == 0 and all four rows zeroed (count: last_note_invalid()).  S and hash(S) never leave the
        device."""
        rp, rl, flags, rk = self._in(r, (4,))
        if len(rl) != 1:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(rl[0])
        bp, bl, fb, bk = self._in(blinder, (4,))
        np_, nl, fn, nk = self._in(nonce, (4,))
        ap, al, fa, ak = self._in(publics_A, (2, 4))
        Bp, Bl, fB, Bk = self._in(publics_B, (2, 4))
        self._same_space(flags, fb, fn, fa, fB, _native.MEM_DEVICE if _is_torch(value) else _native.MEM_HOST)
        self._same_lead("blinder", bl, n)
        self._same_lead("nonce", nl, n)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "publics_A must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(al)))
        na = int(al[0])
        if tuple(Bl) != (na,):
            raise EngineError(-1, "publics_B must have %d rows like publics_A, got leading shape %s" % (na, tuple(Bl)))
        vp, vk = self._values(value, rk, n)
        g, gp = self._base(base), self._base(base_p)
        R = self._result(None, (n, 2, 4), rk)
        pk = self._result(None, (n, 2, 4), rk)
        C = self._result(None, (n, 2, 4), rk)
        cipher = self._result(None, (n, 3, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("note_invalid", flags)
        self._check(self._lib.p252_note_create_batch(self._ctx, rp, vp, bp, np_, n, g.ctypes.data, gp.ctypes.data, ap, Bp,
                                                     na, self._ptr(R), self._ptr(pk), self._ptr(C), self._ptr(cipher),
                                                     self._ptr(ok), ctypes.byref(invalid), flags))
        return R, pk, C, cipher, ok

    def note_open_batch(self, a, R, nonce, cipher, commitment, base, base_p, async_=False):
        """The wallet's checked openings: S_i = [a] R_i, (m0, m1) = decrypt(cipher_i, S_i, nonce_i), and the note opens iff
        the authentication passes, m0 < 2^64, m1 < r_J and [m0] base + [m1] base_p == commitment_i.  a (1 or n, 4)
        p252_jscalar rows (the view key), R (n, 2, 4), nonce (n, 4), cipher (n, 3, 4), commitment (n, 2, 4), base (G) and
        base_p (G') (2, 4) host-read -> (value (n,) (uint64, or int64 like the inputs' tensors), blinder (n, 4), ok (n,)
        uint8).  ok == 0 (value and blinder zeroed) for a note that does not open and for an invalid item (a >= r_J, R not
        a curve point); their count: last_note_failed().  value and blinder are the spend proof's witnesses: keep them as
        private as the note's key."""
        Rp, Rl, flags, Rk = self._in(R, (2, 4))
        if len(Rl) != 1:
            raise EngineError(-1, "R must have shape (n, 2, 4)")
        n = int(Rl[0])
        ap, al, fa, ak = self._in(a, (4,))
        np_, nl, fn, nk = self._in(nonce, (4,))
        cp, cl, fc, ck = self._in(cipher, (3, 4))
        Cp, Cl, fC, Ck = self._in(commitment, (2, 4))
        self._same_space(flags, fa, fn, fc, fC)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "a must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(al)))
        self._same_lead("nonce", nl, n)
        self._same_lead("cipher", cl, n)
        self._same_lead("commitment", Cl, n)
        g, gp = self._base(base), self._base(base_p)
        value = self._result(None, (n,), Rk)
        blinder = self._result(None, (n, 4), Rk)
        ok = self._ok_like(Rk, n)
        flags = self._flags(flags, async_)
        failed = self._counter("note_failed", flags)
        self._check(self._lib.p252_note_open_batch(self._ctx, ap, int(al[0]), Rp, np_, cp, Cp, n, g.ctypes.data,
                                                   gp.ctypes.data, self._ptr(value), self._ptr(blinder), self._ptr(ok),
                                                   ctypes.byref(failed), flags))
        return value, blinder, ok

    def last_note_invalid(self):
        """Invalid items of the last value_commit_batch or note_create_batch (sync() first after async_)."""
        return self._last("note_invalid")

    def last_note_failed(self):
        """Items of the last note_open_batch that did not open, invalid ones included (sync() first after async_)."""
        return self._last("note_failed")

    # -- JubJub ElGamal and the encrypted sender of a note ---------------------------------------------
    def elgamal_encrypt_batch(self, pk, msg, r, base, async_=False):
        """JubJub ElGamal: (c1_i, c2_i) = ([r_i] base, M_i + [r_i] PK_i).  pk (1 or n, 2, 4), msg (n, 2, 4), r (n, 4)
        p252_jscalar rows (one per message, never reused under one key: c2 - c2' would reveal M - M'), base (G) (2, 4),
        host-read -> (c1 (n, 2, 4), c2 (n, 2, 4), ok (n,) uint8).  An item with r >= r_J or PK or M not a curve point
        has ok == 0 and zeroed rows (count: last_elgamal_invalid()).  A base off the curve raises InvalidPoint."""
        rp, rl, flags, rk = self._in(r, (4,))
        if len(rl) != 1:
            raise EngineError(-1, "r must have shape (n, 4)")
        n = int(rl[0])
        pp, pl, fp, _ = self._in(pk, (2, 4))
        mp, ml, fm, _ = self._in(msg, (2, 4))
        self._same_space(flags, fp, fm)
        if len(pl) != 1 or int(pl[0]) not in (1, n):
            raise EngineError(-1, "pk must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(pl)))
        self._same_lead("msg", ml, n)
        g = self._base(base)
        c1 = self._result(None, (n, 2, 4), rk)
        c2 = self._result(None, (n, 2, 4), rk)
        ok = self._ok_like(rk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("elgamal_invalid", flags)
        self._check(self._lib.p252_elgamal_encrypt_batch(self._ctx, pp, int(pl[0]), mp, rp, n, g.ctypes.data,
                                                         self._ptr(c1), self._ptr(c2), self._ptr(ok),
                                                         ctypes.byref(invalid), flags))
        return c1, c2, ok

    def elgamal_decrypt_batch(self, sk, c1, c2, async_=False):
        """JubJub ElGamal decryption: M_i = c2_i - [sk_i] c1_i.  sk (1 or n, 4) p252_jscalar rows, c1 and c2 (n, 2, 4) ->
        (msg (n, 2, 4), ok (n,) uint8).  NOT authenticated: a wrong key gives another curve point with ok == 1.  An item
        with sk >= r_J or c1 or c2 not a curve point has ok == 0 and a zeroed row (count: last_elgamal_invalid())."""
        ap, al, flags, ak = self._in(c1, (2, 4))
        if len(al) != 1:
            raise EngineError(-1, "c1 must have shape (n, 2, 4)")
        n = int(al[0])
        sp, sl, fs, _ = self._in(sk, (4,))
        bp, bl, fb, _ = self._in(c2, (2, 4))
        self._same_space(flags, fs, fb)
        if len(sl) != 1 or int(sl[0]) not in (1, n):
            raise EngineError(-1, "sk must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(sl)))
        self._same_lead("c2", bl, n)
        msg = self._result(None, (n, 2, 4), ak)
        ok = self._ok_like(ak, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("elgamal_invalid", flags)
        self._check(self._lib.p252_elgamal_decrypt_batch(self._ctx, sp, int(sl[0]), ap, bp, n, self._ptr(msg),
                                                         self._ptr(ok), ctypes.byref(invalid), flags))
        return msg, ok

    def note_sender_encrypt_batch(self, note_pk, sender_A, sender_B, blinder, base, async_=False):
        """The encrypted sender of Phoenix notes: enc_i = [c1_A, c2_A, c1_B, c2_B], the ElGamal encryptions of the
        sender's A and B under note_pk_i with the blinders (r_A, r_B) = blinder_i.  note_pk (n, 2, 4), sender_A and
        sender_B (1 or n, 2, 4) with the same number of rows, blinder (n, 2, 4) p252_jscalar rows [r_A, r_B], base (G)
        (2, 4) host-read -> (enc (n, 4, 2, 4), ok (n,) uint8).  An item with a blinder >= r_J or a point not on the curve
        has ok == 0 and a zeroed row (count: last_elgamal_invalid())."""
        pp, pl, flags, pk = self._in(note_pk, (2, 4))
        if len(pl) != 1:
            raise EngineError(-1, "note_pk must have shape (n, 2, 4)")
        n = int(pl[0])
        ap, al, fa, _ = self._in(sender_A, (2, 4))
        bp, bl, fb, _ = self._in(sender_B, (2, 4))
        rp, rl, fr, _ = self._in(blinder, (2, 4))
        self._same_space(flags, fa, fb, fr)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "sender_A must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(al)))
        if tuple(bl) != tuple(al):
            raise EngineError(-1, "sender_B must have %d rows like sender_A, got leading shape %s" % (int(al[0]), tuple(bl)))
        self._same_lead("blinder", rl, n)
        g = self._base(base)
        enc = self._result(None, (n, 4, 2, 4), pk)
        ok = self._ok_like(pk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("elgamal_invalid", flags)
        self._check(self._lib.p252_note_sender_encrypt_batch(self._ctx, pp, ap, bp, int(al[0]), rp, n, g.ctypes.data,
                                                             self._ptr(enc), self._ptr(ok), ctypes.byref(invalid), flags))
        return enc, ok

    def note_sender_decrypt_batch(self, a, b, R, note_pk, enc, base, async_=False):
        """The owner's recovery of the sender: note_sk_i = (hash([a] R_i) + b) mod r_J, hash(P) =
        Hash::digest_truncated(Domain::Other, [P.u, P.v])[0]; where [note_sk_i] base == note_pk_i, A_i = c2_A - [note_sk]
        c1_A and B_i = c2_B - [note_sk] c1_B.  a and b (1 or n, 4) p252_jscalar rows with the same number of rows, R and
        note_pk (n, 2, 4), enc (n, 4, 2, 4) as note_sender_encrypt_batch writes it, base (G) (2, 4) host-read ->
        (A (n, 2, 4), B (n, 2, 4), ok (n,) uint8).  ok == 0 (A and B zeroed) for a note the key does not own and for an
        invalid item (a or b >= r_J, R or a ciphertext point not on the curve); their count: last_sender_failed().
        note_sk never leaves the device."""
        Rp, Rl, flags, Rk = self._in(R, (2, 4))
        if len(Rl) != 1:
            raise EngineError(-1, "R must have shape (n, 2, 4)")
        n = int(Rl[0])
        ap, al, fa, _ = self._in(a, (4,))
        bp, bl, fb, _ = self._in(b, (4,))
        pp, pl, fp, _ = self._in(note_pk, (2, 4))
        ep, el, fe, _ = self._in(enc, (4, 2, 4))
        self._same_space(flags, fa, fb, fp, fe)
        if len(al) != 1 or int(al[0]) not in (1, n):
            raise EngineError(-1, "a must have shape (1 or %d, 4), got leading shape %s" % (n, tuple(al)))
        ns = int(al[0])
        if tuple(bl) != (ns,):
            raise EngineError(-1, "b must have %d rows like a, got leading shape %s" % (ns, tuple(bl)))
        self._same_lead("note_pk", pl, n)
        self._same_lead("enc", el, n)
        g = self._base(base)
        A = self._result(None, (n, 2, 4), Rk)
        B = self._result(None, (n, 2, 4), Rk)
        ok = self._ok_like(Rk, n)
        flags = self._flags(flags, async_)
        failed = self._counter("sender_failed", flags)
        self._check(self._lib.p252_note_sender_decrypt_batch(self._ctx, ap, bp, ns, Rp, pp, ep, n, g.ctypes.data,
                                                             self._ptr(A), self._ptr(B), self._ptr(ok),
                                                             ctypes.byref(failed), flags))
        return A, B, ok

    def last_elgamal_invalid(self):
        """Invalid items of the last elgamal_encrypt_batch, elgamal_decrypt_batch or note_sender_encrypt_batch (sync()
        first after async_)."""
        return self._last("elgamal_invalid")

    def last_sender_failed(self):
        """Items of the last note_sender_decrypt_batch with ok == 0, not owned or invalid (sync() first after async_)."""
        return self._last("sender_failed")

    # -- multi-key wallet scans ---------------------------------------------------------------------
    WALLET_MAX_KEYS = 256

    def wallet_scan_batch(self, a, b, R, note_pk, pos, nonce, cipher, commitment, base, base_p, async_=False):
        """Which of k keys owns each of n notes, and for owned notes their nullifier, checked opening and per-key totals.
        a and b (k, 4) p252_jscalar rows (1 <= k <= WALLET_MAX_KEYS; key j is (a_j, B_j = [b_j] base)), R and note_pk
        (n, 2, 4), pos (n,) (a numpy uint64 array or a CUDA int64 tensor), nonce (n, 4), cipher (n, 3, 4), commitment
        (n, 2, 4), base (G) and base_p (G') (2, 4) host-read -> (owner (n,) int32, nullifier (n, 4), value (n,), blinder
        (n, 4), opened (n,) uint8, key_totals (k, 4)).  owner[i] is the smallest j whose key owns note i (-1: none);
        nullifier, value, blinder and opened are nullifier_batch's and note_open_batch's rows under that key (zeroed for a
        note no key owns; value and blinder also for an owned note that does not open).  key_totals[j] = (value_lo,
        value_hi, n_owned, n_opened): the 128-bit sum of the opened values key j owns, and its counts.  Counts:
        last_wallet_invalid() (notes with R not a curve point or a note_pk coordinate >= p) and last_wallet_bad_keys()
        (a or b >= r_J).  A base off the curve raises InvalidPoint."""
        Rp, Rl, flags, Rk = self._in(R, (2, 4))
        if len(Rl) != 1:
            raise EngineError(-1, "R must have shape (n, 2, 4)")
        n = int(Rl[0])
        ap, al, fa, ak = self._in(a, (4,))
        bp, bl, fb, bk = self._in(b, (4,))
        pkp, pkl, fpk, pkk = self._in(note_pk, (2, 4))
        np_, nl, fn, nk = self._in(nonce, (4,))
        cp, cl, fc, ck = self._in(cipher, (3, 4))
        Cp, Cl, fC, Ck = self._in(commitment, (2, 4))
        self._same_space(flags, fa, fb, fpk, fn, fc, fC, _native.MEM_DEVICE if _is_torch(pos) else _native.MEM_HOST)
        if len(al) != 1 or not 1 <= int(al[0]) <= self.WALLET_MAX_KEYS:
            raise EngineError(-1, "a must have shape (k, 4) with 1 <= k <= %d, got leading shape %s"
                              % (self.WALLET_MAX_KEYS, tuple(al)))
        k = int(al[0])
        self._same_lead("b", bl, k)
        for name, lead in (("note_pk", pkl), ("nonce", nl), ("cipher", cl), ("commitment", Cl)):
            self._same_lead(name, lead, n)
        pp, npos, pk = self._idx(pos, Rk, "pos")
        if npos != n:
            raise EngineError(-1, "pos must have %d entries, got %d" % (n, npos))
        g, gp = self._base(base), self._base(base_p)
        if _is_torch(Rk):
            import torch
            owner = torch.empty((n,), dtype=torch.int32, device=Rk.device)
        else:
            owner = np.empty((n,), dtype=np.int32)
        nul = self._result(None, (n, 4), Rk)
        value = self._result(None, (n,), Rk)
        blinder = self._result(None, (n, 4), Rk)
        opened = self._ok_like(Rk, n)
        if _is_torch(Rk):
            totals = torch.zeros((k, 4), dtype=Rk.dtype, device=Rk.device)    # n == 0 writes nothing
        else:
            totals = np.zeros((k, 4), dtype=np.uint64)
        flags = self._flags(flags, async_)
        invalid, bad = self._counter("wallet_invalid", flags), self._counter("wallet_bad_keys", flags)
        self._check(self._lib.p252_wallet_scan_batch(self._ctx, ap, bp, k, Rp, pkp, pp, np_, cp, Cp, n, g.ctypes.data,
                                                     gp.ctypes.data, self._ptr(owner), self._ptr(nul), self._ptr(value),
                                                     self._ptr(blinder), self._ptr(opened), self._ptr(totals),
                                                     ctypes.byref(invalid), ctypes.byref(bad), flags))
        return owner, nul, value, blinder, opened, totals

    def last_wallet_invalid(self):
        """Invalid notes of the last wallet_scan_batch (sync() first after async_)."""
        return self._last("wallet_invalid")

    def last_wallet_bad_keys(self):
        """Bad keys of the last wallet_scan_batch (sync() first after async_)."""
        return self._last("wallet_bad_keys")

    # -- point compression ------------------------------------------------------------------------
    def points_from_bytes(self, data, out=None, async_=False):
        """JubJubAffine::from_bytes over a batch: (n, 32) uint8 encodings (host) or (n, 4) 64-bit device tensor of the
        same bytes -> (points (n, 2, 4) BlsScalar.0 limbs, ok (n,) uint8).  An encoding whose v is >= p or whose u^2 is
        not a square has ok == 0 and the row (0, 0) (count: last_points_invalid())."""
        if _is_torch(data):
            ptr, lead, flags, keep = self._in(data, (4,))
            if len(lead) != 1:
                raise EngineError(-1, "device bytes must have shape (n, 4)")
            n = int(lead[0])
        else:
            keep = np.ascontiguousarray(data, dtype=np.uint8)
            if keep.ndim != 2 or keep.shape[1] != 32:
                raise EngineError(-1, "host bytes must have shape (n, 32), got %s" % (keep.shape,))
            ptr, n, flags = keep.ctypes.data, int(keep.shape[0]), _native.MEM_HOST
        res = self._result(out, (n, 2, 4), keep)
        ok = self._ok_like(keep, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("points_invalid", flags)
        self._check(self._lib.p252_points_from_bytes(self._ctx, ptr, n, self._ptr(res), self._ptr(ok),
                                                     ctypes.byref(invalid), flags))
        return res, ok

    def points_to_bytes(self, points, async_=False):
        """JubJubAffine::to_bytes over a batch: points (n, 2, 4) BlsScalar.0 limbs -> (bytes, ok (n,) uint8), bytes
        (n, 32) uint8 (host) or an (n, 4) device tensor of the same bytes.  A point with a coordinate >= p or off the curve
        has ok == 0 and 32 bytes of 0xff, which from_bytes rejects (count: last_points_invalid())."""
        pp, pl, flags, pk = self._in(points, (2, 4))
        if len(pl) != 1:
            raise EngineError(-1, "points must have shape (n, 2, 4)")
        n = int(pl[0])
        res = self._out_like(pk, (n, 4)) if _is_torch(pk) else np.empty((n, 32), dtype=np.uint8)
        ok = self._ok_like(pk, n)
        flags = self._flags(flags, async_)
        invalid = self._counter("points_invalid", flags)
        self._check(self._lib.p252_points_to_bytes(self._ctx, pp, n, self._ptr(res), self._ptr(ok),
                                                   ctypes.byref(invalid), flags))
        return res, ok

    def last_points_invalid(self):
        """Invalid items of the last points_from_bytes or points_to_bytes (sync() first after async_)."""
        return self._last("points_invalid")

    # -- multi-scalar multiplication and all-or-nothing Schnorr verification -----------------------------------------
    def jubjub_msm(self, scalars, points, out=None, async_=False):
        """sum [scalars[i]] points[i] by the bucket method: scalars (n, 4) p252_jscalar rows, points (n, 2, 4) BlsScalar.0
        limbs -> the sum (2, 4), affine (the identity (0, 1) for n == 0).  VARIABLE TIME: for public scalars only.  An
        item with a scalar >= r_J, a coordinate >= p or a point off the curve is skipped (count: last_msm_invalid())."""
        sp, sl, flags, sk = self._in(scalars, (4,))
        if len(sl) != 1:
            raise EngineError(-1, "scalars must have shape (n, 4)")
        n = int(sl[0])
        pp, pl, fp, pk = self._in(points, (2, 4))
        self._same_space(flags, fp)
        self._same_lead("points", pl, n)
        res = self._result(out, (2, 4), sk)
        flags = self._flags(flags, async_)
        invalid = self._counter("msm_invalid", flags)
        self._check(self._lib.p252_jubjub_msm(self._ctx, sp, pp, n, self._ptr(res), ctypes.byref(invalid), flags))
        return res

    def last_msm_invalid(self):
        """Skipped items of the last jubjub_msm (sync() first after async_)."""
        return self._last("msm_invalid")

    def schnorr_verify_all(self, pk, u, R, msg, base, weights=None, async_=False):
        """All-or-nothing verification of n signatures by one random linear combination: True iff no item is invalid,
        every R is on the curve and [8] ([sum z u] base + sum [z c] PK - sum [z] R) is the identity, c = challenge(R, msg).
        Except with probability ~2^-128 that is every item passing the cofactored check [8] ([u] G + [c] PK - R) == O
        (for subgroup keys and R, per-item verification).  pk (1 or n, 2, 4), u (n, 4) p252_jscalar rows, R (n, 2, 4),
        msg (n, 4), base (2, 4) (host-read); weights (n, 4) p252_jscalar rows in the memory space of u, or None for fresh
        128-bit weights from `secrets`.  Invalid items (as in schnorr_verify_batch, or a weight >= r_J) are counted in
        last_schnorr_invalid().  VARIABLE TIME (public data only).  async_: returns None; last_verify_all() after sync()."""
        up, ul, flags, uk = self._in(u, (4,))
        if len(ul) != 1:
            raise EngineError(-1, "u must have shape (n, 4)")
        n = int(ul[0])
        if weights is None:
            weights = _random_weights(n, uk)
        pp, pl, fp, pkk = self._in(pk, (2, 4))
        Rp, Rl, fR, Rk = self._in(R, (2, 4))
        mp, ml, fm, mk = self._in(msg, (4,))
        wp, wl, fw, wk = self._in(weights, (4,))
        self._same_space(flags, fp, fR, fm, fw)
        if len(pl) != 1 or int(pl[0]) not in (1, n):
            raise EngineError(-1, "pk must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(pl)))
        self._same_lead("R", Rl, n)
        self._same_lead("msg", ml, n)
        self._same_lead("weights", wl, n)
        b = self._base(base)
        flags = self._flags(flags, async_)
        invalid = self._counter("schnorr_invalid", flags)
        answer = self._counters["verify_all"] = ctypes.c_uint8(0)
        if flags & _native.ASYNC:
            self._keep_until_sync(answer)
            self._keep_until_sync(wk)
        self._check(self._lib.p252_schnorr_verify_all(self._ctx, pp, int(pl[0]), up, Rp, mp, wp, n, b.ctypes.data,
                                                      ctypes.byref(answer), ctypes.byref(invalid), flags))
        return None if flags & _native.ASYNC else bool(answer.value)

    def last_verify_all(self):
        """The answer of the last schnorr_verify_all (sync() first after async_)."""
        return bool(self._last("verify_all"))

    def schnorr_verify_double_all(self, pk, pk_p, u, R, R_p, msg, base, base_p, weights=None, weights_p=None,
                                  async_=False):
        """All-or-nothing verification of n double-key signatures by one random linear combination: True iff no item is
        invalid, every R and R' is on the curve and [8] ([sum z u] base + [sum z' u] base_p + sum [z c] PK
        + sum [z' c] PK' - sum [z] R - sum [z'] R') is the identity, c = challenge2(R, R', msg).  Except with probability
        ~2^-128 that is every item passing both cofactored checks of schnorr_verify_double_batch.  Arguments as for
        schnorr_verify_double_batch; weights and weights_p (n, 4) p252_jscalar rows in the memory space of u, or None for
        fresh 128-bit weights from `secrets`, one array per equation (the two must be independent: equal weights check
        only the sum of an item's two equations).  Invalid items (as in schnorr_verify_double_batch, or a weight >= r_J)
        are counted once in last_schnorr_double_invalid().  VARIABLE TIME (public data only).  async_: returns None;
        last_verify_double_all() after sync()."""
        up, ul, flags, uk = self._in(u, (4,))
        if len(ul) != 1:
            raise EngineError(-1, "u must have shape (n, 4)")
        n = int(ul[0])
        if weights is None:
            weights = _random_weights(n, uk)
        if weights_p is None:
            weights_p = _random_weights(n, uk)
        pp, pl, fp, _ = self._in(pk, (2, 4))
        qp, ql, fq, _ = self._in(pk_p, (2, 4))
        Rp, Rl, fR, _ = self._in(R, (2, 4))
        Sp, Sl, fS, _ = self._in(R_p, (2, 4))
        mp, ml, fm, _ = self._in(msg, (4,))
        wp, wl, fw, wk = self._in(weights, (4,))
        vp, vl, fv, vk = self._in(weights_p, (4,))
        self._same_space(flags, fp, fq, fR, fS, fm, fw, fv)
        if len(pl) != 1 or int(pl[0]) not in (1, n):
            raise EngineError(-1, "pk must have shape (1 or %d, 2, 4), got leading shape %s" % (n, tuple(pl)))
        if tuple(ql) != tuple(pl):
            raise EngineError(-1, "pk_p must have %d rows like pk, got leading shape %s" % (int(pl[0]), tuple(ql)))
        self._same_lead("R", Rl, n)
        self._same_lead("R_p", Sl, n)
        self._same_lead("msg", ml, n)
        self._same_lead("weights", wl, n)
        self._same_lead("weights_p", vl, n)
        g, gp = self._base(base), self._base(base_p)
        flags = self._flags(flags, async_)
        invalid = self._counter("schnorr_double_invalid", flags)
        answer = self._counters["verify_double_all"] = ctypes.c_uint8(0)
        if flags & _native.ASYNC:
            self._keep_until_sync(answer)
            self._keep_until_sync(wk)
            self._keep_until_sync(vk)
        self._check(self._lib.p252_schnorr_verify_double_all(self._ctx, pp, qp, int(pl[0]), up, Rp, Sp, mp, wp, vp, n,
                                                             g.ctypes.data, gp.ctypes.data, ctypes.byref(answer),
                                                             ctypes.byref(invalid), flags))
        return None if flags & _native.ASYNC else bool(answer.value)

    def last_verify_double_all(self):
        """The answer of the last schnorr_verify_double_all (sync() first after async_)."""
        return bool(self._last("verify_double_all"))

    def _crypt_varlen_args(self, data, offsets, secrets_uv, nonces, max_len, key_extra):
        """Shared validation of encrypt_batch_varlen / decrypt_batch_varlen -> (data ptr, n_scalars, offsets ptr, n,
        max_len, secrets ptr, nonces ptr, flags, data keepalive, offsets keepalive, secrets and nonces keepalives).
        key_extra: scalars an item carries beyond its message (0 for messages, 1 for ciphers)."""
        dp, dlead, flags, dk = self._in(data, (4,))
        if len(dlead) != 1:
            raise EngineError(-1, "data must have shape (n_scalars, 4), got leading shape %s" % (tuple(dlead),))
        op, n1, ok_ = self._idx(offsets, dk, "offsets")
        if n1 < 1:
            raise EngineError(-1, "offsets must have n + 1 >= 1 entries")
        n = n1 - 1
        sp, l2, f2, sk = self._in(secrets_uv, (2, 4))
        np_, l3, f3, nk = self._in(nonces, (4,))
        self._same_space(flags, f2, f3)
        self._same_lead("secrets_uv", l2, n)
        self._same_lead("nonces", l3, n)
        if max_len is None:
            max_len = self._longest_item(ok_, n, key_extra)
        return dp, int(dlead[0]), op, n, int(max_len), sp, np_, flags, dk, ok_, (sk, nk)

    def encrypt_batch_varlen(self, data, offsets, secrets_uv, nonces, max_len=None, out=None, async_=False):
        """n x encrypt(data[offsets[i]:offsets[i+1]], secrets_uv[i], nonces[i]) over messages of any lengths, one call.
        data (n_scalars, 4), offsets (n + 1,), secrets_uv (n, 2, 4) and nonces (n, 4) live in one memory space (numpy, or
        CUDA tensors); offsets[0] need not be 0.  Returns (cipher, cipher_offsets): cipher item i is
        cipher[cipher_offsets[i]:cipher_offsets[i+1]] (len + 1 scalars), packed from 0; cipher has n_scalars + n rows, of
        which those past cipher_offsets[-1] are unused (offsets covering only part of data).  cipher_offsets
        (= cipher_offsets(offsets)) is computed in the offsets' memory space.  max_len bounds the message lengths (at most
        VARLEN_MAX_LEN); None takes the longest, which for CUDA tensors costs a device-to-host sync.  Host batches raise on
        an invalid item and write nothing; device batches skip invalid items, write nothing for them and count them
        (last_crypt_rejected())."""
        dp, ns, op, n, max_len, sp, np_, flags, dk, ok_, keep = self._crypt_varlen_args(data, offsets, secrets_uv, nonces,
                                                                                         max_len, 0)
        rows = ns + n
        res = self._rows_like(dk, rows) if out is None else self._check_out(out, (rows, 4), dk)
        flags = self._flags(flags, async_)
        rejected = self._counter("crypt_rejected", flags)
        self._check(self._lib.p252_encrypt_batch_varlen(self._ctx, dp, ns, op, n, max_len, sp, np_, self._ptr(res),
                                                        ctypes.byref(rejected), flags))
        return res, varlen_out_offsets(ok_, 1)

    def decrypt_batch_varlen(self, ciphers, offsets, secrets_uv, nonces, max_len=None, async_=False):
        """n x decrypt(ciphers[offsets[i]:offsets[i+1]], secrets_uv[i], nonces[i]) over ciphers of any lengths, one call.
        Buffers as for encrypt_batch_varlen; max_len bounds the message lengths (cipher length - 1).  Returns
        (msg, msg_offsets, ok): message item i is msg[msg_offsets[i]:msg_offsets[i+1]] (one scalar shorter than its
        cipher), packed from 0 in max(n_scalars - n, 0) rows; ok[i] == 0 where the reference returns
        Error::DecryptionFailed (that message is zeroed) or, for device buffers, the item was invalid and skipped.  Failure
        count: last_decrypt_failures(); invalid device items: last_crypt_rejected()."""
        cp, ns, op, n, max_len, sp, np_, flags, ck, ok_, keep = self._crypt_varlen_args(ciphers, offsets, secrets_uv,
                                                                                         nonces, max_len, 1)
        msg = self._rows_like(ck, max(ns - n, 0))
        ok = self._ok_like(ck, n)
        flags = self._flags(flags, async_)
        failed, rejected = self._counter("decrypt_failures", flags), self._counter("crypt_rejected", flags)
        self._check(self._lib.p252_decrypt_batch_varlen(self._ctx, cp, ns, op, n, max_len, sp, np_, self._ptr(msg),
                                                        self._ptr(ok), ctypes.byref(failed), ctypes.byref(rejected), flags))
        return msg, varlen_out_offsets(ok_, -1), ok

    def last_crypt_rejected(self):
        """Items of the last encrypt_batch_varlen / decrypt_batch_varlen skipped as invalid (device buffers; sync() first
        after async_)."""
        return self._last("crypt_rejected")

    # -- arity-4 Merkle tree ----------------------------------------------------------------------
    def merkle4_level(self, children, out=None, async_=False):
        """children (4*m, 4) -> parents (m, 4)."""
        cp, lead, flags, ck = self._in(children, (4,))
        m = lead[0] // 4
        if lead[0] % 4:
            from .errors import IOPatternViolation
            raise IOPatternViolation()
        res = self._result(out, (m, 4), ck)
        self._check(self._lib.p252_merkle4_level(self._ctx, cp, m, self._ptr(res), self._flags(flags, async_)))
        return res

    def tree_nodes(self, n_leaves):
        ni, nl = ctypes.c_size_t(0), ctypes.c_int(0)
        self._check(self._lib.p252_merkle4_tree_nodes(int(n_leaves), ctypes.byref(ni), ctypes.byref(nl)))
        return int(ni.value), int(nl.value)

    def merkle4_build(self, leaves, out=None, async_=False):
        """leaves (4^k, 4) -> all internal nodes bottom-up ((4^k-1)/3, 4); root = last row."""
        lp, lead, flags, lk = self._in(leaves, (4,))
        n_internal, _ = self.tree_nodes(lead[0])
        res = self._result(out, (n_internal, 4), lk)
        self._check(self._lib.p252_merkle4_build(self._ctx, lp, lead[0], self._ptr(res), self._flags(flags, async_)))
        return res

    def merkle_build(self, leaves, arity=4, out=None, async_=False):
        """leaves (arity^k, 4) -> all internal nodes bottom-up, root last; arity 2 (Domain::Merkle2) or 4."""
        lp, lead, flags, lk = self._in(leaves, (4,))
        ni = ctypes.c_size_t(0)
        self._check(self._lib.p252_merkle_tree_nodes(int(arity), lead[0], ctypes.byref(ni), None))
        res = self._result(out, (int(ni.value), 4), lk)
        self._check(self._lib.p252_merkle_build(self._ctx, int(arity), lp, lead[0], self._ptr(res),
                                                self._flags(flags, async_)))
        return res

    # -- Merkle openings --------------------------------------------------------------------------
    def _idx(self, leaf_idx, like, name="leaf_idx"):
        if _is_torch(like):
            if not _is_torch(leaf_idx) or not leaf_idx.is_cuda or leaf_idx.device != like.device or \
                    str(leaf_idx.dtype) not in ("torch.int64", "torch.uint64") or not leaf_idx.is_contiguous() or leaf_idx.dim() != 1:
                raise EngineError(-1, "%s must be a contiguous 1-D int64/uint64 tensor on %s" % (name, like.device))
            return leaf_idx.data_ptr(), int(leaf_idx.shape[0]), leaf_idx
        a = np.ascontiguousarray(leaf_idx, dtype=np.uint64).reshape(-1)
        return a.ctypes.data, int(a.shape[0]), a

    def merkle_open_batch(self, leaves, nodes, leaf_idx, arity=4, out=None, async_=False):
        """Openings of the leaves `leaf_idx` of the tree (leaves (arity^d, 4), nodes as returned by merkle_build):
        (n, d, arity, 4) -- for every level the whole sibling group of the path node (poseidon-merkle `Opening`)."""
        lp, lead, flags, lk = self._in(leaves, (4,))
        np_, nlead, f2, nk = self._in(nodes, (4,))
        self._same_space(flags, f2)
        ni, nl = ctypes.c_size_t(0), ctypes.c_int(0)
        self._check(self._lib.p252_merkle_tree_nodes(int(arity), lead[0], ctypes.byref(ni), ctypes.byref(nl)))
        self._same_lead("nodes", nlead, int(ni.value))
        ip, n, ik = self._idx(leaf_idx, lk)
        res = self._result(out, (n, int(nl.value), int(arity), 4), lk)
        self._check(self._lib.p252_merkle_open_batch(self._ctx, int(arity), lp, lead[0], np_, ip, n, self._ptr(res),
                                                     self._flags(flags, async_)))
        return res

    def merkle_verify_batch(self, leaf_items, leaf_idx, paths, root, arity=4, async_=False):
        """n x Opening::verify.  leaf_items (n, 4), leaf_idx (n,), paths (n, d, arity, 4), root (4,) host array
        -> ok (n,) uint8.  The failure count is available from last_verify_failures()."""
        if paths.ndim != 4 or int(paths.shape[2]) != int(arity):
            raise EngineError(-1, "paths must have shape (n, depth, arity, 4)")
        depth = int(paths.shape[1])
        pp, plead, flags, pk = self._in(paths, (depth, int(arity), 4))
        n = plead[0]
        lp, llead, f2, lk = self._in(leaf_items, (4,))
        self._same_space(flags, f2)
        self._same_lead("leaf_items", llead, n)
        ip, ni, ik = self._idx(leaf_idx, pk)
        if ni != n:
            raise EngineError(-1, "leaf_idx must have %d entries" % n)
        root = self._host_limbs(root, (4,), "root must be one scalar")
        ok = self._ok_like(pk, n)
        flags = self._flags(flags, async_)
        failed = self._counter("verify_failures", flags)
        self._check(self._lib.p252_merkle_verify_batch(self._ctx, int(arity), depth, lp, ip, pp, root.ctypes.data, n,
                                                       self._ptr(ok), ctypes.byref(failed), flags))
        return ok

    def last_verify_failures(self):
        return self._last("verify_failures")

    def _open_batch(self, describe, fn, tree, idx, name, out, async_):
        """The openings of a tree with a descriptor: `describe` is _mtree, _smtree or _ctree, fn its open_batch call."""
        t, flags, keep = describe(tree)
        ip, n, ik = self._idx(idx, keep[0], name)
        res = self._result(out, (n, int(tree.height), int(tree.arity), 4), keep[0])
        self._check(fn(self._ctx, ctypes.byref(t), ip, n, self._ptr(res), self._flags(flags, async_)))
        return res

    # -- fixed-height trees with batched updates (p252_mtree) ------------------------------------------
    def mtree_layout(self, arity, height, capacity):
        return mtree_layout(arity, height, capacity)

    def _tree_buffers(self, tree):
        """The leaves (leaf_slots, 4) and nodes (node_slots, 4) of a p252_mtree / p252_smtree -> (leaf pointer, node
        pointer, flags, leaves, nodes, leaf_slots + node_slots).  The library writes through them, so host buffers must
        be the caller's own arrays: a converted copy would take the update and be dropped."""
        leaf_slots, node_slots, _ = self.mtree_layout(tree.arity, tree.height, tree.capacity)
        lp, llead, flags, lk = self._in(tree.leaves, (4,))
        np_, nlead, f2, nk = self._in(tree.nodes, (4,))
        self._same_space(flags, f2)
        self._same_lead("leaves", llead, leaf_slots)
        self._same_lead("nodes", nlead, node_slots)
        if not _is_torch(lk) and (lk is not tree.leaves or nk is not tree.nodes or not lk.flags.writeable or not nk.flags.writeable):
            raise EngineError(-1, "host tree buffers must be writable C-contiguous uint64 arrays")
        return lp, np_, flags, lk, nk, leaf_slots + node_slots

    def _mtree(self, tree):
        """tree: anything with arity / height / capacity / n_leaves / leaves (leaf_slots, 4) / nodes (node_slots, 4)
        -> (p252_mtree, flags, keepalive)."""
        lp, np_, flags, lk, nk, _ = self._tree_buffers(tree)
        t = _native.MTree(ctypes.sizeof(_native.MTree), int(tree.arity), int(tree.height), 0, int(tree.capacity),
                          int(tree.n_leaves), lp, np_)
        return t, flags, (lk, nk)

    def mtree_build(self, tree, async_=False):
        """Rebuild every node of `tree` from its occupied leaf prefix."""
        t, flags, keep = self._mtree(tree)
        self._check(self._lib.p252_mtree_build(self._ctx, ctypes.byref(t), self._flags(flags, async_)))

    def mtree_update(self, tree, idx=None, values=None, append=None, async_=False):
        """Overwrite leaves idx[i] with values[i] (n, 4) -- the last write to a leaf wins -- and append the rows of
        `append` (k, 4); only the touched paths are rehashed.  tree.n_leaves advances by k.  Device indices
        >= n_leaves are skipped and counted (last_update_rejected()); host ones raise."""
        t, flags, keep = self._mtree(tree)
        ip = vp = ap = None
        n_upd = n_app = 0
        like = keep[0]
        if idx is not None or values is not None:
            ip, n_upd, ik = self._idx(idx, like)
            vp, vlead, fv, vk = self._in(values, (4,))
            self._same_space(flags, fv)
            self._same_lead("values", vlead, n_upd)
        if append is not None:
            ap, alead, fa, ak = self._in(append, (4,))
            self._same_space(flags, fa)
            n_app = int(alead[0])
        flags = self._flags(flags, async_)
        rejected = self._counter("update_rejected", flags)
        self._check(self._lib.p252_mtree_update(self._ctx, ctypes.byref(t), ip if n_upd else None, vp if n_upd else None,
                                                n_upd, ap if n_app else None, n_app, ctypes.byref(rejected), flags))
        tree.n_leaves = int(t.n_leaves)
        return tree.n_leaves

    def last_update_rejected(self):
        """Updates of the last mtree_update skipped for an index >= n_leaves (device buffers; sync() first after async_)."""
        return self._last("update_rejected")

    def mtree_open_batch(self, tree, leaf_idx, out=None, async_=False):
        """Openings of leaves `leaf_idx`: (n, height, arity, 4), zero slots beyond each level's prefix; they verify with
        merkle_verify_batch (depth = height)."""
        return self._open_batch(self._mtree, self._lib.p252_mtree_open_batch, tree, leaf_idx, "leaf_idx", out, async_)

    # -- sparse fixed-height trees: inserts and removals at any position (p252_smtree) -----------------------------
    def _bytes(self, x, like, name, n, writable=False):
        """A 1-D uint8 buffer of n entries in the memory space of `like` -> (pointer, keepalive).  writable: the library
        writes through it, so a host buffer must be the caller's own C-contiguous array (no copy is made)."""
        if _is_torch(like):
            if not _is_torch(x) or not x.is_cuda or x.device != like.device or str(x.dtype) != "torch.uint8" or \
                    not x.is_contiguous() or tuple(x.shape) != (n,):
                raise EngineError(-1, "%s must be a contiguous uint8 tensor of shape (%d,) on %s" % (name, n, like.device))
            return x.data_ptr(), x
        if writable:
            if not isinstance(x, np.ndarray) or x.dtype != np.uint8 or tuple(x.shape) != (n,) or not x.flags.c_contiguous \
                    or not x.flags.writeable:
                raise EngineError(-1, "%s must be a writable C-contiguous uint8 array of shape (%d,)" % (name, n))
            return x.ctypes.data, x
        if _is_torch(x):
            raise EngineError(-1, "%s must be a host array like the tree's buffers" % name)
        a = np.ascontiguousarray(x, dtype=np.uint8).reshape(-1)
        if a.shape != (n,):
            raise EngineError(-1, "%s must have %d entries" % (name, n))
        return a.ctypes.data, a

    def _smtree(self, tree):
        """tree: anything with arity / height / capacity / leaves (leaf_slots, 4) / nodes (node_slots, 4) / present
        (leaf_slots + node_slots,) uint8 -> (p252_smtree, flags, keepalive)."""
        lp, np_, flags, lk, nk, slots = self._tree_buffers(tree)
        pp, pk = self._bytes(tree.present, lk, "present", slots, writable=True)
        t = _native.SMTree(ctypes.sizeof(_native.SMTree), int(tree.arity), int(tree.height), 0, int(tree.capacity), lp, np_, pp)
        return t, flags, (lk, nk, pk)

    def smtree_build(self, tree, async_=False):
        """Rebuild every node (and node presence byte) of the sparse tree from its leaves and leaf presence bytes; absent
        leaves are zeroed.  Only present nodes are hashed."""
        t, flags, keep = self._smtree(tree)
        self._check(self._lib.p252_smtree_build(self._ctx, ctypes.byref(t), self._flags(flags, async_)))

    def _sparse_update(self, describe, fn, counter, tree, pos, values, op, async_):
        """One batch of inserts and removals on a sparse tree: `describe` is _smtree or _ctree, fn its update call and
        `counter` the name its rejected items are counted under."""
        t, flags, keep = describe(tree)
        like = keep[0]
        ip, n, ik = self._idx(pos, like, "pos")
        if values is None:
            values = self._out_like(like, (n, 4))
            values[:] = 0
            if async_ and flags:
                self._keep_until_sync(values)      # read by the device after this call returns
        vp, vlead, fv, vk = self._in(values, (4,))
        self._same_space(flags, fv)
        self._same_lead("values", vlead, n)
        opp, ok_ = (None, None) if op is None else self._bytes(op, like, "op", n)
        flags = self._flags(flags, async_)
        rejected = self._counter(counter, flags)
        self._check(fn(self._ctx, ctypes.byref(t), ip if n else None, opp if n else None, vp if n else None, n,
                       ctypes.byref(rejected), flags))

    def smtree_update(self, tree, pos, values=None, op=None, async_=False):
        """One batch of operations on a sparse tree: op[i] = 0 inserts / overwrites values[i] at pos[i], op[i] = 1 removes
        pos[i] (op None: all inserts; values None: all zeros, for a batch of removals).  Equal to applying them in batch
        order.  Device items with pos >= capacity or an op other than 0/1 are skipped and counted
        (last_smtree_rejected()); host ones raise."""
        self._sparse_update(self._smtree, self._lib.p252_smtree_update, "smtree_rejected", tree, pos, values, op, async_)

    def last_smtree_rejected(self):
        """Items of the last smtree_update skipped on the device (pos >= capacity or op not 0/1; sync() first after
        async_)."""
        return self._last("smtree_rejected")

    def smtree_len(self, tree):
        """Number of present positions (counted on the device for device buffers)."""
        t, flags, keep = self._smtree(tree)
        c = ctypes.c_uint64(0)
        self._check(self._lib.p252_smtree_len(self._ctx, ctypes.byref(t), ctypes.byref(c), flags))
        return int(c.value)

    def smtree_open_batch(self, tree, pos, out=None, async_=False):
        """Openings of the present positions `pos`: (n, height, arity, 4), absent slots zero; they verify with
        merkle_verify_batch (depth = height).  Host: an absent position raises; device: it gets an all-zero opening."""
        return self._open_batch(self._smtree, self._lib.p252_smtree_open_batch, tree, pos, "pos", out, async_)

    # -- compact sparse trees: sorted present nodes per level (p252_ctree) --------------------------------------------
    def ctree_layout(self, arity, height, max_leaves):
        return ctree_layout(arity, height, max_leaves)

    def _words(self, x, like, name, n):
        """The caller's own writable 1-D buffer of n 64-bit words in the memory space of `like` -> pointer (no copy)."""
        if _is_torch(like):
            if not _is_torch(x) or not x.is_cuda or x.device != like.device or \
                    str(x.dtype) not in ("torch.int64", "torch.uint64") or not x.is_contiguous() or tuple(x.shape) != (n,):
                raise EngineError(-1, "%s must be a contiguous int64/uint64 tensor of shape (%d,) on %s" % (name, n, like.device))
            return x.data_ptr()
        if not isinstance(x, np.ndarray) or x.dtype != np.uint64 or tuple(x.shape) != (n,) or not x.flags.c_contiguous \
                or not x.flags.writeable:
            raise EngineError(-1, "%s must be a writable C-contiguous uint64 array of shape (%d,)" % (name, n))
        return x.ctypes.data

    def _ctree(self, tree):
        """tree: anything with arity / height / max_leaves / keys (total_slots,) / values (total_slots, 4) / count
        (height + 1,) -> (p252_ctree, flags, keepalive)."""
        total, _ = self.ctree_layout(tree.arity, tree.height, tree.max_leaves)
        vp, vlead, flags, vk = self._in(tree.values, (4,))
        self._same_lead("values", vlead, total)
        if not _is_torch(vk) and (vk is not tree.values or not vk.flags.writeable):
            raise EngineError(-1, "host tree buffers must be writable C-contiguous uint64 arrays")
        kp = self._words(tree.keys, vk, "keys", total)
        cp = self._words(tree.count, vk, "count", int(tree.height) + 1)
        t = _native.CTree(ctypes.sizeof(_native.CTree), int(tree.arity), int(tree.height), 0, int(tree.max_leaves), kp, vp, cp)
        return t, flags, (vk, tree.keys, tree.count)

    def ctree_update(self, tree, pos, values=None, op=None, async_=False):
        """One batch of operations on a compact sparse tree: op[i] = 0 inserts / overwrites values[i] at pos[i], op[i] = 1
        removes pos[i] (op None: all inserts; values None: all zeros, for a batch of removals).  Equal to applying them
        in batch order.  Device items with pos >= arity^height or an op other than 0/1 are skipped and counted
        (last_ctree_rejected()); a device batch that would leave more than max_leaves present positions changes nothing
        and counts every item as rejected.  Host: either raises and changes nothing."""
        self._sparse_update(self._ctree, self._lib.p252_ctree_update, "ctree_rejected", tree, pos, values, op, async_)

    def last_ctree_rejected(self):
        """Items of the last ctree_update skipped on the device (pos >= arity^height or op not 0/1; all of them when the
        batch would exceed max_leaves; sync() first after async_)."""
        return self._last("ctree_rejected")

    def ctree_open_batch(self, tree, pos, out=None, async_=False):
        """Openings of the present positions `pos`: (n, height, arity, 4), absent slots zero; they verify with
        merkle_verify_batch (depth = height).  Host: an absent position raises; device: it gets an all-zero opening."""
        return self._open_batch(self._ctree, self._lib.p252_ctree_open_batch, tree, pos, "pos", out, async_)

    def set_small_batch_max(self, max_items):
        """Digest batches up to `max_items` items use the lane-split (5 threads per state) kernel; 0 disables it."""
        self._check(self._lib.p252_set_small_batch_max(self._ctx, int(max_items)))

    # -- introspection ----------------------------------------------------------------------------
    def kernel_info(self):
        """p252_get_kernel_info as a dict (multiplier / DFMA instructions per permutation, launch shape)."""
        info = _native.KernelInfo()
        info.struct_size = ctypes.sizeof(info)
        self._check(self._lib.p252_get_kernel_info(ctypes.byref(info)))
        return {k: int(getattr(info, k)) for k, _ in info._fields_ if k != "struct_size"}

    def tree_level_timings(self):
        """Per-level device times of the last merkle4_build_dist(timing=True): (list of dicts, total_ms)."""
        arr = (_native.LevelTiming * 64)()
        n, total = ctypes.c_int(0), ctypes.c_float(0)
        self._check(self._lib.p252_tree_level_timings(self._ctx, arr, 64, ctypes.byref(n), ctypes.byref(total)))
        return [{k: (float(getattr(arr[i], k)) if k.endswith("_ms") else int(getattr(arr[i], k))) for k, _ in arr[i]._fields_}
                for i in range(n.value)], float(total.value)

    # -- multi-GPU (one process per GPU) ----------------------------------------------------------
    def dist_unique_id(self):
        buf = (ctypes.c_uint8 * _native.NCCL_UNIQUE_ID_BYTES)()
        self._check(self._lib.p252_dist_unique_id(buf))
        return bytes(buf)

    def dist_init(self, unique_id, rank, nranks):
        buf = (ctypes.c_uint8 * _native.NCCL_UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        self._check(self._lib.p252_dist_init(self._ctx, buf, int(rank), int(nranks)))
        self._dist = True

    def dist_finalize(self):
        if self._dist:
            self._check(self._lib.p252_dist_finalize(self._ctx))
            self._dist = False

    def merkle4_build_dist(self, leaves_shard, n_leaves_total, out=None, async_=False, timing=False, no_gather=False):
        """This rank's contiguous shard of the leaves (device tensor) -> complete internal levels
        on every rank (one NCCL all-gather per level)."""
        lp, lead, flags, lk = self._in(leaves_shard, (4,))
        if flags != _native.MEM_DEVICE:
            raise EngineError(-1, "merkle4_build_dist takes device tensors")
        n_internal, _ = self.tree_nodes(n_leaves_total)
        res = self._result(out, (n_internal, 4), lk)
        self._check(self._lib.p252_merkle4_build_dist(self._ctx, lp, int(n_leaves_total), self._ptr(res),
                                                      self._flags(flags, async_) |
                                                      (_native.TIMING if timing else 0) | (_native.NO_GATHER if no_gather else 0)))
        return res


def mtree_layout(arity, height, capacity):
    """p252_mtree_layout (host arithmetic, no GPU): -> (leaf_slots, node_slots, level_offset) with level_offset[l] the
    first slot of level l inside the node array (l >= 1; level_offset[0] = 0)."""
    lib = _native.lib()
    ls, ns = ctypes.c_uint64(0), ctypes.c_uint64(0)
    offs = (ctypes.c_uint64 * (min(max(int(height), 0), 64) + 1))()
    raise_for_status(lib.p252_mtree_layout(int(arity), int(height), int(capacity), ctypes.byref(ls), ctypes.byref(ns), offs), lib)
    return int(ls.value), int(ns.value), [int(v) for v in offs]


def ctree_layout(arity, height, max_leaves):
    """p252_ctree_layout (host arithmetic, no GPU): -> (total_slots, level_offset) with level_offset[l] the first slot of
    level l, l = 0..height; level l has min(max_leaves, arity^(height - l)) slots."""
    lib = _native.lib()
    total = ctypes.c_uint64(0)
    offs = (ctypes.c_uint64 * (min(max(int(height), 0), 64) + 1))()
    raise_for_status(lib.p252_ctree_layout(int(arity), int(height), int(max_leaves), ctypes.byref(total), offs), lib)
    return int(total.value), [int(v) for v in offs]


def varlen_out_offsets(offsets, delta):
    """offsets - offsets[0] + delta * i for i = 0..n: the offsets of a CSR batch whose item i is `delta` scalars longer
    (encrypt: +1) or shorter (decrypt: -1) than input item i, packed from 0.  Computed in the offsets' own memory space
    (numpy uint64, or a CUDA tensor of the offsets' dtype, without a host sync).  Pure arithmetic."""
    if _is_torch(offsets):
        import torch
        o = offsets.view(torch.int64)
        r = o - o[:1] + delta * torch.arange(o.shape[0], dtype=torch.int64, device=o.device)
        return r.view(offsets.dtype)
    a = np.ascontiguousarray(offsets, dtype=np.uint64).reshape(-1)
    if a.shape[0] == 0:
        raise EngineError(-1, "offsets must have n + 1 >= 1 entries")
    step = np.arange(a.shape[0], dtype=np.uint64)
    return (a - a[0]) + step if delta > 0 else (a - a[0]) - step     # uint64 arithmetic: wraps like the C ABI's


def default_engine(device=0):
    """Process-wide engine per device (created on first use)."""
    if device not in _DEFAULT:
        _DEFAULT[device] = Engine(device)
    return _DEFAULT[device]


def _engine_for(engine, like=None):
    """The engine a module-level call runs on: the caller's, else the process-wide one of the device the CUDA tensor
    `like` lives on (device 0 for host arrays and for no buffer at all)."""
    return engine or default_engine(like.device.index if hasattr(like, "is_cuda") else 0)
