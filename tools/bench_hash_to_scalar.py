#!/usr/bin/env python
"""Benchmark of batched BlsScalar::hash_to_scalar (p252_hash_to_scalar_batch): BLAKE2b-512 of byte strings, reduced into
the scalar field, one message per device thread.

    python tools/bench_hash_to_scalar.py [--steps K] [--warmup W] [--items N] > hash_to_scalar.json

Workloads of N messages (default 2^20): fixed lengths 32, 128 (both one block: no sort), 200 and 1024 bytes (sorted by
block count), lengths uniform 0..4096, and a heavy tail (lengths uniform 0..200 plus one message of
P252_HASH_TO_SCALAR_MAX_LEN bytes, which one thread hashes alone).  Arms per workload:
  device : data, offsets and output device-resident, one call
  host   : numpy buffers, one call; the library stages the bytes to the device and the rows back, so this includes the
           PCIe copies
  (both: CUDA events on the engine's stream around each of --steps calls after --warmup; the median is reported, with
  the fastest and slowest call)
  loop   : a single-thread loop over the existing host p252_hash_to_scalar through ctypes, once over all N messages
  hashlib: a Python loop of hashlib.blake2b and a big-integer from_bytes_wide, once over all N messages (context only)
Message bytes per second count the message bytes of one call.  In-run parity: the device rows equal the host-call rows
and the ctypes loop's rows on every row, and hashlib's on 4096 sampled rows.  The line carries the device, its power
limit and the SM clocks of the timed region (bench.py's ClockSampler, imported unchanged).  Writes nothing in the
repository tree.
"""
import argparse
import ctypes
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import ClockSampler  # noqa: E402

P = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
R = (1 << 256) % P


def workloads(n, rng, max_len):
    import numpy as np
    tail = rng.integers(0, 201, n)
    tail[n // 2] = max_len
    return {"fixed_32": np.full(n, 32), "fixed_128": np.full(n, 128), "fixed_200": np.full(n, 200),
            "fixed_1024": np.full(n, 1024), "mixed_0_4096": rng.integers(0, 4097, n), "heavy_tail": tail}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--items", type=int, default=1 << 20)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.items < 2:
        ap.error("--steps must be >= 1, --warmup >= 0, --items >= 2")
    import numpy as np
    import torch
    import poseidon252_b200 as pb
    from poseidon252_b200 import _native
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    lib = _native.lib()
    max_len_cap = _native.HASH_TO_SCALAR_MAX_LEN

    def timed(fn, reps):
        """per-call times (ms) between CUDA events recorded around each call"""
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
        with torch.cuda.stream(stream):
            ev[0].record(stream)
            for k in range(reps):
                fn()
                ev[k + 1].record(stream)
        stream.synchronize()
        return [ev[k].elapsed_time(ev[k + 1]) for k in range(reps)]

    def measure(fn, r, arm):
        """the median call time; the spread over the steps goes into r as well"""
        if args.warmup:
            timed(fn, args.warmup)
        t = sorted(timed(fn, args.steps))
        r[arm + "_ms_min"], r[arm + "_ms_max"] = t[0], t[-1]
        return t[len(t) // 2]

    rng = np.random.default_rng(7)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, lens in workloads(args.items, rng, max_len_cap).items():
        n = lens.shape[0]
        offs_h = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        total = int(offs_h[-1])
        max_len = int(lens.max())
        data_h = np.frombuffer(rng.bytes(total), dtype=np.uint8)
        with torch.cuda.stream(stream):
            data_d = torch.from_numpy(data_h.copy()).cuda()
            offs_d = torch.from_numpy(offs_h.view(np.int64)).cuda()
            out_d = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        out_h = np.empty((n, 4), dtype=np.uint64)
        stream.synchronize()

        def device():
            eng.hash_to_scalar_batch(data_d, offs_d, max_len=max_len, out=out_d, async_=True)

        def host():
            eng.hash_to_scalar_batch(data_h, offs_h, max_len=max_len, out=out_h)

        r = {"items": n, "message_bytes": total, "max_len": max_len, "blocks": int(np.maximum(1, (lens + 127) // 128).sum())}
        r["device_ms"] = measure(device, r, "device")
        r["host_ms"] = measure(host, r, "host")
        # the existing host call, one message at a time through ctypes
        loop_out = np.empty((n, 4), dtype=np.uint64)
        f, base, op = lib.p252_hash_to_scalar, data_h.ctypes.data, loop_out.ctypes.data
        starts, ls = offs_h[:-1].tolist(), lens.tolist()
        t0 = time.perf_counter()
        for i in range(n):
            f(base + starts[i], ls[i], op + 32 * i)
        r["loop_ms"] = (time.perf_counter() - t0) * 1e3
        mv = memoryview(data_h)
        t0 = time.perf_counter()
        hl = [int.from_bytes(hashlib.blake2b(mv[starts[i]:starts[i] + ls[i]], digest_size=64).digest(), "little") % P
              for i in range(n)]
        r["hashlib_ms"] = (time.perf_counter() - t0) * 1e3
        for arm in ("device", "host", "loop", "hashlib"):
            r[arm + "_bytes_per_s"] = total / (r[arm + "_ms"] * 1e-3)
        r["device_speedup_over_loop"] = r["loop_ms"] / r["device_ms"]
        r["host_speedup_over_loop"] = r["loop_ms"] / r["host_ms"]
        got = out_d.cpu().numpy().view(np.uint64)
        rows = rng.choice(n, min(n, 4096), replace=False)
        sampled = np.frombuffer(b"".join((hl[i] * R % P).to_bytes(32, "little") for i in rows),
                                dtype=np.uint64).reshape(-1, 4)
        parity[name] = bool(np.array_equal(got, out_h) and np.array_equal(got, loop_out) and
                            np.array_equal(got[rows], sampled))
        res[name] = r
        del data_d, offs_d, out_d, data_h, out_h, loop_out, hl
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "hash_to_scalar_bytes_per_s", "value": res["mixed_0_4096"]["device_bytes_per_s"], "unit": "B/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
            "config": {"workload": "p252_hash_to_scalar_batch, %d messages per call" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
