#!/usr/bin/env python
"""Benchmark of variable-length digest batches (p252_hash_batch_varlen) against the status quo of one p252_hash_batch
per distinct length.

    python tools/bench_varlen.py [--steps K] [--warmup W] [--items N] > varlen.json

Three workloads of N items (default 2^20), Domain::Other, one output scalar, all buffers device-resident:
  (a) every length 4        : one varlen call vs one hash_batch call (the cost of the keys, the sort and the indirection)
  (b) lengths uniform 1..64 : one varlen call vs grouped calls (per length: gather, hash_batch, scatter)
  (c) heavy tail            : lengths uniform 1..16 plus 32 items of length 4096, same two arms as (b)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  perm/s counts
sum(ceil(len/4) + ceil(out_len/4) - 1) permutations per call.  The line also carries the flat Merkle4 rate of the same
run, the device and its power limit, and in-run parity: for every workload the varlen output equals the grouped output
(and, for (a), the hash_batch output).  Writes nothing in the repository tree.  The clock sampler and the device-side
input generator are bench.py's, imported unchanged.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import ClockSampler, device_random_scalars  # noqa: E402


def workloads(n, rng):
    import numpy as np
    tail = rng.integers(1, 17, n)
    tail[rng.choice(n, 32, replace=False)] = 4096
    return {"a_len4": np.full(n, 4), "b_uniform_1_64": rng.integers(1, 65, n), "c_heavy_tail": tail}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--items", type=int, default=1 << 20)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.items < 1:
        ap.error("--steps and --items must be >= 1, --warmup >= 0")
    import numpy as np
    import torch
    import poseidon252_b200 as pb
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    other = pb.Domain.Other

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / reps

    def measure(fn):
        if args.warmup:
            timed(fn, args.warmup)
        return timed(fn, args.steps)

    # flat Merkle4 digests (the headline kernel) in the same run, for comparison
    flat_n = 1 << 20
    with torch.cuda.stream(stream):
        flat_in = device_random_scalars(torch, 4 * flat_n, 92).view(flat_n, 4, 4)
        flat_out = torch.empty((flat_n, 1, 4), dtype=torch.int64, device="cuda")
    flat = lambda: eng.hash_batch(pb.Domain.Merkle4, flat_in, out=flat_out, async_=True)
    flat_rate = flat_n / (measure(flat) * 1e-3)
    del flat_in, flat_out

    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for seed, (name, lens) in enumerate(workloads(args.items, np.random.default_rng(7)).items()):
        n = lens.shape[0]
        offs_h = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        max_len = int(lens.max())
        perms = int(np.sum((lens + 3) // 4))                  # out_len 1: ceil(out/4) - 1 = 0
        with torch.cuda.stream(stream):
            data = device_random_scalars(torch, int(offs_h[-1]), 100 + seed)
            offs = torch.from_numpy(offs_h).cuda()
            out_v = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
            out_g = torch.zeros((n, 1, 4), dtype=torch.int64, device="cuda")
            groups = []                                       # per length: item ids and their gather index
            for L in np.unique(lens):
                sel = np.nonzero(lens == L)[0]
                idx = offs_h[sel][:, None] + np.arange(L)[None, :]
                groups.append((int(L), torch.from_numpy(sel).cuda(), torch.from_numpy(idx.reshape(-1)).cuda()))
        stream.synchronize()

        def varlen():
            eng.hash_batch_varlen(other, data, offs, 1, max_len=max_len, out=out_v, async_=True)

        def grouped():
            for L, sel, idx in groups:
                x = data.index_select(0, idx).view(-1, L, 4)
                out_g.index_copy_(0, sel, eng.hash_batch(other, x, 1, async_=True))

        with torch.cuda.stream(stream):
            r = {"items": n, "max_len": max_len, "perms_per_call": perms, "distinct_lengths": len(groups)}
            r["varlen_ms"] = measure(varlen)
            r["grouped_ms"] = measure(grouped)
            if name == "a_len4":
                out_f = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
                fixed = lambda: eng.hash_batch(other, data.view(n, 4, 4), 1, out=out_f, async_=True)
                r["hash_batch_ms"] = measure(fixed)
        stream.synchronize()
        r["varlen_perm_per_s"] = perms / (r["varlen_ms"] * 1e-3)
        r["grouped_perm_per_s"] = perms / (r["grouped_ms"] * 1e-3)
        r["varlen_speedup_over_grouped"] = r["grouped_ms"] / r["varlen_ms"]
        ok = bool(torch.equal(out_v, out_g))
        if name == "a_len4":
            r["hash_batch_perm_per_s"] = perms / (r["hash_batch_ms"] * 1e-3)
            ok = ok and bool(torch.equal(out_v, out_f))
            del out_f
        parity[name] = ok
        res[name] = r
        del data, offs, out_v, out_g, groups
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "varlen_perm_per_s", "value": res["b_uniform_1_64"]["varlen_perm_per_s"], "unit": "perm/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
            "config": {"workload": "p252_hash_batch_varlen, Domain::Other, out_len 1, device buffers, %d items per call"
                                   % args.items},
            "workloads": res, "flat_merkle4_perm_per_s": flat_rate, "clocks": clocks, "device": props.name,
            "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
