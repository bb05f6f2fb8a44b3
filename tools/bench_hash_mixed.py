#!/usr/bin/env python
"""Benchmark of mixed digest batches (p252_hash_batch_mixed) against the status quo of one call per group.

    python tools/bench_hash_mixed.py [--steps K] [--warmup W] [--items N] > hash_mixed.json

Workload: N items (default 2^20, seed 7) in random order, the mix a node sees: 40 % Merkle4 nodes, 20 % Domain::Other
6 -> 1 (note hashes), 20 % truncated Other 2, 3 or 5 -> 1 (stealth hashes, Schnorr challenges), 20 % Other of lengths
1..64 and out_len 1..8, half of them truncated.
  (a) one mixed call, HOST (numpy) and DEVICE (torch) buffers.
  (b) the status quo: one p252_hash_batch_varlen per (domain, out_len) for the finalized items and one
      p252_hash_batch_truncated per (domain, len, out_len) for the truncated ones; the grouping is planned once on the
      host, and each timed call gathers and scatters (numpy for HOST, on the device for DEVICE).
  (c) the cost of the tags derived on the device and of the sort: the mixed call against p252_hash_batch on N uniform
      Merkle4 items and against p252_hash_batch_varlen on N Other items of lengths 1..64 (device buffers).
DEVICE arms are timed with CUDA events on the engine's stream, HOST arms with a host clock around synchronous calls, each
over --steps calls after --warmup calls.  The line carries the device, its power limit and in-run parity: (a) equals (b)
on every row for both memory spaces, and the (c) arms agree.  Writes nothing in the repository tree.  The clock sampler
and the device-side input generator are bench.py's, imported unchanged.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

TRUNC = 0x80        # P252_MIXED_TRUNCATED
MERKLE4, OTHER = 0, 3


def workload(n, seed=7):
    """-> (mode (n,) uint8, lens (n,), out_lens (n,)) of the node mix above, in random order"""
    rng = np.random.default_rng(seed)
    k = [int(n * f) for f in (0.4, 0.2, 0.2)]
    k.append(n - sum(k))
    mode = np.concatenate([np.full(k[0], MERKLE4), np.full(k[1], OTHER), np.full(k[2], OTHER | TRUNC),
                           OTHER | np.where(rng.random(k[3]) < 0.5, TRUNC, 0)]).astype(np.uint8)
    lens = np.concatenate([np.full(k[0], 4), np.full(k[1], 6), rng.choice([2, 3, 5], k[2]), rng.integers(1, 65, k[3])])
    out_lens = np.concatenate([np.ones(k[0] + k[1] + k[2], dtype=np.int64), rng.integers(1, 9, k[3])])
    p = rng.permutation(n)
    return mode[p], lens[p], out_lens[p]


def csr(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)


def groups(mode, lens, out_lens):
    """the status quo's plan: [(truncated, domain, len or None, out_len, item ids)], one call each"""
    plan = []
    trunc = (mode & TRUNC) != 0
    dom = mode & 3
    for d in np.unique(dom):
        for ol in np.unique(out_lens):
            sel = np.nonzero(~trunc & (dom == d) & (out_lens == ol))[0]
            if sel.size:
                plan.append((False, int(d), None, int(ol), sel))
            for L in np.unique(lens[trunc & (dom == d) & (out_lens == ol)]):
                sel = np.nonzero(trunc & (dom == d) & (out_lens == ol) & (lens == L))[0]
                plan.append((True, int(d), int(L), int(ol), sel))
    return plan


def status_quo_host(eng, plan, data, offsets, out_offsets):
    """arm (b), HOST buffers: per group, gather on the host, one call, scatter into the mixed layout"""
    import poseidon252_b200 as pb
    out = np.zeros((int(out_offsets[-1]), 4), dtype=np.uint64)
    offs = offsets.astype(np.int64)
    oo = out_offsets.astype(np.int64)
    for trunc, d, L, ol, sel in plan:
        rows = (oo[sel][:, None] + np.arange(ol)[None, :]).reshape(-1)
        if trunc:
            x = data[offs[sel][:, None] + np.arange(L)[None, :]]
            out[rows] = eng.hash_batch_truncated(pb.Domain(d), x, ol).reshape(-1, 4)
        else:
            lens = offs[sel + 1] - offs[sel]
            idx = np.repeat(offs[sel] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
            out[rows] = eng.hash_batch_varlen(pb.Domain(d), data[idx], csr(lens), ol, max_len=int(lens.max())).reshape(-1, 4)
    return out


def device_plan(torch, plan, offsets, out_offsets):
    """arm (b), DEVICE buffers: per group, the gather index of its input rows and its output rows, on the device"""
    offs = offsets.astype(np.int64)
    oo = out_offsets.astype(np.int64)
    dp = []
    for trunc, d, L, ol, sel in plan:
        lens = offs[sel + 1] - offs[sel]
        idx = np.repeat(offs[sel] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
        rows = (oo[sel][:, None] + np.arange(ol)[None, :]).reshape(-1)
        dp.append((trunc, d, L, ol, len(sel), torch.from_numpy(idx).cuda(), torch.from_numpy(csr(lens).view(np.int64)).cuda(),
                   int(lens.max()), torch.from_numpy(rows).cuda()))
    return dp


def status_quo_device(eng, dplan, data, out):
    import poseidon252_b200 as pb
    for trunc, d, L, ol, n, idx, goffs, longest, rows in dplan:
        x = data.index_select(0, idx)
        if trunc:
            y = eng.hash_batch_truncated(pb.Domain(d), x.view(n, L, 4), ol, async_=True)
        else:
            y = eng.hash_batch_varlen(pb.Domain(d), x, goffs, ol, max_len=longest, async_=True)
        out.index_copy_(0, rows, y.view(-1, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--items", type=int, default=1 << 20)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.items < 1:
        ap.error("--steps and --items must be >= 1, --warmup >= 0")
    import torch
    import poseidon252_b200 as pb
    from bench import ClockSampler, device_random_scalars
    from poseidon252_b200.scalar import random_limbs_fast
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)

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

    def measure_host(fn):
        for _ in range(args.warmup):
            fn()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    sampler = ClockSampler(0)
    sampler.start()
    n = args.items
    mode, lens, out_lens = workload(n)
    offsets, out_offsets = csr(lens), csr(out_lens)
    max_len, max_out = int(lens.max()), int(out_lens.max())
    perms = int(np.sum((lens + 3) // 4 + (out_lens + 3) // 4 - 1))
    plan = groups(mode, lens, out_lens)
    data_h = random_limbs_fast(np.random.default_rng(11), int(offsets[-1]))
    res, parity = {"items": n, "perms_per_call": perms, "status_quo_calls": len(plan)}, {}

    # (a) vs (b), HOST buffers
    mixed_h = eng.hash_batch_mixed(mode, data_h, offsets, out_offsets, max_len, max_out)
    parity["host_a_equals_b"] = bool(np.array_equal(mixed_h, status_quo_host(eng, plan, data_h, offsets, out_offsets)))
    res["host_mixed_ms"] = measure_host(lambda: eng.hash_batch_mixed(mode, data_h, offsets, out_offsets, max_len, max_out,
                                                                     out=mixed_h))
    res["host_status_quo_ms"] = measure_host(lambda: status_quo_host(eng, plan, data_h, offsets, out_offsets))

    # (a) vs (b), DEVICE buffers
    with torch.cuda.stream(stream):
        data = torch.from_numpy(data_h.view(np.int64)).cuda()
        mode_d = torch.from_numpy(mode).cuda()
        offs_d = torch.from_numpy(offsets.view(np.int64)).cuda()
        oofs_d = torch.from_numpy(out_offsets.view(np.int64)).cuda()
        out_m = torch.empty((int(out_offsets[-1]), 4), dtype=torch.int64, device="cuda")
        out_b = torch.zeros_like(out_m)
        dplan = device_plan(torch, plan, offsets, out_offsets)
    stream.synchronize()
    mixed = lambda: eng.hash_batch_mixed(mode_d, data, offs_d, oofs_d, max_len, max_out, out=out_m, async_=True)
    res["device_mixed_ms"] = measure(mixed)
    res["device_status_quo_ms"] = measure(lambda: status_quo_device(eng, dplan, data, out_b))
    parity["device_a_equals_b"] = bool(torch.equal(out_m, out_b))
    parity["device_equals_host"] = bool(np.array_equal(out_m.cpu().numpy().view(np.uint64), mixed_h))
    for mem in ("host", "device"):
        res["%s_mixed_perm_per_s" % mem] = perms / (res["%s_mixed_ms" % mem] * 1e-3)
        res["%s_speedup_over_status_quo" % mem] = res["%s_status_quo_ms" % mem] / res["%s_mixed_ms" % mem]
    del data, mode_d, offs_d, oofs_d, out_m, out_b, dplan
    torch.cuda.empty_cache()

    # (c) the mixed call on the inputs of the fixed-length and the varlen calls
    cost = {}
    for name, lens_c, dom in (("uniform_merkle4", np.full(n, 4), MERKLE4),
                              ("other_1_64", np.random.default_rng(13).integers(1, 65, n), OTHER)):
        offs_c, oofs_c = csr(lens_c), csr(np.ones(n, dtype=np.int64))
        with torch.cuda.stream(stream):
            data = device_random_scalars(torch, int(offs_c[-1]), 21)
            mode_d = torch.full((n,), dom, dtype=torch.uint8, device="cuda")
            offs_d = torch.from_numpy(offs_c.view(np.int64)).cuda()
            oofs_d = torch.from_numpy(oofs_c.view(np.int64)).cuda()
            out_m = torch.empty((n, 4), dtype=torch.int64, device="cuda")
            out_r = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        ml = int(lens_c.max())
        r = {"mixed_ms": measure(lambda: eng.hash_batch_mixed(mode_d, data, offs_d, oofs_d, ml, 1, out=out_m, async_=True))}
        if dom == MERKLE4:
            ref = lambda: eng.hash_batch(pb.Domain.Merkle4, data.view(n, 4, 4), 1, out=out_r, async_=True)
            r["hash_batch_ms"] = measure(ref)
        else:
            ref = lambda: eng.hash_batch_varlen(pb.Domain.Other, data, offs_d, 1, max_len=ml, out=out_r, async_=True)
            r["hash_batch_varlen_ms"] = measure(ref)
        r["mixed_over_reference"] = r["mixed_ms"] / [v for k, v in r.items() if k != "mixed_ms"][0]
        parity["c_" + name] = bool(torch.equal(out_m, out_r.view(n, 4)))
        cost[name] = r
        del data, mode_d, offs_d, oofs_d, out_m, out_r
        torch.cuda.empty_cache()
    res["c"] = cost
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "mixed_perm_per_s", "value": res["device_mixed_perm_per_s"], "unit": "perm/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
            "config": {"workload": "p252_hash_batch_mixed, node mix (40%% Merkle4, 20%% Other 6->1, 20%% truncated Other "
                                   "2/3/5->1, 20%% Other 1..64 -> 1..8 half truncated), %d items per call" % n},
            "results": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
