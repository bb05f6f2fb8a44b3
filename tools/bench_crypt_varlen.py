#!/usr/bin/env python
"""Benchmark of variable-length encrypt / decrypt batches (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen) against
the fixed-length calls.

    python tools/bench_crypt_varlen.py [--steps K] [--warmup W] [--items N] > crypt_varlen.json

Three workloads, each encrypted and decrypted, all buffers device-resident:
  (a) N items (default 2^20) of length 2 (the benches/encrypt.rs shape): one varlen call vs one p252_encrypt_batch /
      p252_decrypt_batch call (the cost of the keys, the sort and the per-lane bookkeeping)
  (b) N items of lengths uniform in 1..64: one varlen call vs grouped calls (per length: gather, fixed-length call,
      scatter, all on the device and inside the timed region)
  (c) 64 items of lengths uniform in 1..64 (the lane-split kernel's regime): the same two arms as (b)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  perm/s counts
sum(2 * ceil(L/4)) permutations per call.  The line carries the device, its power limit and SM clocks sampled during the
run, and in-run parity: the varlen cipher equals the grouped (or fixed-length) cipher, the varlen decrypt equals the
grouped decrypt, and the round trip restores every message with every ok set.  Writes nothing in the repository tree.
The clock sampler and the device-side input generator are bench.py's, imported unchanged.
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
    return {"a_len2": np.full(n, 2), "b_uniform_1_64": rng.integers(1, 65, n), "c_small_64_items": rng.integers(1, 65, 64)}


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

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
        stream.synchronize()
        eng.sync()                                            # releases the failure counters of async decrypts
        return e0.elapsed_time(e1) / reps

    def measure(fn):
        if args.warmup:
            timed(fn, args.warmup)
        return timed(fn, args.steps)

    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for seed, (name, lens) in enumerate(workloads(args.items, np.random.default_rng(7)).items()):
        n = lens.shape[0]
        offs_h = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        coff_h = offs_h + np.arange(n + 1)
        max_len = int(lens.max())
        perms = int(np.sum(2 * ((lens + 3) // 4)))
        with torch.cuda.stream(stream):
            data = device_random_scalars(torch, int(offs_h[-1]), 200 + seed)
            uv = device_random_scalars(torch, 2 * n, 300 + seed).view(n, 2, 4)
            non = device_random_scalars(torch, n, 400 + seed)
            offs, coffs = torch.from_numpy(offs_h).cuda(), torch.from_numpy(coff_h).cuda()
            c_v = torch.empty((int(coff_h[-1]), 4), dtype=torch.int64, device="cuda")
            c_g = torch.zeros_like(c_v)
            m_g = torch.zeros_like(data)
            ok_g = torch.zeros((n,), dtype=torch.uint8, device="cuda")
            groups = []                                       # per length: item ids, message and cipher gather indices
            for L in np.unique(lens):
                sel = np.nonzero(lens == L)[0]
                midx = offs_h[sel][:, None] + np.arange(L)[None, :]
                cidx = coff_h[sel][:, None] + np.arange(L + 1)[None, :]
                groups.append((int(L), torch.from_numpy(sel).cuda(), torch.from_numpy(midx.reshape(-1)).cuda(),
                               torch.from_numpy(cidx.reshape(-1)).cuda()))
        stream.synchronize()
        out = {}

        def enc_varlen():
            eng.encrypt_batch_varlen(data, offs, uv, non, max_len=max_len, out=c_v, async_=True)

        def enc_grouped():
            for L, sel, midx, cidx in groups:
                c = eng.encrypt_batch(data.index_select(0, midx).view(-1, L, 4), uv.index_select(0, sel),
                                      non.index_select(0, sel), async_=True)
                c_g.index_copy_(0, cidx, c.view(-1, 4))

        def dec_varlen():
            out["m"], _, out["ok"] = eng.decrypt_batch_varlen(c_v, coffs, uv, non, max_len=max_len, async_=True)

        def dec_grouped():
            for L, sel, midx, cidx in groups:
                m, ok = eng.decrypt_batch(c_v.index_select(0, cidx).view(-1, L + 1, 4), uv.index_select(0, sel),
                                          non.index_select(0, sel), async_=True)
                m_g.index_copy_(0, midx, m.view(-1, 4))
                ok_g.index_copy_(0, sel, ok)

        fixed = name == "a_len2"
        arm = "fixed" if fixed else "grouped"
        with torch.cuda.stream(stream):
            r = {"items": n, "max_len": max_len, "perms_per_call": perms, "distinct_lengths": len(groups)}
            r["encrypt_varlen_ms"] = measure(enc_varlen)
            if fixed:
                c_f = torch.empty((n, 3, 4), dtype=torch.int64, device="cuda")
                r["encrypt_fixed_ms"] = measure(lambda: eng.encrypt_batch(data.view(n, 2, 4), uv, non, out=c_f, async_=True))
            else:
                r["encrypt_grouped_ms"] = measure(enc_grouped)
            r["decrypt_varlen_ms"] = measure(dec_varlen)
            if fixed:
                def dec_fixed():
                    out["mf"], out["okf"] = eng.decrypt_batch(c_v.view(n, 3, 4), uv, non, async_=True)
                r["decrypt_fixed_ms"] = measure(dec_fixed)
            else:
                r["decrypt_grouped_ms"] = measure(dec_grouped)
        stream.synchronize()
        eng.sync()
        for op in ("encrypt", "decrypt"):
            r["%s_varlen_perm_per_s" % op] = perms / (r["%s_varlen_ms" % op] * 1e-3)
            r["%s_%s_perm_per_s" % (op, arm)] = perms / (r["%s_%s_ms" % (op, arm)] * 1e-3)
            r["%s_varlen_speedup_over_%s" % (op, arm)] = r["%s_%s_ms" % (op, arm)] / r["%s_varlen_ms" % op]
        if fixed:
            same_c = bool(torch.equal(c_v.view(n, 3, 4), c_f))
            same_m = bool(torch.equal(out["m"].view(n, 2, 4), out["mf"])) and bool(torch.equal(out["ok"], out["okf"]))
            del c_f
        else:
            same_c = bool(torch.equal(c_v, c_g))
            same_m = bool(torch.equal(out["m"], m_g)) and bool(torch.equal(out["ok"], ok_g))
        round_trip = bool(torch.equal(out["m"], data)) and bool(out["ok"].all())
        parity[name] = {"cipher_equal": same_c, "decrypt_equal": same_m, "round_trip": round_trip}
        res[name] = r
        del data, uv, non, offs, coffs, c_v, c_g, m_g, ok_g, groups, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "encrypt_varlen_perm_per_s", "value": res["b_uniform_1_64"]["encrypt_varlen_perm_per_s"],
            "unit": "perm/s", "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "data": "synthetic",
            "config": {"workload": "p252_encrypt_batch_varlen / p252_decrypt_batch_varlen, device buffers, %d items per call "
                                   "(c: 64)" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
