#!/usr/bin/env python
"""Benchmark of the fixed-base JubJub scalar multiplication (p252_fixed_base_batch) and of the sender's encrypt batch
(p252_encrypt_batch_ephemeral), each against the variable-base calls that computed the same thing before.

    python tools/bench_fixed_base.py [--steps K] [--warmup W] [--items N] > fixed_base.json

All buffers device-resident, inputs seeded (r_i, the receiver key, messages and nonces from a fixed-seed generator):
  (a) p252_fixed_base_batch, N items (default 2^20) with the generator G, against p252_dhke_batch in the (n, 1) shape
      (G passed as an ordinary point) on the same secrets: ms per call, items/s, and the outputs equal
  (b) the sender of N notes at L = 2: p252_encrypt_batch_ephemeral against p252_dhke_batch(r, G) +
      p252_encrypt_batch_dhke(msg, r, pk): R and the ciphers equal
  (c) (a) and (b) on a batch of 64 items (the latency regime)
  (d) the first call with a new base (table build + k_fixed_base) against a call with the cached base, 64 items
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  The line carries the
device, its power limit and SM clocks sampled during the run, and in-run parity, including sampled rows of (a) against the
Python model (tests/jubjub_oracle.py).  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported
unchanged.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench import ClockSampler  # noqa: E402


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
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    from poseidon252_b200.scalar import jubjub_limbs
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
        eng.sync()
        return e0.elapsed_time(e1) / reps

    def measure(fn):
        if args.warmup:
            timed(fn, args.warmup)
        return timed(fn, args.steps)

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()

    def host(t):
        a = t.cpu().numpy()
        return a.view(np.uint64) if a.dtype == np.int64 else a

    rng = np.random.default_rng(12)
    L = 2
    g_h = jo.points_mont([jo.GENERATOR])
    g, gb = dev(g_h), g_h[0]
    a = jo.random_secret(rng)
    pk_h = jo.points_mont([jo.mul(a, jo.GENERATOR)])
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("ab_items", args.items), ("c_small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        with torch.cuda.stream(stream):
            r = dev(r_h)
            pk = dev(pk_h)
            msg = dev(rng.integers(0, 1 << 62, (n, L, 4), dtype=np.uint64))
            non = dev(rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64))
            R_f = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            R_d = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            c_f = torch.empty((n, L + 1, 4), dtype=torch.int64, device="cuda")
            R_s = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            c_s = torch.empty((n, L + 1, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        out = {}

        def fixed():
            out["R"], out["ok"] = eng.fixed_base_batch(r, gb, out=R_f, async_=True)

        def dhke_n1():
            out["Rd"], out["okd"] = eng.dhke_batch(r, g, out=R_d, async_=True)

        def fused():
            out["cf"], out["Rf"], out["okf"] = eng.encrypt_batch_ephemeral(msg, r, gb, pk, non, out=c_f, R_out=R_s)

        def separate():
            out["Rs"], _ = eng.dhke_batch(r, g, out=R_d, async_=True)
            out["cs"], out["oks"] = eng.encrypt_batch_dhke(msg, r, pk, non, out=c_s, async_=True)

        rr = {"items": n, "L": L}
        rr["fixed_base_ms"] = measure(fixed)
        rr["fixed_base_per_s"] = n / (rr["fixed_base_ms"] * 1e-3)
        rr["dhke_n1_ms"] = measure(dhke_n1)
        rr["fixed_base_speedup_over_dhke_n1"] = rr["dhke_n1_ms"] / rr["fixed_base_ms"]
        rr["sender_fused_ms"] = measure(fused)
        rr["sender_separate_ms"] = measure(separate)
        rr["sender_speedup_over_separate"] = rr["sender_separate_ms"] / rr["sender_fused_ms"]
        rr["notes_per_s_fused"] = n / (rr["sender_fused_ms"] * 1e-3)
        stream.synchronize()
        eng.sync()
        rows = rng.choice(n, min(n, 8), replace=False)
        want = jo.points_mont([jo.mul(sum(int(r_h[i, k]) << (64 * k) for k in range(4)), jo.GENERATOR) for i in rows])
        parity[name] = {"fixed_base_rows_match_oracle": bool(np.array_equal(host(out["R"])[rows], want)) and
                        bool(host(out["ok"]).all()),
                        "fixed_base_equals_dhke_n1": bool(torch.equal(out["R"], out["Rd"])) and bool(out["okd"].all()),
                        "sender_R_equal": bool(torch.equal(out["Rf"], out["Rs"])) and bool(torch.equal(out["Rf"], out["R"])),
                        "sender_ciphers_equal": bool(torch.equal(out["cf"], out["cs"])) and
                        bool(torch.equal(out["okf"], out["oks"])) and bool(out["okf"].all())}
        res[name] = rr
        del r, pk, msg, non, R_f, R_d, c_f, R_s, c_s, out
        torch.cuda.empty_cache()
    # (d) table build: alternate two bases, so that every call rebuilds, against the cached generator
    r64 = dev(jubjub_limbs([jo.random_secret(rng) for _ in range(64)]))
    other = jo.points_mont([jo.random_point(rng)])[0]
    flip = {"k": 0}

    def rebuild():
        flip["k"] ^= 1
        eng.fixed_base_batch(r64, other if flip["k"] else gb, async_=True)

    def cached():
        eng.fixed_base_batch(r64, gb, async_=True)

    res["d_table_64_items"] = {"new_base_ms": measure(rebuild), "cached_base_ms": measure(cached)}
    res["d_table_64_items"]["table_build_ms"] = res["d_table_64_items"]["new_base_ms"] - \
        res["d_table_64_items"]["cached_base_ms"]
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "fixed_base_per_s", "value": res["ab_items"]["fixed_base_per_s"], "unit": "items/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_fixed_base_batch with G vs p252_dhke_batch (n, 1); "
                                   "p252_encrypt_batch_ephemeral vs p252_dhke_batch + p252_encrypt_batch_dhke at L = 2; "
                                   "device buffers, %d items per call (c, d: 64)" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
