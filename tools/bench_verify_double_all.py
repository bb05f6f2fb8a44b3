#!/usr/bin/env python
"""Benchmark of all-or-nothing verification of double-key signatures (p252_schnorr_verify_double_all) against per-item
verification (p252_schnorr_verify_double_batch), with single-key p252_schnorr_verify_all for reference.

    python tools/bench_verify_double_all.py [--steps K] [--warmup W] [--items N] > verify_double_all.json

All buffers device-resident, inputs seeded: N signatures (default 2^20) of schnorr_sign_double_batch under four key
pairs (n_public = n) and under one (n_public = 1), G the tests' generator and G' a seeded point of the prime-order
subgroup.  Arms:
  (a) verify_double_all against verify_double_batch on the same signatures, n_public = n and n_public = 1
  (b) for reference, verify_all against verify_batch on N single-key signatures, n_public = n
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls, with fixed weights
(two independent 128-bit arrays).  The line carries the device, its power limit and SM clocks sampled during the run,
and in-run parity: verify_double_all == 1 == AND(verify_double_batch) on the genuine batch, and 0 with one item's
message changed.  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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
    if args.steps < 1 or args.warmup < 0 or args.items < 2:
        ap.error("--steps must be >= 1, --items >= 2, --warmup >= 0")
    import numpy as np
    import torch
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    N = jo.R_J

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

    def below(rng, n, top):
        x = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        x[:, 3] %= np.uint64(top >> 192)
        return x

    def weights(rng, n):
        return dev(np.concatenate([rng.integers(1, 1 << 62, (n, 2), dtype=np.uint64), np.zeros((n, 2), np.uint64)], 1))

    rng = np.random.default_rng(41)
    n = args.items
    g = jo.points_mont([jo.GENERATOR])[0]
    gp = jo.points_mont([jo.random_subgroup_point(np.random.default_rng(42))])[0]
    sk_h = below(rng, 4, N)
    who = rng.integers(0, 4, n)
    r, m = dev(below(rng, n, N)), dev(below(rng, n, jo.P))
    w, wp = weights(rng, n), weights(rng, n)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, one in (("a_n_public_n", False), ("a_n_public_1", True)):
        sk = dev(sk_h[:1] if one else sk_h[who])
        keys = dev(sk_h[:1] if one else sk_h)
        pk4, ok1 = eng.fixed_base_batch(keys, g)
        pkp4, ok2 = eng.fixed_base_batch(keys, gp)
        pick = torch.from_numpy(np.zeros(1, np.int64) if one else who).cuda()
        pk, pkp = pk4[pick].contiguous(), pkp4[pick].contiguous()
        u, R, Rp, ok = eng.schnorr_sign_double_batch(sk, r, m, g, gp)
        t_batch = measure(lambda: eng.schnorr_verify_double_batch(pk, pkp, u, R, Rp, m, g, gp))
        ver = eng.schnorr_verify_double_batch(pk, pkp, u, R, Rp, m, g, gp)
        per_item = bool(host(ver).all()) and eng.last_schnorr_double_verified() == n
        out = {}

        def all_():
            out["a"] = eng.schnorr_verify_double_all(pk, pkp, u, R, Rp, m, g, gp, weights=w, weights_p=wp)

        t_all = measure(all_)
        m2 = m.clone()
        m2[n // 2, 0] ^= 1
        tampered = eng.schnorr_verify_double_all(pk, pkp, u, R, Rp, m2, g, gp, weights=w, weights_p=wp)
        res[name] = {"signatures": n, "verify_double_batch_ms": t_batch, "verify_double_all_ms": t_all,
                     "verify_double_all_speedup": t_batch / t_all}
        parity[name] = (bool(host(ok).all() and host(ok1).all() and host(ok2).all()) and per_item and out["a"] is True
                        and tampered is False and eng.last_schnorr_double_invalid() == 0)

    sk = dev(sk_h[who])
    pk4, _ = eng.fixed_base_batch(dev(sk_h), g)
    pk = pk4[torch.from_numpy(who).cuda()].contiguous()
    u, R, ok = eng.schnorr_sign_batch(sk, r, m, g)
    t_batch = measure(lambda: eng.schnorr_verify_batch(pk, u, R, m, g))
    out = {}

    def single():
        out["a"] = eng.schnorr_verify_all(pk, u, R, m, g, weights=w)

    t_all = measure(single)
    res["b_single_key_n_public_n"] = {"signatures": n, "verify_batch_ms": t_batch, "verify_all_ms": t_all,
                                      "verify_all_speedup": t_batch / t_all}
    parity["b_single_key_n_public_n"] = bool(host(ok).all()) and out["a"] is True
    res["a_double_over_single_verify_all"] = res["a_n_public_n"]["verify_double_all_ms"] / t_all
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "schnorr_verify_double_all_speedup", "value": res["a_n_public_n"]["verify_double_all_speedup"],
            "unit": "x over p252_schnorr_verify_double_batch", "higher_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_schnorr_verify_double_all vs p252_schnorr_verify_double_batch (n_public = n "
                                   "and 1), p252_schnorr_verify_all vs p252_schnorr_verify_batch; device buffers"},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
