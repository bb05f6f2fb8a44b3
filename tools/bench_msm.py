#!/usr/bin/env python
"""Benchmark of the JubJub multi-scalar multiplication (p252_jubjub_msm) and of all-or-nothing Schnorr verification
(p252_schnorr_verify_all) against per-item verification (p252_schnorr_verify_batch).

    python tools/bench_msm.py [--steps K] [--warmup W] [--sizes 16,18,20,22] [--items N] > msm.json

All buffers device-resident, inputs seeded, base G.  Arms:
  (a) MSM of 2^k points P_i = [k_i] G (from fixed_base_batch) with random scalars < r_J, for each k of --sizes
  (b) MSM of 2^20 points with every scalar equal (all digits of a window in one bucket: the worst skew)
  (c) verify_all against verify_batch on the same N signatures (default 2^20), n_public = n and n_public = 1
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  The line carries the
device, its power limit and SM clocks sampled during the run, and in-run parity: every MSM against fixed_base_batch of
[sum s_i k_i mod r_J] G (an identity that does not use the bucket code), and verify_all == 1 == AND(verify_batch).
Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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
    ap.add_argument("--sizes", default="16,18,20,22")
    ap.add_argument("--items", type=int, default=1 << 20)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.items < 1:
        ap.error("--steps and --items must be >= 1, --warmup >= 0")
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

    def rows(vals):
        out = np.zeros((len(vals), 4), dtype=np.uint64)
        for k in range(4):
            out[:, k] = [(v >> (64 * k)) & ((1 << 64) - 1) for v in vals]
        return out

    rng = np.random.default_rng(21)
    gb = jo.points_mont([jo.GENERATOR])[0]
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}

    def msm_arm(name, n, equal):
        k = [int(x) for x in rng.integers(1, 1 << 62, n)]
        pts, ok = eng.fixed_base_batch(dev(jo.jscalar_limbs(k)), gb)
        if equal:
            s_h = np.tile(rows([N - 12345]), (n, 1))
        else:
            s_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
            s_h[:, 3] %= np.uint64(N >> 192)                  # < r_J
        s = [int(a) | int(b) << 64 | int(c) << 128 | int(d) << 192 for a, b, c, d in s_h.tolist()]
        sc = dev(s_h)
        out = torch.empty((2, 4), dtype=torch.int64, device="cuda")
        ms = measure(lambda: eng.jubjub_msm(sc, pts, out=out))
        want, _ = eng.fixed_base_batch(jo.jscalar_limbs([sum(a * b for a, b in zip(s, k)) % N]), gb)
        res[name] = {"points": n, "ms": ms, "points_per_s": n / (ms * 1e-3)}
        parity[name] = bool(host(ok).all()) and np.array_equal(host(out).reshape(2, 4), want[0])

    for b in [int(x) for x in args.sizes.split(",") if x]:
        msm_arm("a_msm_2^%d_random" % b, 1 << b, False)
    msm_arm("b_msm_2^20_all_equal", 1 << 20, True)
    res["b_equal_over_random_2^20"] = res["b_msm_2^20_all_equal"]["ms"] / res["a_msm_2^20_random"]["ms"] \
        if "a_msm_2^20_random" in res else None

    n = args.items
    sks = [jo.random_secret(rng) for _ in range(4)]
    pks = [jo.mul(x, jo.GENERATOR) for x in sks]
    who = rng.integers(0, 4, n)
    r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    r_h[:, 3] %= np.uint64(N >> 192)
    m_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    m_h[:, 3] %= np.uint64(jo.P >> 192)
    r, m = dev(r_h), dev(m_h)
    for name, one in (("c_n_public_n", False), ("c_n_public_1", True)):
        sk = dev(jo.jscalar_limbs(sks[:1] if one else sks)[np.zeros(1, np.int64) if one else who])
        pk = dev(jo.points_mont(pks[:1] if one else pks)[np.zeros(1, np.int64) if one else who])
        u, R, ok = eng.schnorr_sign_batch(sk, r, m, gb)
        w = eng_weights = dev(np.concatenate([rng.integers(1, 1 << 62, (n, 2), dtype=np.uint64), np.zeros((n, 2), np.uint64)], 1))
        ver = torch.empty((n,), dtype=torch.uint8, device="cuda")
        out = {}
        t_batch = measure(lambda: eng.schnorr_verify_batch(pk, u, R, m, gb, out=ver))
        per_item = bool(host(ver).all()) and eng.last_schnorr_verified() == n

        def all_():
            out["a"] = eng.schnorr_verify_all(pk, u, R, m, gb, weights=w)

        t_all = measure(all_)
        res[name] = {"signatures": n, "verify_batch_ms": t_batch, "verify_all_ms": t_all,
                     "verify_all_speedup": t_batch / t_all}
        parity[name] = bool(host(ok).all()) and per_item and out["a"] is True
        del eng_weights
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "schnorr_verify_all_speedup", "value": res["c_n_public_n"]["verify_all_speedup"],
            "unit": "x over p252_schnorr_verify_batch", "higher_is_better": True, "n_gpus": 1, "steps": args.steps,
            "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_jubjub_msm (random and all-equal scalars), p252_schnorr_verify_all vs "
                                   "p252_schnorr_verify_batch; device buffers"},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
