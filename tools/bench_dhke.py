#!/usr/bin/env python
"""Benchmark of the JubJub key exchange (p252_dhke_batch) and of the decrypt batch that derives its shared secret on the
device (p252_decrypt_batch_dhke).

    python tools/bench_dhke.py [--steps K] [--warmup W] [--items N] > dhke.json

The wallet-scan shape throughout: one view key a against n ephemeral keys R_i = [r_i] G, all buffers device-resident,
inputs seeded (r_i, messages and nonces from a fixed-seed generator; R_i, pk = [a] G and the ciphers are made on the device
before timing):
  (a) p252_dhke_batch, N items (default 2^20) in the (1, n) shape: ms per call and dhke/s
  (b) p252_decrypt_batch_dhke at L = 2 against p252_dhke_batch + p252_decrypt_batch on the same inputs
  (c) the same three calls on a batch of 64 items (the latency regime)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  The line carries the
device, its power limit and SM clocks sampled during the run, and in-run parity: sampled rows of (a) against the Python
model (tests/jubjub_oracle.py), the two arms of (b) equal, and every note decrypting back to its message.  Writes nothing in
the repository tree.  The clock sampler is bench.py's, imported unchanged.
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

    rng = np.random.default_rng(11)
    L = 2
    g = dev(jo.points_mont([jo.GENERATOR]))
    a = jo.random_secret(rng)
    sk = dev(jubjub_limbs([a]))
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("ab_items", args.items), ("c_small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        with torch.cuda.stream(stream):
            r = dev(r_h)
            msg = dev(rng.integers(0, 1 << 62, (n, L, 4), dtype=np.uint64))
            non = dev(rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64))
            pk, _ = eng.dhke_batch(sk, g)
            R, _ = eng.dhke_batch(r, g)                      # the notes' ephemeral keys
            uv, _ = eng.dhke_batch(r, pk)                    # the senders' shared secrets
            cip = eng.encrypt_batch(msg, uv, non)
            shared = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            m_f = torch.empty((n, L, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        out = {}

        def dhke():
            out["s"], out["sok"] = eng.dhke_batch(sk, R, out=shared, async_=True)

        def fused():
            out["mf"], out["okf"] = eng.decrypt_batch_dhke(cip, sk, R, non, out=m_f, async_=True)

        def separate():
            s, _ = eng.dhke_batch(sk, R, async_=True)
            out["ms"], out["oks"] = eng.decrypt_batch(cip, s, non, async_=True)

        rr = {"items": n, "L": L}
        rr["dhke_ms"] = measure(dhke)
        rr["dhke_per_s"] = n / (rr["dhke_ms"] * 1e-3)
        rr["decrypt_dhke_fused_ms"] = measure(fused)
        rr["decrypt_dhke_separate_ms"] = measure(separate)
        rr["fused_speedup_over_separate"] = rr["decrypt_dhke_separate_ms"] / rr["decrypt_dhke_fused_ms"]
        rr["notes_per_s_fused"] = n / (rr["decrypt_dhke_fused_ms"] * 1e-3)
        stream.synchronize()
        eng.sync()
        rows = rng.choice(n, min(n, 8), replace=False)
        got = host(out["s"])[rows]
        want = jo.points_mont([jo.dhke(a, p) for p in jo.points_from_mont(host(R)[rows])])
        parity[name] = {"dhke_rows_match_oracle": bool(np.array_equal(got, want)) and bool(host(out["sok"]).all()),
                        "shared_equals_sender": bool(torch.equal(out["s"], uv)),
                        "fused_equals_separate": bool(torch.equal(out["mf"], out["ms"])) and
                        bool(torch.equal(out["okf"], out["oks"])),
                        "round_trip": bool(torch.equal(out["mf"], msg)) and bool(out["okf"].all())}
        res[name] = rr
        del r, msg, non, pk, R, uv, cip, shared, m_f, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "dhke_per_s", "value": res["ab_items"]["dhke_per_s"], "unit": "dhke/s", "higher_is_better": True,
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_dhke_batch (1, n) and p252_decrypt_batch_dhke at L = 2, device buffers, %d items "
                                   "per call (c: 64)" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
