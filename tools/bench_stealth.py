#!/usr/bin/env python
"""Benchmark of the stealth addresses: the receiver's ownership scan (p252_stealth_owns_batch) and the sender's note keys
(p252_stealth_address_batch).

    python tools/bench_stealth.py [--steps K] [--warmup W] [--items N] > stealth.json

All buffers device-resident, inputs seeded.  The notes are made by the sender call for two receivers, a quarter of them
for the scanning receiver (view key a, spend key B), with base G:
  (a) the scan of N notes (default 2^20) with (a, B)
  (b) the chain a caller has without the scan: p252_dhke_batch (1, n) + p252_hash_batch_truncated +
      p252_fixed_base_batch over the same notes.  It has no "+ B" and no comparison, so it is a lower bound for the
      separate path
  (c) p252_decrypt_batch_dhke at L = 2 over the same notes' R, for scale (trial decryption)
  (d) the sender of N notes with n_public = n
  (e) (a), (b) and (d) on 64 items (the latency regime)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  The line carries the
device, its power limit and SM clocks sampled during the run, and in-run parity: sampled sender rows against the Python
model (tests/stealth_oracle.py), the scan's owned flags and count against the construction, and sampled chain rows plus
B against the note keys.  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--items", type=int, default=1 << 20)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.items < 1:
        ap.error("--steps and --items must be >= 1, --warmup >= 0")
    import numpy as np
    import torch
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    import stealth_oracle as so
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

    def s_int(row):
        return sum(int(row[k]) << (64 * k) for k in range(4))

    rng = np.random.default_rng(14)
    L = 2
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    keys = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(2)]
    pub = [so.keys(a, b) for a, b in keys]
    a0, B0 = keys[0][0], pub[0][1]
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("abcd_items", args.items), ("e_small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        who = (rng.random(n) >= 0.25).astype(np.int64)        # receiver 0 (the scanner) for about a quarter
        A_h = jo.points_mont([p[0] for p in pub])[who]
        B_h = jo.points_mont([p[1] for p in pub])[who]
        with torch.cuda.stream(stream):
            r, A, B = dev(r_h), dev(A_h), dev(B_h)
            va = dev(jo.jscalar_limbs([a0]))
            R = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            pk = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            owned = torch.empty((n,), dtype=torch.uint8, device="cuda")
            shared = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            h = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
            hG = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            cip = dev(rng.integers(0, 1 << 62, (n, L + 1, 4), dtype=np.uint64))
            non = dev(rng.integers(0, 1 << 62, (n, 4), dtype=np.uint64))
            msg = torch.empty((n, L, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        out = {}

        def sender():
            out["R"], out["pk"], out["ok"] = eng.stealth_address_batch(r, gb, A, B, R_out=R, out=pk)

        def scan():
            out["owned"] = eng.stealth_owns_batch(va, B0m, gb, R, pk, out=owned)

        def chain():
            eng.dhke_batch(va, R, out=shared, async_=True)
            eng.hash_batch_truncated(pb.Domain.Other, shared, out=h, async_=True)
            eng.fixed_base_batch(h.view(n, 4), gb, out=hG, async_=True)

        def trial_decrypt():
            eng.decrypt_batch_dhke(cip, va, R, non, out=msg)

        B0m = jo.points_mont([B0])[0]
        rr = {"items": n}
        rr["sender_ms"] = measure(sender)
        rr["sender_notes_per_s"] = n / (rr["sender_ms"] * 1e-3)
        rr["scan_ms"] = measure(scan)
        rr["scan_notes_per_s"] = n / (rr["scan_ms"] * 1e-3)
        rr["scan_owned"] = eng.last_stealth_owned()
        rr["chain_ms"] = measure(chain)
        rr["scan_speedup_over_chain"] = rr["chain_ms"] / rr["scan_ms"]
        if n > 64:
            rr["decrypt_dhke_L2_ms"] = measure(trial_decrypt)
        stream.synchronize()
        eng.sync()
        rows = rng.choice(n, min(n, 6), replace=False)
        want = [so.stealth_address(s_int(r_h[i]), pub[who[i]][0], pub[who[i]][1]) for i in rows]
        Rh, pkh, hGh = host(out["R"]), host(out["pk"]), host(hG)
        mine = np.flatnonzero(who == 0)[:4]
        parity[name] = {
            "sender_rows_match_model": bool(host(out["ok"]).all()) and
            jo.points_from_mont(Rh[rows]) == [w[0] for w in want] and jo.points_from_mont(pkh[rows]) == [w[1] for w in want],
            "scan_owned_equals_construction": bool(np.array_equal(host(out["owned"]), (who == 0).astype(np.uint8))) and
            rr["scan_owned"] == int((who == 0).sum()) and eng.last_stealth_invalid() == 0,
            "chain_plus_B_equals_note_pk": all(jo.add(p, B0) == q for p, q in zip(jo.points_from_mont(hGh[mine]),
                                                                                  jo.points_from_mont(pkh[mine])))}
        res[name] = rr
        del r, A, B, va, R, pk, owned, shared, h, hG, cip, non, msg, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "stealth_scan_notes_per_s", "value": res["abcd_items"]["scan_notes_per_s"], "unit": "notes/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_stealth_owns_batch vs p252_dhke_batch (1, n) + p252_hash_batch_truncated + "
                                   "p252_fixed_base_batch vs p252_decrypt_batch_dhke at L = 2; p252_stealth_address_batch "
                                   "with n_public = n; device buffers, %d notes per call (e: 64)" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
