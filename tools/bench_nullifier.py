#!/usr/bin/env python
"""Benchmark of the note nullifiers (p252_nullifier_batch).

    python tools/bench_nullifier.py [--steps K] [--warmup W] [--items N] > nullifier.json

All buffers device-resident, inputs seeded.  The notes are made by p252_stealth_address_batch for one wallet (a, b) with
base G, at seeded positions below 2^63; G' is a seeded point of the prime-order subgroup:
  (a) the fused call on N notes (default 2^20), n_secret = 1
  (b) the chain a caller has without it: p252_dhke_batch (1, n) + p252_hash_batch_truncated, a copy to the host,
      (h + b) mod r_J there (vectorised numpy), a copy back, p252_fixed_base_batch with G', the rows [u, v, pos] packed on
      the device (the positions' Montgomery images precomputed outside the timed window), p252_hash_batch.  Packing on
      the device and precomputing the positions make it a lower bound for the chain
  (c) p252_stealth_owns_batch of the same notes, for scale (the wallet's scan that finds them)
  (d) (a) and (b) on 64 items (the latency regime)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls; the chain's host step
is inside the window.  The line carries the device, its power limit and SM clocks sampled during the run, and in-run
parity: (a) equals (b) on every row, sampled rows of (a) against the Python model (tests/nullifier_oracle.py), and the
scan owns every note.  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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


def add_mod_order(h, b, order):
    """(h + b) mod r_J for rows h (n, 4) uint64 < 2^250 and one b < r_J, limb by limb on the host"""
    import numpy as np
    n = h.shape[0]
    s, d = np.empty_like(h), np.empty_like(h)
    carry = np.zeros(n, dtype=np.uint64)
    for k in range(4):
        t = h[:, k] + np.uint64(b[k])
        c1 = t < h[:, k]
        s[:, k] = t + carry
        carry = (c1 | (s[:, k] < t)).astype(np.uint64)
    borrow = np.zeros(n, dtype=np.uint64)
    for k in range(4):
        t = s[:, k] - np.uint64(order[k])
        b1 = s[:, k] < np.uint64(order[k])
        d[:, k] = t - borrow
        borrow = (b1 | (t < borrow)).astype(np.uint64)
    return np.where((borrow != 0)[:, None], s, d)          # borrow: s < r_J


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
    import nullifier_oracle as no
    import poseidon252_b200 as pb
    import stealth_oracle as so
    from poseidon252_b200.scalar import to_mont
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

    rng = np.random.default_rng(15)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    Gp = jo.random_subgroup_point(rng)
    gpb = jo.points_mont([Gp])[0]
    a0, b0 = jo.random_secret(rng), jo.random_secret(rng)
    A0, B0 = so.keys(a0, b0)
    order = jo.jscalar_limbs([jo.R_J])[0]
    b_limbs = jo.jscalar_limbs([b0])[0]
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("abc_items", args.items), ("d_small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        pool = rng.integers(0, 1 << 63, 256, dtype=np.uint64)
        sel = rng.integers(0, len(pool), n)
        pos_h, pm_h = pool[sel], to_mont([int(x) for x in pool])[sel]
        with torch.cuda.stream(stream):
            al, bl = dev(jo.jscalar_limbs([a0])), dev(jo.jscalar_limbs([b0]))
            pos, pm = dev(pos_h), dev(pm_h).reshape(n, 1, 4)
            R, pk, _ = eng.stealth_address_batch(dev(r_h), gb, dev(jo.points_mont([A0])), dev(jo.points_mont([B0])))
            nul = torch.empty((n, 4), dtype=torch.int64, device="cuda")
            owned = torch.empty((n,), dtype=torch.uint8, device="cuda")
            shared = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            h = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
            pkp = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            rows = torch.empty((n, 3, 4), dtype=torch.int64, device="cuda")
            chain_out = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        out = {}

        def fused():
            out["nul"], out["ok"] = eng.nullifier_batch(al, bl, gpb, R, pos, out=nul)

        def chain():
            eng.dhke_batch(al, R, out=shared, async_=True)
            eng.hash_batch_truncated(pb.Domain.Other, shared, out=h, async_=True)
            stream.synchronize()
            sk = dev(add_mod_order(host(h).reshape(n, 4), b_limbs, order))
            eng.fixed_base_batch(sk, gpb, out=pkp, async_=True)
            with torch.cuda.stream(stream):
                torch.cat([pkp, pm], dim=1, out=rows)
            eng.hash_batch(pb.Domain.Other, rows, out=chain_out, async_=True)

        def scan():
            out["owned"] = eng.stealth_owns_batch(al, jo.points_mont([B0])[0], gb, R, pk, out=owned)

        rr = {"items": n}
        rr["fused_ms"] = measure(fused)
        rr["fused_notes_per_s"] = n / (rr["fused_ms"] * 1e-3)
        rr["chain_ms"] = measure(chain)
        rr["fused_speedup_over_chain"] = rr["chain_ms"] / rr["fused_ms"]
        if n > 64:
            rr["scan_ms"] = measure(scan)
            rr["fused_over_scan"] = rr["fused_ms"] / rr["scan_ms"]
        stream.synchronize()
        eng.sync()
        nh, Rh = host(out["nul"]), host(R)
        picks = rng.choice(n, min(n, 4), replace=False)
        model = [no.nullifier(a0, b0, jo.points_from_mont(Rh[i:i + 1])[0], int(pos_h[i]), Gp) for i in picks]
        check = {"fused_equals_chain": bool(host(out["ok"]).all()) and bool(np.array_equal(nh, host(chain_out).reshape(n, 4))),
                 "fused_rows_match_model": all(m is not None and int(pb.scalar.from_mont(nh[i])) == m
                                               for i, m in zip(picks, model))}
        if n > 64:
            check["scan_owns_every_note"] = bool(host(out["owned"]).all()) and eng.last_stealth_owned() == n
        parity[name] = check
        res[name] = rr
        del al, bl, pos, pm, R, pk, nul, owned, shared, h, pkp, rows, chain_out, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "nullifier_notes_per_s", "value": res["abc_items"]["fused_notes_per_s"], "unit": "notes/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_nullifier_batch (n_secret = 1) vs p252_dhke_batch (1, n) + "
                                   "p252_hash_batch_truncated + host add mod r_J + p252_fixed_base_batch (G') + "
                                   "p252_hash_batch vs p252_stealth_owns_batch; device buffers, %d notes per call "
                                   "(d: 64)" % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
