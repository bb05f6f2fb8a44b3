#!/usr/bin/env python
"""Benchmark of the multi-key wallet scan (p252_wallet_scan_batch) against the chain of existing calls a wallet would
otherwise run.

    python tools/bench_wallet.py [--steps K] [--warmup W] > wallet.json

All buffers device-resident, inputs seeded; G' is a seeded point of the prime-order subgroup.  The notes are made by
p252_note_create_batch: a quarter of them for the k keys (spread evenly), the rest for a stranger.  Shapes: 2^20 notes at
k = 1 and 4, 2^18 at k = 16, and 64 notes at k = 1 (the latency regime).  The chain, per key: p252_stealth_owns_batch over
every note, a torch gather of the owned rows, p252_nullifier_batch and p252_note_open_batch on them, and a torch sum of
the opened values.  The chain is favoured: its G and G' calls run on two engines (the scan's and the nullifier's single
base slot hold one table each, so nothing is rebuilt), and it does not resolve duplicate keys.  The ratios the product
counts predict (DESIGN.md section 4) are printed beside the measured ones.  Each arm is timed with CUDA events on the
engines' shared stream over --steps calls after --warmup calls.  The line carries the device, its power limit and SM
clocks sampled during the run, and in-run parity: the fused call's owner, nullifier, value, blinder, opened and totals
equal the chain's, and two sampled notes equal the Python model (tests/wallet_oracle.py).  Writes nothing in the
repository tree.  The clock sampler is bench.py's, imported unchanged.
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

PERM, DHKE, OWNS, NUL_KEY, OPEN_VALUE, SELECT = 365, 2819, 456, 867, 568, 4
PAIR = DHKE + PERM + OWNS                       # [a_j] R_i, its hash, the ownership check
OWNED_FUSED = NUL_KEY + PERM + 2 * PERM + OPEN_VALUE
OWNED_CHAIN = (DHKE + PERM + NUL_KEY + PERM) + (DHKE + 2 * PERM + OPEN_VALUE)
SHAPES = (("n20_k1", 1 << 20, 1), ("n20_k4", 1 << 20, 4), ("n18_k16", 1 << 18, 16), ("n64_k1", 64, 1))


def predicted(k, owned=0.25):
    return (k * PAIR + owned * OWNED_CHAIN) / (k * PAIR + SELECT + owned * OWNED_FUSED)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1, --warmup >= 0")
    import numpy as np
    import torch
    import hades_oracle as ho
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    import stealth_oracle as so
    import wallet_oracle as wo
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    eng_p = pb.Engine(0, stream=stream.cuda_stream)          # the chain's nullifier calls: G' in their single-base slot

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
        a = np.ascontiguousarray(a)
        return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()

    def host(t):
        a = t.cpu().numpy()
        return a.view(np.uint64) if a.dtype == np.int64 else a

    def fr_int(row):                                          # Montgomery limbs -> canonical int
        return sum(int(row[q]) << (64 * q) for q in range(4)) * pow(ho.R, -1, jo.P) % jo.P

    rng = np.random.default_rng(23)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    Gp = jo.random_subgroup_point(rng)
    gpb = jo.points_mont([Gp])[0]
    stranger = so.keys(jo.random_secret(rng), jo.random_secret(rng))
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n, k in SHAPES:
        keys = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(k)]
        pubs = [so.keys(a, b) for a, b in keys]
        pick = rng.integers(0, 4 * k, n)
        A_h = jo.points_mont([p[0] for p in pubs] + [stranger[0]])
        B_h = jo.points_mont([p[1] for p in pubs] + [stranger[1]])
        sel = np.where(pick < k, pick, k)
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        bl_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        bl_h[:, 3] %= np.uint64(jo.R_J >> 192)
        v_h = rng.integers(0, 1 << 62, n, dtype=np.uint64)
        nonce_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        nonce_h[:, 3] %= np.uint64(jo.P >> 192)               # < p
        with torch.cuda.stream(stream):
            nonce = dev(nonce_h)
            R, pk, C, cipher, ok = eng.note_create_batch(dev(r_h), dev(v_h), dev(bl_h), nonce, gb, gpb, dev(A_h[sel]),
                                                         dev(B_h[sel]))
            pos = dev(rng.integers(0, 1 << 62, n, dtype=np.uint64))
            a = dev(jo.jscalar_limbs([x[0] for x in keys]))
            b = dev(jo.jscalar_limbs([x[1] for x in keys]))
        stream.synchronize()
        eng.sync()
        assert host(ok).all()
        Bm = [jo.points_mont([jo.mul(x[1], G)])[0] for x in keys]
        out = {}

        def fused():
            out["f"] = eng.wallet_scan_batch(a, b, R, pk, pos, nonce, cipher, C, gb, gpb)

        def chain():
            rows = []
            for j in range(k):
                owned = eng.stealth_owns_batch(a[j:j + 1], Bm[j], gb, R, pk)
                idx = torch.nonzero(owned).flatten()
                nul, _ = eng_p.nullifier_batch(a[j:j + 1], b[j:j + 1], gpb, R[idx], pos[idx])
                vo, bo, oko = eng.note_open_batch(a[j:j + 1], R[idx], nonce[idx], cipher[idx], C[idx], gb, gpb)
                rows.append((idx, nul, vo, bo, oko, torch.sum(vo * oko)))
            out["c"] = rows

        rr = {"notes": n, "keys": k}
        rr["fused_ms"] = measure(fused)
        rr["chain_ms"] = measure(chain)
        rr["fused_notes_per_s"] = n / (rr["fused_ms"] * 1e-3)
        rr["chain_over_fused"] = rr["chain_ms"] / rr["fused_ms"]
        rr["predicted_chain_over_fused"] = predicted(k)
        stream.synchronize()
        eng.sync()
        owner, nul, value, blinder, opened, totals = (host(x) for x in out["f"])
        w_owner = np.full(n, -1, np.int32)
        w_nul, w_val = np.zeros((n, 4), np.uint64), np.zeros(n, np.uint64)
        w_bl, w_op = np.zeros((n, 4), np.uint64), np.zeros(n, np.uint8)
        w_tot = np.zeros((k, 4), np.uint64)
        for j, (idx, nl, vo, bo, oko, _) in enumerate(out["c"]):
            i = host(idx).astype(np.int64)
            w_owner[i], w_nul[i], w_val[i], w_bl[i], w_op[i] = j, host(nl), host(vo), host(bo), host(oko)
            s = int(host(vo).astype(object).sum()) if len(i) else 0
            w_tot[j] = [s & ((1 << 64) - 1), s >> 64, len(i), int(host(oko).sum())]
        picks = [int(x) for x in rng.choice(n, 2, replace=False)]
        picks[0] = int(np.flatnonzero(pick < k)[0])             # one owned note among the samples

        def note(i):
            """note i as the model takes it: canonical ints"""
            fr = jo.points_from_mont
            Ri, pki, Ci = (fr(host(t)[i:i + 1])[0] for t in (R, pk, C))
            return Ri, pki, int(host(pos)[i]), fr_int(nonce_h[i]), [fr_int(c) for c in host(cipher)[i]], Ci

        model = wo.scan(keys, [note(i) for i in picks], Gp)
        parity[name] = {
            "all_notes_created": True,
            "owned_fraction": float((owner >= 0).mean()),
            "equals_chain": bool(np.array_equal(owner, w_owner) and np.array_equal(nul, w_nul)
                                 and np.array_equal(value, w_val) and np.array_equal(blinder, w_bl)
                                 and np.array_equal(opened, w_op) and np.array_equal(totals, w_tot)),
            "samples_match_model": bool([int(owner[i]) for i in picks] == model["owner"]
                                        and [int(value[i]) for i in picks] == model["value"]
                                        and [int(opened[i]) for i in picks] == model["opened"]),
        }
        res[name] = rr
        del R, pk, C, cipher, ok, nonce, pos, a, b, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(v["equals_chain"] and v["samples_match_model"] for v in parity.values())
    line = {"metric": "wallet_scan_notes_per_s", "value": res["n20_k4"]["fused_notes_per_s"], "unit": "notes/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_wallet_scan_batch vs per key stealth_owns_batch + gather + nullifier_batch + "
                                   "note_open_batch + sum; device buffers, a quarter of the notes owned"},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng_p.close()
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
