#!/usr/bin/env python
"""Benchmark of the Schnorr signatures over JubJub: verification (p252_schnorr_verify_batch) and signing
(p252_schnorr_sign_batch).

    python tools/bench_schnorr.py [--steps K] [--warmup W] [--items N] > schnorr.json

All buffers device-resident, inputs seeded, base G.  The signatures are made by the signing call, by four keys:
  (a) verification of N signatures (default 2^20), n_public = n (one key per signature)
  (b) verification of N signatures of one key, n_public = 1
  (c) signing of N messages with one sk (fresh nonces)
  (d) the composition a caller has without verification, on the signatures of (a): the rows [R.u, R.v, m] packed with
      torch, p252_hash_batch_truncated (c), p252_dhke_batch (n, n) of (c, PK) and p252_fixed_base_batch (u).  Only the
      device part is timed; the point addition [u] G + [c] PK and the comparison with R are MISSING from it (the library
      has no device call for them), so it is a lower bound for that path
  (e) signing and verification of 64 items (the latency regime)
Each arm is timed with CUDA events on the engine's stream over --steps calls after --warmup calls.  The line carries the
device, its power limit and SM clocks sampled during the run, and in-run parity: sampled signatures against the Python
model (tests/schnorr_oracle.py), every signature of (c) verified, and the verified counts of (a) and (b).  Writes
nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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
    import hades_oracle as ho
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    import schnorr_oracle as so
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
    gb = jo.points_mont([jo.GENERATOR])[0]
    sks = [jo.random_secret(rng) for _ in range(4)]
    pks = [so.public_key(k) for k in sks]
    rinv = pow(ho.R, -1, jo.P)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("abcd_items", args.items), ("e_small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        m_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        m_h[:, 3] %= np.uint64(jo.P >> 192)                   # < p
        who = rng.integers(0, 4, n)
        with torch.cuda.stream(stream):
            r, m = dev(r_h), dev(m_h)
            sk_n = dev(jo.jscalar_limbs(sks)[who])
            sk_1 = dev(jo.jscalar_limbs(sks[:1]))
            pk_n = dev(jo.points_mont(pks)[who])
            pk_1 = dev(jo.points_mont(pks[:1]))
            u_a = torch.empty((n, 4), dtype=torch.int64, device="cuda")
            R_a = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            u_c = torch.empty((n, 4), dtype=torch.int64, device="cuda")
            R_c = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            ver = torch.empty((n,), dtype=torch.uint8, device="cuda")
            c = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
            cP = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
            uG = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
        stream.synchronize()
        _, _, ok_a = eng.schnorr_sign_batch(sk_n, r, m, gb, u_out=u_a, R_out=R_a)   # the signatures of (a)
        ok_a = bool(host(ok_a).all())
        out = {}

        def verify_n():
            out["va"] = eng.schnorr_verify_batch(pk_n, u_a, R_a, m, gb, out=ver)

        def verify_1():
            out["vb"] = eng.schnorr_verify_batch(pk_1, u_c, R_c, m, gb, out=ver)

        def sign_1():
            out["ok_c"] = eng.schnorr_sign_batch(sk_1, r, m, gb, u_out=u_c, R_out=R_c)[2]

        def composition():
            rows = torch.cat([R_a, m.view(n, 1, 4)], dim=1)
            eng.hash_batch_truncated(pb.Domain.Other, rows, out=c, async_=True)
            eng.dhke_batch(c.view(n, 4), pk_n, out=cP, async_=True)
            eng.fixed_base_batch(u_a, gb, out=uG, async_=True)

        rr = {"items": n}
        rr["c_sign_ms"] = measure(sign_1)
        rr["c_sign_per_s"] = n / (rr["c_sign_ms"] * 1e-3)
        rr["a_verify_n_public_n_ms"] = measure(verify_n)
        rr["a_verify_per_s"] = n / (rr["a_verify_n_public_n_ms"] * 1e-3)
        a_verified = eng.last_schnorr_verified()
        rr["b_verify_n_public_1_ms"] = measure(verify_1)
        rr["b_verify_per_s"] = n / (rr["b_verify_n_public_1_ms"] * 1e-3)
        b_verified = eng.last_schnorr_verified()
        if n > 64:
            rr["d_composition_device_ms"] = measure(composition)
            rr["d_composition_missing"] = "the addition [u] G + [c] PK and the comparison with R"
            rr["a_speedup_over_d"] = rr["d_composition_device_ms"] / rr["a_verify_n_public_n_ms"]
        stream.synchronize()
        eng.sync()
        rows = rng.choice(n, min(n, 4), replace=False)
        uh, Rh, uch, Rch = host(u_a), host(R_a), host(u_c), host(R_c)
        want = [so.sign(sks[who[i]], s_int(r_h[i]), s_int(m_h[i]) * rinv % jo.P) for i in rows]
        want_c = [so.sign(sks[0], s_int(r_h[i]), s_int(m_h[i]) * rinv % jo.P) for i in rows[:2]]
        parity[name] = {
            "a_rows_match_model": ok_a and [s_int(uh[i]) for i in rows] == [w[0] for w in want] and
            jo.points_from_mont(Rh[rows]) == [w[1] for w in want],
            "c_rows_match_model": [s_int(uch[i]) for i in rows[:2]] == [w[0] for w in want_c] and
            jo.points_from_mont(Rch[rows[:2]]) == [w[1] for w in want_c],
            "a_all_verified": a_verified == n,
            "c_all_sign_ok_and_verify_under_pk": bool(host(out["ok_c"]).all()) and b_verified == n and
            bool(host(out["vb"]).all())}
        res[name] = rr
        del r, m, sk_n, sk_1, pk_n, pk_1, u_a, R_a, u_c, R_c, ver, c, cP, uG, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "schnorr_verify_per_s", "value": res["abcd_items"]["a_verify_per_s"], "unit": "signatures/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_schnorr_verify_batch (n_public = n and 1), p252_schnorr_sign_batch (one sk) vs "
                                   "p252_hash_batch_truncated + p252_dhke_batch (n, n) + p252_fixed_base_batch (device "
                                   "part only, no addition or comparison); device buffers, %d items per call (e: 64)"
                                   % args.items},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all_ok else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
