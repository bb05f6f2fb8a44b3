#!/usr/bin/env python
"""Benchmark of the double-key Schnorr signatures (p252_schnorr_sign_double_batch, p252_schnorr_verify_double_batch,
p252_note_sign_double_batch) against the single-key calls (p252_schnorr_sign_batch, p252_schnorr_verify_batch).

    python tools/bench_schnorr_double.py [--steps K] [--warmup W] [--items N] > schnorr_double.json

All buffers device-resident, inputs seeded, one key for the batch (n_secret = n_public = 1); G' is a seeded point of the
prime-order subgroup.  For N items (default 2^20) and for 64 items (the latency regime):
  sign_double, verify_double and note sign (one wallet key, notes made by p252_stealth_address_batch), and
  p252_schnorr_sign_batch / p252_schnorr_verify_batch on the same keys, nonces and messages.
The ratios the product counts predict (DESIGN.md section 4), printed beside the measured ones: verify_double / verify
~ 2 (2 x 2850 products; the challenge's one extra permutation is small next to them); sign_double / sign ~ 2 (two
fixed-base walks of 866 products against one; the digest and the two order products are small); note sign / sign_double
~ (1732 + 2819 + 866) / 1732 = 3.1, plus two digests.  Each arm is timed with CUDA events on the engine's stream over
--steps calls after --warmup calls.  The line carries the device, its power limit and SM clocks sampled during the run,
and in-run parity: every signature verifies (double under (PK, PK'), single under PK), sampled rows of sign_double and
of the note signer against the Python model (tests/schnorr_double_oracle.py), and the single-key R equals the double
R.  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
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

PREDICTED = {"verify_double_over_verify": 2.0, "sign_double_over_sign": 2.0,
             "note_sign_over_sign_double": (1732 + 2819 + 866) / 1732}


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
    import schnorr_double_oracle as sdo
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

    rng = np.random.default_rng(16)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    Gp = jo.random_subgroup_point(rng)
    gpb = jo.points_mont([Gp])[0]
    sk0 = jo.random_secret(rng)
    PK, PKp = sdo.key_pair(sk0, Gp)
    a0, b0 = jo.random_secret(rng), jo.random_secret(rng)
    A0, B0 = so.keys(a0, b0)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("items", args.items), ("small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        m_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        m_h[:, 3] %= np.uint64(jo.P >> 192)                   # < p
        with torch.cuda.stream(stream):
            sk, r, m = dev(jo.jscalar_limbs([sk0])), dev(r_h), dev(m_h)
            pk, pkp = dev(jo.points_mont([PK])), dev(jo.points_mont([PKp]))
            al, bl = dev(jo.jscalar_limbs([a0])), dev(jo.jscalar_limbs([b0]))
            Rn, note_pk, _ = eng.stealth_address_batch(dev(r_h[::-1]), gb, dev(jo.points_mont([A0])),
                                                       dev(jo.points_mont([B0])))
        stream.synchronize()
        out = {}

        def sign_double():
            out["sd"] = eng.schnorr_sign_double_batch(sk, r, m, gb, gpb)

        def verify_double():
            u, R, Rp, _ = out["sd"]
            out["vd"] = eng.schnorr_verify_double_batch(pk, pkp, u, R, Rp, m, gb, gpb)
            out["vd_n"] = eng.last_schnorr_double_verified()

        def note_sign():
            out["ns"] = eng.note_sign_double_batch(al, bl, Rn, r, m, gb, gpb)

        def sign():
            out["s"] = eng.schnorr_sign_batch(sk, r, m, gb)

        def verify():
            u, R, _ = out["s"]
            out["v"] = eng.schnorr_verify_batch(pk, u, R, m, gb)
            out["v_n"] = eng.last_schnorr_verified()

        rr = {"items": n}
        for arm, fn in (("sign_double", sign_double), ("verify_double", verify_double), ("note_sign", note_sign),
                        ("sign", sign), ("verify", verify)):
            rr[arm + "_ms"] = measure(fn)
            rr[arm + "_per_s"] = n / (rr[arm + "_ms"] * 1e-3)
        rr["verify_double_over_verify"] = rr["verify_double_ms"] / rr["verify_ms"]
        rr["sign_double_over_sign"] = rr["sign_double_ms"] / rr["sign_ms"]
        rr["note_sign_over_sign_double"] = rr["note_sign_ms"] / rr["sign_double_ms"]
        stream.synchronize()
        eng.sync()
        u, R, Rp, ok = (host(x) for x in out["sd"])
        nu, nR, nRp, npk, nok = (host(x) for x in out["ns"])
        nv = eng.schnorr_verify_double_batch(note_pk, dev(npk), dev(nu), dev(nR), dev(nRp), m, gb, gpb)
        torch.cuda.synchronize()
        picks = rng.choice(n, min(n, 3), replace=False)
        rn = jo.points_from_mont(host(Rn))
        check = {"all_signed": bool(ok.all()) and bool(nok.all()) and bool(host(out["s"][2]).all()),
                 "double_verifies": out["vd_n"] == n, "single_verifies": out["v_n"] == n,
                 "note_signatures_verify_under_note_pk": bool(host(nv).all()),
                 "single_R_equals_double_R": bool(np.array_equal(host(out["s"][1]), R))}
        sd_model, ns_model = True, True
        for i in picks:
            mi = int(pb.scalar.from_mont(m_h[i]))
            uu, RR, RRp = sdo.sign_double(sk0, s_int(r_h[i]), mi, Gp)
            sd_model &= s_int(u[i]) == uu and jo.points_from_mont(R[i:i + 1])[0] == RR
            (nuu, _, _), npp = sdo.note_sign_double(a0, b0, rn[i], s_int(r_h[i]), mi, Gp)
            ns_model &= s_int(nu[i]) == nuu and jo.points_from_mont(npk[i:i + 1])[0] == npp
        check["sign_double_rows_match_model"] = bool(sd_model)
        check["note_sign_rows_match_model"] = bool(ns_model)
        parity[name] = check
        res[name] = rr
        del sk, r, m, pk, pkp, al, bl, Rn, note_pk, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "schnorr_verify_double_per_s", "value": res["items"]["verify_double_per_s"], "unit": "signatures/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_schnorr_sign_double_batch, p252_schnorr_verify_double_batch, "
                                   "p252_note_sign_double_batch vs p252_schnorr_sign_batch, p252_schnorr_verify_batch; "
                                   "device buffers, one key, %d items per call (and 64)" % args.items},
            "workloads": res, "predicted_ratios_from_product_counts": PREDICTED, "clocks": clocks, "device": props.name,
            "power_limit_w": clocks.get("power_limit_w"), "parity": "ok" if all_ok else "MISMATCH",
            "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
