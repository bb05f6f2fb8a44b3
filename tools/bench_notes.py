#!/usr/bin/env python
"""Benchmark of the note value calls (p252_value_commit_batch, p252_note_create_batch, p252_note_open_batch) against the
chains of existing calls a caller would otherwise run.

    python tools/bench_notes.py [--steps K] [--warmup W] [--items N] > notes.json

All buffers device-resident, inputs seeded, one receiver (A, B) and one view key for the batch; G' is a seeded point of
the prime-order subgroup.  For N items (default 2^20) and for 64 items (the latency regime), each arm against its chain:
  commit  vs  p252_fixed_base_batch(v, G) + p252_fixed_base_batch(blinder, G')
  create  vs  p252_stealth_address_batch + p252_encrypt_batch_ephemeral([Fr(v), Fr(blinder)]) + the two fixed-base calls
  open    vs  p252_decrypt_batch_dhke (L = 2) + p252_value_commit_batch
The chains are favoured: the two fixed-base calls run on two engines (one table each, no rebuild), the point addition of
the commitment is left out (the library has no call for it), and the message rows of the sender and the (v, blinder) of
the wallet's check are given, not converted.  The ratios the product counts predict (DESIGN.md section 4) are printed
beside the measured ones.  Each arm is timed with CUDA events on the engines' shared stream over --steps calls after
--warmup calls.  The line carries the device, its power limit and SM clocks sampled during the run, and in-run parity:
every note opens with its (v, blinder), the created R, note_pk, commitment and cipher equal the chain's, and sampled
commitments equal the Python model (tests/note_oracle.py).  Writes nothing in the repository tree.  The clock sampler is
bench.py's, imported unchanged.
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

FB, DHKE, DERIVE, COMMIT, CREATE_VALUE, OPEN_VALUE = 866, 2819, 879, 985, 987, 568
PREDICTED = {"commit_chain_over_commit": 2 * FB / COMMIT,
             "create_chain_over_create": (FB + DHKE + DERIVE + FB + DHKE + 2 * FB) / (FB + DHKE + CREATE_VALUE + DERIVE),
             "open_chain_over_open": (DHKE + COMMIT) / (DHKE + OPEN_VALUE)}


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
    import note_oracle as nto
    import poseidon252_b200 as pb
    import stealth_oracle as so
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    eng_p = pb.Engine(0, stream=stream.cuda_stream)          # the chains' second fixed-base table (G')

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

    rng = np.random.default_rng(17)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    Gp = jo.random_subgroup_point(rng)
    gpb = jo.points_mont([Gp])[0]
    a0, b0 = jo.random_secret(rng), jo.random_secret(rng)
    A0, B0 = so.keys(a0, b0)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("items", args.items), ("small_64_items", 64)):
        r_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        r_h[:, 3] %= np.uint64(jo.R_J >> 192)                 # < r_J
        b_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        b_h[:, 3] %= np.uint64(jo.R_J >> 192)
        v_h = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
        nonce_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        nonce_h[:, 3] %= np.uint64(jo.P >> 192)               # < p
        vrow_h = np.zeros((n, 4), dtype=np.uint64)
        vrow_h[:, 0] = v_h
        with torch.cuda.stream(stream):
            r, b, v, nonce, vrow = dev(r_h), dev(b_h), dev(v_h), dev(nonce_h), dev(vrow_h)
            A, B, a = dev(jo.points_mont([A0])), dev(jo.points_mont([B0])), dev(jo.jscalar_limbs([a0]))
            # the sender's message rows [Fr(v), Fr(blinder)], made once (the chain is not charged for them)
            msg = torch.stack([eng.scalars_from_bytes(x)[0] for x in (vrow, b)], dim=1).contiguous()
        stream.synchronize()
        out = {}

        def commit():
            out["c"] = eng.value_commit_batch(v, b, gb, gpb)

        def commit_chain():
            out["cc"] = (eng.fixed_base_batch(vrow, gb), eng_p.fixed_base_batch(b, gpb))

        def create():
            out["n"] = eng.note_create_batch(r, v, b, nonce, gb, gpb, A, B)

        def create_chain():
            out["nc"] = (eng.stealth_address_batch(r, gb, A, B), eng.encrypt_batch_ephemeral(msg, r, gb, A, nonce),
                         eng.fixed_base_batch(vrow, gb), eng_p.fixed_base_batch(b, gpb))

        def open_():
            R, _, C, cipher, _ = out["n"]
            out["o"] = eng.note_open_batch(a, R, nonce, cipher, C, gb, gpb)

        def open_chain():
            R, _, C, cipher, _ = out["n"]
            out["oc"] = (eng.decrypt_batch_dhke(cipher, a, R, nonce), eng.value_commit_batch(v, b, gb, gpb))

        rr = {"items": n}
        for arm, fn in (("commit", commit), ("commit_chain", commit_chain), ("create", create),
                        ("create_chain", create_chain), ("open", open_), ("open_chain", open_chain)):
            rr[arm + "_ms"] = measure(fn)
            rr[arm + "_per_s"] = n / (rr[arm + "_ms"] * 1e-3)
        for arm in ("commit", "create", "open"):
            rr[arm + "_chain_over_" + arm] = rr[arm + "_chain_ms"] / rr[arm + "_ms"]
        stream.synchronize()
        eng.sync()
        C, okc = out["c"]
        R, pk, Cn, cipher, okn = out["n"]
        vo, bo, oko = out["o"]
        (R1, pk1, _), (cipher1, _, _) = out["nc"][0], out["nc"][1]
        picks = rng.choice(n, min(n, 3), replace=False)
        hc = jo.points_from_mont(host(C)[picks])
        model = all(hc[k] == nto.commit(int(v_h[i]), s_int(b_h[i]), Gp) for k, i in enumerate(picks))
        check = {"all_valid": bool(host(okc).all()) and bool(host(okn).all()),
                 "every_note_opens": bool(host(oko).all()) and np.array_equal(host(vo), v_h) and np.array_equal(host(bo), b_h),
                 "create_equals_chain": bool(torch.equal(R, R1) and torch.equal(pk, pk1) and torch.equal(cipher, cipher1)
                                             and torch.equal(Cn, C)),
                 "commitments_match_model": bool(model)}
        parity[name] = check
        res[name] = rr
        del r, b, v, nonce, vrow, A, B, a, msg, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "note_create_per_s", "value": res["items"]["create_per_s"], "unit": "notes/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_value_commit_batch, p252_note_create_batch, p252_note_open_batch vs the chains of "
                                   "existing calls; device buffers, one receiver and one view key, %d items per call (and "
                                   "64)" % args.items},
            "workloads": res, "predicted_ratios_from_product_counts": PREDICTED, "clocks": clocks, "device": props.name,
            "power_limit_w": clocks.get("power_limit_w"), "parity": "ok" if all_ok else "MISMATCH",
            "parity_checks": parity}
    eng_p.close()
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
