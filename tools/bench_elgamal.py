#!/usr/bin/env python
"""Benchmark of JubJub ElGamal and the encrypted note sender (p252_elgamal_encrypt_batch, p252_elgamal_decrypt_batch,
p252_note_sender_encrypt_batch, p252_note_sender_decrypt_batch) against the chains of existing calls a caller would
otherwise run.

    python tools/bench_elgamal.py [--steps K] [--warmup W] [--items N] > elgamal.json

All buffers device-resident, inputs seeded: per-item keys PK = [sk] G and messages M = [m] G made on the device, one
receiver (a, b) whose stealth notes carry the sender fields, and a seeded G' for the nullifier yardstick.  For N items
(default 2^20) and for 64 items (the latency regime), each arm against its chain:
  encrypt         vs  p252_fixed_base_batch(r, G) + p252_dhke_batch(r, PK)
  sender encrypt  vs  twice that chain (r_A and r_B)
  decrypt         vs  p252_dhke_batch(sk, c1)
  sender decrypt  vs  p252_nullifier_batch + 2 x p252_dhke_batch: a yardstick for the same secret-key work (one key
                      exchange and hash per note, then two variable-base walks), not a chain that computes the sender
The chains are favoured: the point additions and subtractions they would still need are left out (the library has no call
for them), and the nullifier yardstick runs on a second engine so that G' and G keep their tables.  The ratios the
product counts predict (DESIGN.md section 4; a Hades permutation counted as 365 products) are printed beside the measured
ones.  Each arm is timed with CUDA events on the engines' shared stream over --steps calls after --warmup calls.  The line
carries the device, its power limit and SM clocks sampled during the run, and in-run parity: c1 equals the fixed-base
call's rows and c2 with M = the identity the key exchange's, every message and every sender decrypts back, the sender
call equals two encrypt calls, and sampled rows equal the Python model (tests/elgamal_oracle.py).  Writes nothing in the
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

FB, DHKE, NUL_KEY, PERM = 866, 2819, 867, 365
ENC, SENDER_ENC, DEC, SENDER_DEC = 3284, 6022, 2832, 5699
PREDICTED = {"encrypt_chain_over_encrypt": (FB + DHKE) / ENC,
             "sender_encrypt_chain_over_sender_encrypt": 2 * (FB + DHKE) / SENDER_ENC,
             "decrypt_chain_over_decrypt": DHKE / DEC,
             "sender_decrypt_yardstick_over_sender_decrypt": (DHKE + PERM + NUL_KEY + PERM + 2 * DHKE) / (DHKE + PERM + SENDER_DEC)}


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
    import elgamal_oracle as eo
    import jubjub_oracle as jo
    import poseidon252_b200 as pb
    import stealth_oracle as so
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    eng_p = pb.Engine(0, stream=stream.cuda_stream)          # the nullifier yardstick's table of G'

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

    def scalars(n):
        x = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        x[:, 3] %= np.uint64(jo.R_J >> 192)                   # < r_J
        return x

    rng = np.random.default_rng(23)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    gpb = jo.points_mont([jo.random_subgroup_point(rng)])[0]
    a0, b0 = jo.random_secret(rng), jo.random_secret(rng)
    A0, B0 = so.keys(a0, b0)
    sampler = ClockSampler(0)
    sampler.start()
    res, parity = {}, {}
    for name, n in (("items", args.items), ("small_64_items", 64)):
        sk_h, m_h, r_h, rb_h, rn_h = scalars(n), scalars(n), scalars(n), scalars(2 * n), scalars(n)
        with torch.cuda.stream(stream):
            sk, r, rb, rn = dev(sk_h), dev(r_h), dev(rb_h.reshape(n, 2, 4)), dev(rn_h)
            PK, _ = eng.fixed_base_batch(sk, gb)
            M, _ = eng.fixed_base_batch(dev(m_h), gb)
            ident = dev(np.tile(jo.points_mont([jo.IDENTITY]), (n, 1, 1)))
            A, B = dev(jo.points_mont([A0])), dev(jo.points_mont([B0]))
            a, b = dev(jo.jscalar_limbs([a0])), dev(jo.jscalar_limbs([b0]))
            R, note_pk, _ = eng.stealth_address_batch(rn, gb, A, B)
            pos = torch.arange(n, dtype=torch.int64, device="cuda")
            rA, rB = rb[:, 0].contiguous(), rb[:, 1].contiguous()
        stream.synchronize()
        out = {}

        def encrypt():
            out["e"] = eng.elgamal_encrypt_batch(PK, M, r, gb)

        def encrypt_chain():
            out["ec"] = (eng.fixed_base_batch(r, gb), eng.dhke_batch(r, PK))

        def sender_encrypt():
            out["s"] = eng.note_sender_encrypt_batch(note_pk, M, PK, rb, gb)

        def sender_encrypt_chain():
            out["sc"] = (eng.fixed_base_batch(rA, gb), eng.dhke_batch(rA, note_pk), eng.fixed_base_batch(rB, gb),
                         eng.dhke_batch(rB, note_pk))

        def decrypt():
            c1, c2, _ = out["e"]
            out["d"] = eng.elgamal_decrypt_batch(sk, c1, c2)

        def decrypt_chain():
            out["dc"] = eng.dhke_batch(sk, out["e"][0])

        def sender_decrypt():
            out["sd"] = eng.note_sender_decrypt_batch(a, b, R, note_pk, out["s"][0], gb)

        def sender_decrypt_yardstick():
            enc = out["s"][0]
            out["sy"] = (eng_p.nullifier_batch(a, b, gpb, R, pos), eng.dhke_batch(sk, enc[:, 0].contiguous()),
                         eng.dhke_batch(sk, enc[:, 2].contiguous()))

        rr = {"items": n}
        for arm, fn in (("encrypt", encrypt), ("encrypt_chain", encrypt_chain), ("sender_encrypt", sender_encrypt),
                        ("sender_encrypt_chain", sender_encrypt_chain), ("decrypt", decrypt), ("decrypt_chain", decrypt_chain),
                        ("sender_decrypt", sender_decrypt), ("sender_decrypt_yardstick", sender_decrypt_yardstick)):
            rr[arm + "_ms"] = measure(fn)
            rr[arm + "_per_s"] = n / (rr[arm + "_ms"] * 1e-3)
        for arm in ("encrypt", "sender_encrypt", "decrypt"):
            rr[arm + "_chain_over_" + arm] = rr[arm + "_chain_ms"] / rr[arm + "_ms"]
        rr["sender_decrypt_yardstick_over_sender_decrypt"] = rr["sender_decrypt_yardstick_ms"] / rr["sender_decrypt_ms"]
        with torch.cuda.stream(stream):
            i1, i2, oki = eng.elgamal_encrypt_batch(PK, ident, r, gb)
            a1, a2, oka = eng.elgamal_encrypt_batch(note_pk, M, rA, gb)
            b1, b2, okb = eng.elgamal_encrypt_batch(note_pk, PK, rB, gb)
        stream.synchronize()
        eng.sync()
        c1, c2, oke = out["e"]
        (f, okf), (s, oks) = out["ec"]
        msg, okd = out["d"]
        enc, oks2 = out["s"]
        gA, gB, oksd = out["sd"]
        picks = rng.choice(n, min(n, 3), replace=False)
        hPK, hM = jo.points_from_mont(host(PK)[picks]), jo.points_from_mont(host(M)[picks])
        hc1, hc2 = jo.points_from_mont(host(c1)[picks]), jo.points_from_mont(host(c2)[picks])
        model = all((hc1[k], hc2[k]) == eo.encrypt(hPK[k], hM[k], s_int(r_h[i])) for k, i in enumerate(picks))
        check = {"all_valid": all(bool(host(x).all()) for x in (oke, okf, oks, oki, oka, okb, okd, oks2)),
                 "c1_equals_fixed_base": bool(torch.equal(c1, f) and torch.equal(i1, f)),
                 "c2_of_identity_equals_dhke": bool(torch.equal(i2, s)),
                 "every_message_decrypts": bool(torch.equal(msg, M)),
                 "sender_equals_two_encrypts": bool(torch.equal(enc, torch.stack([a1, a2, b1, b2], dim=1))),
                 "every_sender_recovered": bool(host(oksd).all()) and bool(torch.equal(gA, M) and torch.equal(gB, PK)),
                 "encryptions_match_model": bool(model)}
        parity[name] = check
        res[name] = rr
        del sk, r, rb, rn, PK, M, ident, A, B, a, b, R, note_pk, pos, rA, rB, out
        torch.cuda.empty_cache()
    eng.sync()
    clocks = sampler.stop()
    props = torch.cuda.get_device_properties(0)
    all_ok = all(all(v.values()) for v in parity.values())
    line = {"metric": "elgamal_encrypt_per_s", "value": res["items"]["encrypt_per_s"], "unit": "items/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_elgamal_{encrypt,decrypt}_batch, p252_note_sender_{encrypt,decrypt}_batch vs the "
                                   "chains of existing calls; device buffers, per-item keys, one receiver, %d items per "
                                   "call (and 64)" % args.items},
            "workloads": res, "predicted_ratios_from_product_counts": PREDICTED, "clocks": clocks, "device": props.name,
            "power_limit_w": clocks.get("power_limit_w"), "parity": "ok" if all_ok else "MISMATCH",
            "parity_checks": parity}
    eng_p.close()
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
