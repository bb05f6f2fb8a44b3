#!/usr/bin/env python
"""Benchmark of the point compression: p252_points_from_bytes / p252_points_to_bytes, and the share decoding adds to the
wallet scan when the notes arrive as wire bytes.

    python tools/bench_points.py [--steps K] [--warmup W] [--items N] > points.json

Inputs seeded; the points are [k] G for random k (p252_fixed_base_batch), the notes are made by
p252_stealth_address_batch for two receivers, a quarter of them for the scanning receiver (view key a, spend key B):
  (a) N decompressions (default 2^20), device buffers, and (b) N compressions, device buffers
  (c) (a) and (b) with host buffers (numpy in, numpy out: staged through the library's chunk pipeline)
  (d) the scan from wire bytes: decompress R and note_pk on the device, then p252_stealth_owns_batch, all device buffers,
      against (e) p252_stealth_owns_batch alone on the same decoded notes
Device arms are timed with CUDA events on the engine's stream over --steps calls after --warmup calls; host arms, which
return only when their copies back are done, with the host clock.  The line carries the device, its power limit and SM
clocks sampled during the run, and in-run parity: sampled decoded and encoded rows against the Python model
(tests/points_oracle.py), host and device results equal, and the owned flags of (d) equal to (e)'s and to the
construction.  Writes nothing in the repository tree.  The clock sampler is bench.py's, imported unchanged.
"""
import argparse
import json
import os
import sys
import time

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
    import points_oracle as po
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

    def timed_host(fn, reps):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) * 1e3 / reps

    def measure(fn, clock=timed):
        if args.warmup:
            clock(fn, args.warmup)
        return clock(fn, args.steps)

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()

    def host(t):
        a = t.cpu().numpy()
        return a.view(np.uint64) if a.dtype == np.int64 else a

    n = args.items
    rng = np.random.default_rng(15)
    G = jo.GENERATOR
    gb = jo.points_mont([G])[0]
    keys = [(jo.random_secret(rng), jo.random_secret(rng)) for _ in range(2)]
    pub = [so.keys(a, b) for a, b in keys]
    a0, B0m = keys[0][0], jo.points_mont([pub[0][1]])[0]
    k_h = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    k_h[:, 3] %= np.uint64(jo.R_J >> 192)                     # < r_J
    who = (rng.random(n) >= 0.25).astype(np.int64)            # receiver 0 (the scanner) for about a quarter
    sampler = ClockSampler(0)
    sampler.start()
    with torch.cuda.stream(stream):
        pts, okp = eng.fixed_base_batch(dev(k_h), gb)
        enc, oke = eng.points_to_bytes(pts)
        R, pk, okn = eng.stealth_address_batch(dev(k_h), gb, dev(jo.points_mont([p[0] for p in pub])[who]),
                                               dev(jo.points_mont([p[1] for p in pub])[who]))
        Rb, okRb = eng.points_to_bytes(R)
        Pb, okPb = eng.points_to_bytes(pk)
        va = dev(jo.jscalar_limbs([a0]))
        dec = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
        R2 = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
        P2 = torch.empty((n, 2, 4), dtype=torch.int64, device="cuda")
        owned = torch.empty((n,), dtype=torch.uint8, device="cuda")
        owned2 = torch.empty((n,), dtype=torch.uint8, device="cuda")
    stream.synchronize()
    eng.sync()
    setup_ok = all(bool(host(x).all()) for x in (okp, oke, okn, okRb, okPb))
    enc_h, pts_h = host(enc).view(np.uint8).reshape(n, 32).copy(), host(pts)
    out = {}

    def decompress():
        out["dec"], out["okd"] = eng.points_from_bytes(enc, out=dec, async_=True)

    def compress():
        b, out["okc"] = eng.points_to_bytes(dec, async_=True)
        out["enc"] = b

    def decompress_host():
        out["dec_h"], out["okd_h"] = eng.points_from_bytes(enc_h)

    def compress_host():
        out["enc_h"], out["okc_h"] = eng.points_to_bytes(pts_h)

    def scan_from_bytes():
        eng.points_from_bytes(Rb, out=R2, async_=True)
        eng.points_from_bytes(Pb, out=P2, async_=True)
        eng.stealth_owns_batch(va, B0m, gb, R2, P2, out=owned, async_=True)

    def scan():
        eng.stealth_owns_batch(va, B0m, gb, R2, P2, out=owned2, async_=True)

    res = {"items": n}
    res["from_bytes_device_ms"] = measure(decompress)
    res["from_bytes_device_points_per_s"] = n / (res["from_bytes_device_ms"] * 1e-3)
    res["to_bytes_device_ms"] = measure(compress)
    res["to_bytes_device_points_per_s"] = n / (res["to_bytes_device_ms"] * 1e-3)
    res["from_bytes_host_ms"] = measure(decompress_host, timed_host)
    res["from_bytes_host_points_per_s"] = n / (res["from_bytes_host_ms"] * 1e-3)
    res["to_bytes_host_ms"] = measure(compress_host, timed_host)
    res["to_bytes_host_points_per_s"] = n / (res["to_bytes_host_ms"] * 1e-3)
    res["scan_from_bytes_ms"] = measure(scan_from_bytes)
    res["scan_alone_ms"] = measure(scan)
    res["decode_share_of_scan_from_bytes"] = 1 - res["scan_alone_ms"] / res["scan_from_bytes_ms"]
    stream.synchronize()
    eng.sync()
    clocks = sampler.stop()
    rows = rng.choice(n, min(n, 8), replace=False)
    dec_d = host(out["dec"])
    own, own2 = host(owned), host(owned2)
    parity = {
        "setup_ok": setup_ok,
        "decoded_rows_match_model": jo.points_from_mont(dec_d[rows]) == [po.decode(enc_h[i].tobytes()) for i in rows],
        "decoded_equals_points": bool(np.array_equal(dec_d, pts_h)) and bool(host(out["okd"]).all()),
        "encoded_rows_match_model": all(host(out["enc"]).view(np.uint8).reshape(n, 32)[i].tobytes() ==
                                        po.encode(jo.points_from_mont(pts_h[i:i + 1])[0]) for i in rows),
        "host_equals_device": bool(np.array_equal(out["dec_h"], dec_d)) and bool(np.array_equal(out["enc_h"], enc_h)) and
        bool(out["okd_h"].all()) and bool(out["okc_h"].all()),
        "scan_from_bytes_equals_scan_and_construction": bool(np.array_equal(own, own2)) and
        bool(np.array_equal(own, (who == 0).astype(np.uint8)))}
    props = torch.cuda.get_device_properties(0)
    line = {"metric": "points_from_bytes_per_s", "value": res["from_bytes_device_points_per_s"], "unit": "points/s",
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic, seeded",
            "config": {"workload": "p252_points_from_bytes / p252_points_to_bytes on device and host buffers; "
                                   "2 x p252_points_from_bytes + p252_stealth_owns_batch vs p252_stealth_owns_batch alone; "
                                   "%d points per call" % n},
            "workloads": res, "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if all(parity.values()) else "MISMATCH", "parity_checks": parity}
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
