"""Developer timing helper: latency of small Merkle4 digest batches -- lane-split kernel vs throughput kernel vs the
CPU port (oracle/hades_ref.c, test infrastructure) -- device-resident buffers, CUDA events, median of 20.
    python tools/small_batch.py > small_batch.json"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import numpy as np
import torch

import poseidon252_b200 as pb
from poseidon252_b200.scalar import random_limbs_fast, to_mont


def gpu_ms(eng, st, x, out, reps=20):
    for _ in range(3):
        pb.Hash.digest_batch(pb.Domain.Merkle4, x, engine=eng, out=out, async_=True)
    st.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            a.record(st)
            pb.Hash.digest_batch(pb.Domain.Merkle4, x, engine=eng, out=out, async_=True)
            b.record(st)
        st.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    import c_oracle
    import hades_oracle as o
    st = torch.cuda.Stream()
    eng = pb.Engine(0, stream=st.cuda_stream)
    rng = np.random.default_rng(0)
    tag = to_mont(o.hash_to_scalar(o.tag_input([o.Absorb(4), o.Squeeze(1)], o.Domain.Merkle4)))
    threads = len(os.sched_getaffinity(0))
    rows = []
    for n in (1, 6, 32, 256, 1024, 2048, 4096, 6144, 8192, 16384, 65536):
        h = random_limbs_fast(rng, (n, 4))
        with torch.cuda.stream(st):
            x = torch.from_numpy(h.view(np.int64)).cuda()
            out = torch.empty((n, 1, 4), dtype=torch.int64, device="cuda")
        st.synchronize()
        eng.set_small_batch_max(1 << 30)
        coop = gpu_ms(eng, st, x, out)
        a = out.cpu().numpy().copy()
        eng.set_small_batch_max(0)
        main_ms = gpu_ms(eng, st, x, out)
        assert np.array_equal(a, out.cpu().numpy())
        th = 1 if n < 64 else threads
        c_oracle.digest(tag, h, 4, 1, threads=th)
        t0 = time.perf_counter()
        for _ in range(3):
            c_oracle.digest(tag, h, 4, 1, threads=th)
        cpu_ms = (time.perf_counter() - t0) / 3 * 1e3
        rows.append({"n": n, "lane_split_ms": round(coop, 4), "throughput_kernel_ms": round(main_ms, 4),
                     "cpu_port_ms": round(cpu_ms, 4), "cpu_threads": th})
        print(rows[-1], file=sys.stderr)
    print(json.dumps({"workload": "Merkle4 digests, device-resident, median of 20 launches (CUDA events)", "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
