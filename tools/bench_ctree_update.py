#!/usr/bin/env python
"""Benchmark of compact sparse tree updates (p252_ctree_update): positions anywhere in u64, storage proportional to the
present leaves.

    python tools/bench_ctree_update.py [--steps K] [--warmup W] [--inserts I] [--removals R] > ctree_update.json

Tree: arity 4, height 32 (4^32 = 2^64 positions), 2^22 present positions drawn from a seed over all of u64, on device
buffers laid out for max_leaves = 2^23.  The build is one p252_ctree_update inserting the 2^22 leaves into the empty
tree (timed once after one untimed build).  One timed step = one p252_ctree_update with I inserts (default 2^14; half at
present positions, i.e. overwrites, half anywhere) and R removals of present positions (default 2^12), interleaved,
timed with CUDA events on the engine's stream.  The split of an update into merge, hash and other device time comes from
torch.profiler kernel events over three further updates: hash = the Merkle digest kernels, merge = the per-level merge
(mark, exclusive scans, scatter, count, commit), other = keys, sort, selects and gathers.  Openings per second: one
p252_ctree_open_batch of 2^16 present positions.  Prints one JSON line with the device and its power limit, and an
in-run parity verdict (outside the timed region): level 0 equals a host model of the batches, and 64 sampled openings
hash level by level to the root with the C oracle.  Writes nothing in the repository tree.  The clock sampler and the
device-side input generator are bench.py's.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench import ClockSampler, device_random_scalars, usable_cores  # noqa: E402

MERGE_KERNELS = ("k_ctree_mark", "k_ctree_scatter", "k_ctree_count", "k_ctree_commit", "DeviceScan")


def model_apply(keys, vals, pos, op, new_vals):
    """host model of one batch: sorted keys (uint64) and their values (k, 4) -> the same after the batch"""
    import numpy as np
    rev = pos[::-1]
    u, first = np.unique(rev, return_index=True)                 # last operation per position
    last = pos.shape[0] - 1 - first
    keep = ~np.isin(keys, u)
    ins = op[last] == 0
    k2 = np.concatenate([keys[keep], u[ins]])
    v2 = np.concatenate([vals[keep], new_vals[last[ins]]])
    order = np.argsort(k2, kind="stable")
    return k2[order], v2[order]


def ctree_update_line(args, eng, torch, stream, local):
    import numpy as np
    import mtree_oracle
    from poseidon252_b200 import merkle
    arity, height, n0, max_leaves = 4, 32, 1 << 22, 1 << 23
    n_ins, n_rem = args.inserts, args.removals
    rng = np.random.default_rng(201)
    keys = np.unique(rng.integers(0, 1 << 64, n0 + 4096, dtype=np.uint64))
    keys = rng.permutation(keys)[:n0]
    tree = merkle.CompactTree(arity, height, max_leaves, engine=eng, device=local)
    init_vals = device_random_scalars(torch, n0, 202)
    init_pos = torch.from_numpy(keys.view(np.int64)).to(stream.device)

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / reps

    def build():
        with torch.cuda.stream(stream):
            tree.keys.zero_()
            tree.values.zero_()
            tree.count.zero_()
        return timed(lambda: eng.ctree_update(tree, init_pos, values=init_vals, async_=True), 1)

    build()
    build_ms = build()
    assert eng.last_ctree_rejected() == 0
    order = np.argsort(keys)
    m_keys, m_vals = keys[order], init_vals.cpu().numpy().view(np.uint64)[order]

    total = args.warmup + args.steps + 3
    plan = []
    for i in range(total):
        ins = np.where(rng.random(n_ins) < 0.5, rng.choice(m_keys, n_ins), rng.integers(0, 1 << 64, n_ins, dtype=np.uint64))
        rem = rng.choice(m_keys, n_rem, replace=False)
        pos = np.concatenate([ins, rem]).astype(np.uint64)
        op = np.concatenate([np.zeros(n_ins, dtype=np.uint8), np.ones(n_rem, dtype=np.uint8)])
        perm = rng.permutation(pos.shape[0])                     # inserts and removals interleaved in batch order
        pos, op = pos[perm], op[perm]
        vals = device_random_scalars(torch, pos.shape[0], 1000 + i)
        m_keys, m_vals = model_apply(m_keys, m_vals, pos, op, vals.cpu().numpy().view(np.uint64))
        plan.append({"pos": torch.from_numpy(pos.view(np.int64)).to(stream.device),
                     "op": torch.from_numpy(op).to(stream.device), "vals": vals})
    torch.cuda.synchronize()
    steps = plan[:args.warmup + args.steps]
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in steps]
    sampler = ClockSampler(local)
    sampler.start()
    launches0 = None
    with torch.cuda.stream(stream):
        for i, st in enumerate(steps):
            if i == args.warmup:
                launches0 = eng.launch_count
            ev[i][0].record(stream)
            eng.ctree_update(tree, st["pos"], values=st["vals"], op=st["op"], async_=True)
            ev[i][1].record(stream)
    stream.synchronize()
    eng.sync()
    clocks = sampler.stop()
    launches = eng.launch_count - launches0
    ms = [ev[i][0].elapsed_time(ev[i][1]) for i in range(args.warmup, len(steps))]
    rejected = eng.last_ctree_rejected()

    # merge / hash / other split from kernel events of three more updates
    from torch.profiler import ProfilerActivity, profile
    split = {"hash": 0.0, "merge": 0.0, "other": 0.0}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(stream):
            for st in plan[len(steps):]:
                eng.ctree_update(tree, st["pos"], values=st["vals"], op=st["op"], async_=True)
        stream.synchronize()
    for e in prof.events():
        if getattr(e, "device_type", None) is None or "cuda" not in str(e.device_type).lower():
            continue
        name = e.name
        if "Memcpy" in name or "Memset" in name:
            continue
        dur = e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0
        if "k_mtree_digest" in name:
            split["hash"] += dur
        elif any(k in name for k in MERGE_KERNELS):
            split["merge"] += dur
        else:
            split["other"] += dur
    split = {k: v / 3 for k, v in split.items()}

    # openings of 2^16 present positions
    live = m_keys
    op_pos = torch.from_numpy(rng.choice(live, 1 << 16).view(np.int64)).to(stream.device)
    out = torch.empty((1 << 16, height, arity, 4), dtype=torch.int64, device=stream.device)
    timed(lambda: eng.ctree_open_batch(tree, op_pos, out=out, async_=True), 2)
    open_ms = timed(lambda: eng.ctree_open_batch(tree, op_pos, out=out, async_=True), 5)
    eng.sync()

    # parity, outside the timed region
    c0 = int(tree.count[0])
    lk = tree.keys[:c0].cpu().numpy().view(np.uint64)
    lv = tree.values[:c0].cpu().numpy().view(np.uint64)
    ok_model = c0 == m_keys.shape[0] and bool(np.array_equal(lk, m_keys)) and bool(np.array_equal(lv, m_vals)) \
        and rejected == 0
    hg = mtree_oracle.c_hash_groups(arity, threads=usable_cores())
    sample = rng.choice(m_keys.shape[0], 64, replace=False)
    sp = torch.from_numpy(m_keys[sample].view(np.int64)).to(stream.device)
    paths = eng.ctree_open_batch(tree, sp).cpu().numpy().view(np.uint64)
    root = tree.root.cpu().numpy().view(np.uint64)
    ok_paths = True
    for k, j in enumerate(sample):
        idx = int(m_keys[j])
        cur = m_vals[j]
        for l in range(height):
            slot = (idx >> (2 * l)) & 3
            ok_paths = ok_paths and bool(np.array_equal(paths[k, l, slot], cur))
            cur = hg(np.ascontiguousarray(paths[k, l][None]))[0]
        ok_paths = ok_paths and bool(np.array_equal(cur, root))
    props = torch.cuda.get_device_properties(local)
    ms_mean = statistics.mean(ms)
    ops = n_ins + n_rem
    return {"metric": "ctree_update_ops_per_sec", "value": ops / (ms_mean * 1e-3), "unit": "ops/s", "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_mean, "ms_per_update": ms_mean,
            "ms_per_update_median": statistics.median(ms), "higher_is_better": True, "data": "synthetic",
            "config": {"workload": "p252_ctree_update on device buffers: arity %d, height %d, max_leaves 2^23, 2^22 present "
                                   "positions over all of u64; per step %d inserts (half overwrites) + %d removals of "
                                   "present positions, interleaved" % (arity, height, n_ins, n_rem),
                       "inserts_per_step": n_ins, "removals_per_step": n_rem},
            "build_2e22_ms": build_ms, "build_leaves_per_s": n0 / (build_ms * 1e-3),
            "update_split_ms": split, "present_after": int(c0),
            "openings_per_s": (1 << 16) / (open_ms * 1e-3), "open_2e16_ms": open_ms,
            "gpu_launches_per_update": launches / args.steps,
            "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": bool(ok_model and ok_paths),
            "parity_checks": {"level0_equals_model": ok_model, "64_openings_hash_to_root_c_oracle": ok_paths}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--inserts", type=int, default=1 << 14, help="inserts per step (half of them overwrites)")
    ap.add_argument("--removals", type=int, default=1 << 12, help="removals of present positions per step")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0 or args.inserts < 0 or args.removals < 0 or args.inserts + args.removals < 1:
        ap.error("--steps must be >= 1, the other counts >= 0, and a step must hold at least one operation")
    import torch
    import poseidon252_b200 as pb
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    eng = pb.Engine(0, stream=stream.cuda_stream)
    line = ctree_update_line(args, eng, torch, stream, 0)
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
