#!/usr/bin/env python
"""Benchmark of sparse fixed-height tree updates (p252_smtree_update): inserts and removals at any position, only the
touched paths revisited.

    python tools/bench_smtree_update.py [--steps K] [--warmup W] [--inserts I] [--removals R] > smtree_update.json

Tree: arity 4, height 17, capacity 2^22, 2^21 present positions drawn from a seed and built once on device buffers.
One timed step = one p252_smtree_update with I random inserts (default 2^14; half at present positions, i.e.
overwrites, half anywhere) and R removals of present positions (default 2^12), timed with CUDA events on the engine's
stream.  Prints one JSON line: ms per update (mean and median), distinct dirty nodes and nodes emptied without hashing
per step (computed on the host from a numpy model of the presence), dirty nodes/s, and in the same run the time of a
sparse p252_smtree_build of the initial tree (and of a tree of the same capacity with 1 000 present positions), and
of a p252_mtree_update of the same batch size on a 2^21-leaf prefix
tree, the device and its power limit, and an in-run parity verdict (outside the timed region: the tree equals a fresh
p252_smtree_build over its final leaves and presence, and 64 random dirty leaf-to-root paths match the C oracle).
Writes nothing in the repository tree.  The clock sampler and the device-side input generator are bench.py's.
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


def node_presence(leaf_present, arity, height):
    """presence of every level, leaves first (numpy bool arrays over whole groups)"""
    import numpy as np
    levels = [leaf_present]
    cur = leaf_present
    for _ in range(height):
        pad = (-cur.shape[0]) % arity
        if pad:
            cur = np.concatenate([cur, np.zeros(pad, dtype=bool)])
        cur = cur.reshape(-1, arity).any(axis=1)
        levels.append(cur)
    return levels


def dirty_counts(pos, presence_after, arity, height):
    """(distinct nodes above the leaves one update revisits, how many of them end up absent = zeroed without hashing)"""
    import numpy as np
    d = np.unique(np.asarray(pos, dtype=np.int64))
    total = emptied = 0
    for l in range(1, height + 1):
        d = np.unique(d // arity)
        total += int(d.shape[0])
        emptied += int((~presence_after[l][d]).sum())
    return total, emptied


def smtree_update_line(args, eng, torch, stream, local):
    import numpy as np
    import mtree_oracle
    from poseidon252_b200 import merkle
    arity, height, capacity, n0 = 4, 17, 1 << 22, 1 << 21
    n_ins, n_rem = args.inserts, args.removals
    rng = np.random.default_rng(101)
    present = np.zeros(capacity, dtype=bool)
    present[rng.choice(capacity, n0, replace=False)] = True
    tree = merkle.SparseTree(arity, height, capacity, engine=eng, device=local)
    with torch.cuda.stream(stream):
        init = torch.from_numpy(np.flatnonzero(present)).to(stream.device)
        tree.leaves[init] = device_random_scalars(torch, n0, 102)
        tree.leaf_present[init] = 1
    stream.synchronize()

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / reps

    timed(lambda: tree.build(async_=True), 1)
    build_ms = timed(lambda: tree.build(async_=True), 3)
    build_nodes = int(sum(p.sum() for p in node_presence(present, arity, height)[1:]))
    # the build's work follows the present nodes: the same capacity with 1 000 present positions
    small = merkle.SparseTree(arity, height, capacity, engine=eng, device=local)
    with torch.cuda.stream(stream):
        few = torch.from_numpy(rng.choice(capacity, 1000, replace=False)).to(stream.device)
        small.leaves[few] = device_random_scalars(torch, 1000, 105)
        small.leaf_present[few] = 1
    stream.synchronize()
    timed(lambda: small.build(async_=True), 1)
    small_build_ms = timed(lambda: small.build(async_=True), 3)
    del small

    # a p252_mtree_update of the same batch size (overwrites) on a 2^21-leaf prefix tree, in the same run
    dense = merkle.Tree(arity, height, capacity, engine=eng, device=local)
    with torch.cuda.stream(stream):
        dense.leaves[:n0] = device_random_scalars(torch, n0, 103)
    stream.synchronize()
    dense.n_leaves = n0
    dense.build()
    d_idx = torch.from_numpy(rng.integers(0, n0, n_ins + n_rem)).to(stream.device)
    d_vals = device_random_scalars(torch, n_ins + n_rem, 104)
    mtree_step = lambda: eng.mtree_update(dense, idx=d_idx, values=d_vals, async_=True)  # noqa: E731
    timed(mtree_step, 2)
    mtree_ms = timed(mtree_step, 10)
    eng.sync()
    del dense, d_idx, d_vals

    # every step's inputs and the host model are made before the timed loop
    total = args.warmup + args.steps
    plan = []
    for i in range(total):
        live = np.flatnonzero(present)
        ins = np.where(rng.random(n_ins) < 0.5, rng.choice(live, n_ins), rng.integers(0, capacity, n_ins))
        rem = rng.choice(live, n_rem, replace=False)
        pos = np.concatenate([ins, rem]).astype(np.int64)
        op = np.concatenate([np.zeros(n_ins, dtype=np.uint8), np.ones(n_rem, dtype=np.uint8)])
        perm = rng.permutation(pos.shape[0])                     # inserts and removals interleaved in batch order
        pos, op = pos[perm], op[perm]
        last = {}
        for k, p_ in enumerate(pos):
            last[int(p_)] = k
        keys = np.fromiter(last.keys(), dtype=np.int64)
        present[keys] = op[np.fromiter(last.values(), dtype=np.int64)] == 0
        dirty, emptied = dirty_counts(pos, node_presence(present, arity, height), arity, height)
        plan.append({"pos_host": pos, "dirty": dirty, "emptied": emptied, "pos": torch.from_numpy(pos).to(stream.device),
                     "op": torch.from_numpy(op).to(stream.device), "vals": device_random_scalars(torch, pos.shape[0], 1000 + i)})
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(total)]
    sampler = ClockSampler(local)
    sampler.start()
    launches0 = None
    with torch.cuda.stream(stream):
        for i, st in enumerate(plan):
            if i == args.warmup:
                launches0 = eng.launch_count
            ev[i][0].record(stream)
            eng.smtree_update(tree, st["pos"], values=st["vals"], op=st["op"], async_=True)
            ev[i][1].record(stream)
    stream.synchronize()
    eng.sync()
    clocks = sampler.stop()
    launches = eng.launch_count - launches0
    ms = [ev[i][0].elapsed_time(ev[i][1]) for i in range(args.warmup, total)]
    dirty = [plan[i]["dirty"] for i in range(args.warmup, total)]
    emptied = [plan[i]["emptied"] for i in range(args.warmup, total)]

    # parity, outside the timed region: the presence model, a fresh build over the final leaves and presence, and 64
    # random dirty paths of the last step recomputed with the C oracle
    ok_model = bool(np.array_equal(tree.leaf_present[:capacity].cpu().numpy().astype(bool), present)) and \
        len(tree) == int(present.sum())
    fresh = merkle.SparseTree(arity, height, capacity, engine=eng, device=local)
    fresh.leaves.copy_(tree.leaves)
    fresh.leaf_present.copy_(tree.leaf_present)
    fresh.build()
    ok_fresh = bool(torch.equal(fresh.nodes, tree.nodes) and torch.equal(fresh.present, tree.present))
    del fresh
    hg = mtree_oracle.c_hash_groups(arity, threads=usable_cores())
    off = tree.level_offset
    below, below_p, ok_paths = tree.leaves, tree.leaf_present, True
    cur = rng.choice(plan[-1]["pos_host"], 64)
    for l in range(1, height + 1):
        g = cur // arity
        slots = torch.from_numpy((g[:, None] * arity + np.arange(arity)[None, :]).reshape(-1)).cuda()
        grp = below[slots].cpu().numpy().view(np.uint64).reshape(-1, arity, 4)
        gp = below_p[slots].cpu().numpy().reshape(-1, arity).any(axis=1)
        gt = torch.from_numpy(g).cuda()
        got = tree.nodes[off[l]:][gt].cpu().numpy().view(np.uint64)
        got_p = tree.node_present[off[l]:][gt].cpu().numpy()
        ok_paths = ok_paths and bool(np.array_equal(got_p, gp.astype(np.uint8))) and not got[~gp].any()
        if gp.any():
            ok_paths = ok_paths and bool(np.array_equal(hg(np.ascontiguousarray(grp[gp])), got[gp]))
        below, below_p, cur = tree.nodes[off[l]:], tree.node_present[off[l]:], g
    props = torch.cuda.get_device_properties(local)
    value = sum(dirty) / (sum(ms) * 1e-3)
    ms_mean = statistics.mean(ms)
    return {"metric": "smtree_dirty_nodes_per_sec", "value": value, "unit": "nodes/s", "n_gpus": 1, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_mean, "ms_per_update": ms_mean, "ms_per_update_median": statistics.median(ms),
            "higher_is_better": True, "data": "synthetic",
            "config": {"workload": "p252_smtree_update on device buffers: arity %d, height %d, capacity 2^22, 2^21 present "
                                   "positions built once; per step %d inserts (half overwrites) + %d removals of present "
                                   "positions, interleaved" % (arity, height, n_ins, n_rem),
                       "inserts_per_step": n_ins, "removals_per_step": n_rem},
            "dirty_nodes_per_step": statistics.mean(dirty), "emptied_nodes_per_step": statistics.mean(emptied),
            "dirty_nodes_per_s": value, "sparse_build_ms": build_ms, "sparse_build_present_nodes": build_nodes,
            "sparse_build_1000_present_ms": small_build_ms,
            "mtree_update_same_batch_ms": mtree_ms, "gpu_launches_per_update": launches / args.steps,
            "clocks": clocks, "device": props.name, "power_limit_w": clocks.get("power_limit_w"),
            "parity": "ok" if (ok_model and ok_fresh and ok_paths) else "MISMATCH",
            "parity_checks": {"presence_equals_model": ok_model, "equals_fresh_build": ok_fresh,
                              "64_dirty_paths_vs_c_oracle": ok_paths}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
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
    line = smtree_update_line(args, eng, torch, stream, 0)
    eng.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
