"""Tiny drivers for ncu captures of the auxiliary kernels (tools/collect_profiles.sh)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import poseidon252_b200 as pb
from poseidon252_b200.scalar import random_limbs_fast

what = sys.argv[1]
eng = pb.Engine(0)
rng = np.random.default_rng(1)
if what == "verify":
    k = 10
    leaves = torch.from_numpy(random_limbs_fast(rng, 4 ** k).view(np.int64)).cuda()
    nodes = eng.merkle4_build(leaves)
    idx = torch.from_numpy(rng.integers(0, 4 ** k, size=1 << 18).astype(np.int64)).cuda()
    paths = eng.merkle_open_batch(leaves, nodes, idx)
    ok = eng.merkle_verify_batch(leaves[idx], idx, paths, nodes[-1].cpu().numpy())
    print("verified", int(ok.sum().item()), "of", idx.numel(), "failures", eng.last_verify_failures())
else:
    x = torch.from_numpy(random_limbs_fast(rng, (3168, 4)).view(np.int64)).cuda()
    for _ in range(3):
        out = pb.Hash.digest_batch(pb.Domain.Merkle4, x, engine=eng)
    print(out.shape)
eng.close()
