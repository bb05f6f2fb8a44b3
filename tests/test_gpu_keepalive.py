"""What an asynchronous device call leaves for the stream stays alive until sync(): the counter a host function writes
through, the zero `values` the engine makes for a batch of removals and the op vector `remove` makes.  A later call
replaces the counter the engine reads, not the one the stream still writes."""
import ctypes
import gc
import weakref

import numpy as np
import pytest
import torch

import poseidon252_b200 as pb
from poseidon252_b200.scalar import random_scalars

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["sparse", "compact"])
def test_async_temporaries_live_until_sync(engine, kind):
    rng = np.random.default_rng(21)
    engine.sync()
    tree = pb.SparseTree(4, 3, 64, engine=engine, device=0) if kind == "sparse" else \
        pb.CompactTree(4, 3, 64, engine=engine, device=0)
    last = engine.last_smtree_rejected if kind == "sparse" else engine.last_ctree_rejected
    like = tree.leaves if kind == "sparse" else tree.values
    pos = torch.arange(40, dtype=torch.int64, device=like.device)
    vals = torch.from_numpy(random_scalars(rng, 40).view(np.int64)).to(like.device)
    tree.insert(pos, vals)
    assert engine._kept_until_sync == []                 # a synchronous call leaves nothing behind

    tree.remove(pos[:10], async_=True)
    kept = list(engine._kept_until_sync)
    assert len(kept) == 3 and sum(isinstance(o, ctypes.c_size_t) for o in kept) == 1           # the counter
    assert sorted(tuple(o.shape) for o in kept if torch.is_tensor(o)) == [(10,), (10, 4)]      # op, zero values
    refs = [weakref.ref(o) for o in kept]
    del kept
    tree.insert(pos[:5], vals[:5], async_=True)          # replaces the counter last_*_rejected() reads
    gc.collect()
    assert all(r() is not None for r in refs)

    engine.sync()
    gc.collect()
    assert engine._kept_until_sync == [] and all(r() is None for r in refs)
    assert last() == 0 and len(tree) == 35
