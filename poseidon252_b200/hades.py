"""`hades` -- the permutation seam (src/hades.rs, src/hades/permutation.rs).
`permute` = Safe::permute for one state; `permute_batch` = NEW batch entry."""
import numpy as np

from .engine import _engine_for

WIDTH = 5            # src/hades.rs:34 (re-exported as dusk_poseidon::HADES_WIDTH, src/lib.rs:19)
FULL_ROUNDS = 8      # src/hades.rs:29
PARTIAL_ROUNDS = 60  # src/hades.rs:31


def permute(state, engine=None):
    """ScalarPermutation::permute (src/hades/permutation/scalar.rs:25-27) on one (5, 4) state."""
    s = np.ascontiguousarray(state, dtype=np.uint64).reshape(1, WIDTH, 4)
    return _engine_for(engine).permute_batch(s)[0]


def permute_batch(states, engine=None, dense=False, async_=False):
    """n independent width-5 permutations; states (n, 5, 4), returns a new array/tensor."""
    eng = _engine_for(engine, states)
    return eng.permute_batch(states, dense=dense, async_=async_)
