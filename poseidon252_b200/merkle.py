"""Merkle trees of Domain::Merkle4 / Merkle2 digests (node = Hash::digest(Domain::Merkle{A}, A children),
src/hash.rs:22-31).  Tree logic itself left the reference crate in 0.29.0
(CHANGELOG.md:164-168); only the node hash is defined there.  Dense builders (n_leaves = arity^k), `Tree`, a
fixed-height tree with batched appends and overwrites (p252_mtree), `SparseTree`, a fixed-height tree with batched
inserts and removals at any position (p252_smtree), and `CompactTree`, the same at any height with storage
proportional to the present leaves (p252_ctree)."""
from .engine import _engine_for, _is_torch, default_engine


def merkle4_level(children, engine=None, out=None, async_=False):
    eng = _engine_for(engine, children)
    return eng.merkle4_level(children, out=out, async_=async_)


def merkle4_build(leaves, engine=None, out=None, async_=False):
    """leaves (4^k, 4) -> internal nodes bottom-up, root last."""
    eng = _engine_for(engine, leaves)
    return eng.merkle4_build(leaves, out=out, async_=async_)


def merkle2_build(leaves, engine=None, out=None, async_=False):
    """Binary tree of Domain::Merkle2 digests (src/hash.rs:27-31): leaves (2^k, 4) -> internal nodes, root last."""
    eng = _engine_for(engine, leaves)
    return eng.merkle_build(leaves, arity=2, out=out, async_=async_)


def open_batch(leaves, nodes, leaf_idx, arity=4, engine=None, out=None, async_=False):
    """Openings of the leaves `leaf_idx`: (n, depth, arity, 4) -- per level the whole sibling group of the path
    node, level 0 = the leaf's own group (the `branch` of a poseidon-merkle `Opening`, AGENTS.md:62-66)."""
    eng = _engine_for(engine, leaves)
    return eng.merkle_open_batch(leaves, nodes, leaf_idx, arity=arity, out=out, async_=async_)


def verify_batch(leaf_items, leaf_idx, paths, root, arity=4, engine=None, async_=False):
    """n x Opening::verify on the device (depth chained Merkle digests per item) -> ok (n,) uint8."""
    eng = _engine_for(engine, paths)
    return eng.merkle_verify_batch(leaf_items, leaf_idx, paths, root, arity=arity, async_=async_)


def positions(leaf_idx, depth, arity=4):
    """Offset of the path node inside its sibling group at every level (the `positions` of an Opening)."""
    out, i = [], int(leaf_idx)
    for _ in range(depth):
        out.append(i % arity)
        i //= arity
    return out


class Opening:
    """Host-side mirror of poseidon-merkle's `Opening<T, H, A>`: `root`, `branch[level][slot]`, `positions[level]`
    (level 0 = leaf level here).  `verify(item)` runs the batch verifier on a batch of one."""

    def __init__(self, root, branch, leaf_idx, arity=4):
        import numpy as np
        self.root = np.ascontiguousarray(root, dtype=np.uint64).reshape(4)
        self.branch = np.ascontiguousarray(branch, dtype=np.uint64)
        if self.branch.ndim != 3 or self.branch.shape[1:] != (arity, 4):
            raise ValueError("branch must have shape (depth, arity, 4)")
        self.arity = int(arity)
        self.leaf_idx = int(leaf_idx)
        self.positions = positions(leaf_idx, self.branch.shape[0], arity)

    def verify(self, item, engine=None):
        import numpy as np
        ok = verify_batch(np.ascontiguousarray(item, dtype=np.uint64).reshape(1, 4),
                          np.array([self.leaf_idx], dtype=np.uint64), self.branch[None], self.root, arity=self.arity,
                          engine=engine)
        return bool(ok[0])


def level_offsets(n_leaves, arity=4):
    """[(offset, size)] of each internal level inside the node array, bottom-up."""
    out, off, m = [], 0, n_leaves // arity
    while m >= 1:
        out.append((off, m))
        off += m
        if m == 1:
            break
        m //= arity
    return out


def shard_plan(n_leaves_total, nranks, rank):
    """The per-level partition of the multi-GPU build (p252_merkle4_shard_plan): list of dicts with
    level_offset, level_size, my_offset, my_count, sharded -- bottom-up."""
    import ctypes

    from . import _native
    from .errors import raise_for_status
    lib = _native.lib()
    n = ctypes.c_int(0)
    raise_for_status(lib.p252_merkle4_shard_plan(int(n_leaves_total), int(nranks), int(rank), None, 0, ctypes.byref(n)), lib)
    arr = (_native.LevelPlan * n.value)()
    raise_for_status(lib.p252_merkle4_shard_plan(int(n_leaves_total), int(nranks), int(rank), arr, n.value, ctypes.byref(n)), lib)
    return [{f: int(getattr(a, f)) for f in ("level_offset", "level_size", "my_offset", "my_count", "sharded")} for a in arr]


class Tree:
    """Fixed-height tree of the poseidon-merkle `Tree<T, H, A>` shape (p252_mtree): room for `capacity` <= arity^height
    leaves, an occupied prefix of `n_leaves`, empty slots and empty subtrees are the zero scalar (src/hash.rs:24-26).
    `extend` appends, `update` overwrites; both rehash only the touched paths.  Buffers are numpy arrays
    (device=None) or CUDA int64 tensors on cuda:`device`; `leaves` / `nodes` are laid out as p252_mtree_layout says
    and their slots beyond the prefixes belong to the library."""

    def __init__(self, arity, height, capacity, engine=None, device=None):
        import numpy as np
        self.engine = engine or default_engine(0 if device is None else int(device))
        self.arity, self.height, self.capacity = int(arity), int(height), int(capacity)
        leaf_slots, node_slots, self.level_offset = self.engine.mtree_layout(self.arity, self.height, self.capacity)
        if device is None:
            self.leaves = np.zeros((leaf_slots, 4), dtype=np.uint64)
            self.nodes = np.zeros((node_slots, 4), dtype=np.uint64)
        else:
            import torch
            self.leaves = torch.zeros((leaf_slots, 4), dtype=torch.int64, device=torch.device("cuda", int(device)))
            self.nodes = torch.zeros((node_slots, 4), dtype=torch.int64, device=self.leaves.device)
        self.n_leaves = 0                      # all-zero buffers are the empty tree (root 0)

    def extend(self, values, async_=False):
        """Append the rows of `values` (k, 4) at [n_leaves, n_leaves + k)."""
        return self.engine.mtree_update(self, append=values, async_=async_)

    def update(self, idx, values, async_=False):
        """leaves[idx[i]] = values[i] for indices < n_leaves (the last write to a leaf wins)."""
        return self.engine.mtree_update(self, idx=idx, values=values, async_=async_)

    def build(self, async_=False):
        """Recompute every node from the leaf prefix (e.g. after writing leaves[:n_leaves] directly)."""
        self.engine.mtree_build(self, async_=async_)

    @property
    def root(self):
        return self.nodes[-1]

    def level_sizes(self):
        """Occupied nodes per level, leaves first: ceil(n_leaves / arity^l)."""
        m = [self.n_leaves]
        for _ in range(self.height):
            m.append(-(-m[-1] // self.arity))
        return m

    def levels(self):
        """Views of the occupied prefix of every level, leaves first, [root] last."""
        m = self.level_sizes()
        return [self.leaves[:m[0]]] + [self.nodes[self.level_offset[l]:self.level_offset[l] + m[l]]
                                       for l in range(1, self.height + 1)]

    def open(self, idx, async_=False):
        """Openings of the leaves `idx`: (n, height, arity, 4), zero slots beyond each level's prefix."""
        return self.engine.mtree_open_batch(self, idx, async_=async_)

    def opening(self, i):
        """poseidon-merkle `Opening` of leaf i (host arrays)."""
        import numpy as np
        if _is_torch(self.leaves):
            import torch
            branch = self.open(torch.tensor([int(i)], dtype=torch.int64, device=self.leaves.device))[0]
            branch, root = branch.cpu().numpy().view(np.uint64), self.root.cpu().numpy().view(np.uint64)
        else:
            branch, root = self.open(np.array([int(i)], dtype=np.uint64))[0], self.root
        return Opening(root, branch, int(i), arity=self.arity)


def _remove(update, tree, like, pos, async_):
    """A batch of removals through the engine's `update` call: an op vector of ones in the memory space of `like`, one
    of the tree's buffers."""
    if _is_torch(like):
        import torch
        op = torch.ones((len(pos),), dtype=torch.uint8, device=like.device)
    else:
        import numpy as np
        op = np.ones((len(pos),), dtype=np.uint8)
    update(tree, pos, op=op, async_=async_)
    if async_ and _is_torch(op):
        tree.engine._keep_until_sync(op)          # read by the device after the call returns


class SparseTree:
    """Sparse fixed-height tree of the poseidon-merkle `Tree<T, H, A>` shape with `insert` and `remove` at any position
    (p252_smtree): each position in [0, capacity) is present or absent; an absent leaf and a node with no present leaf
    below it are the zero scalar and are never hashed (src/hash.rs:24-26), a present leaf of value zero is not absent.
    Buffers are numpy arrays (device=None) or CUDA tensors on cuda:`device`: `leaves` / `nodes` (int64 or uint64, laid
    out as p252_mtree_layout says) and `present` (uint8, one byte per slot, leaves then nodes; `leaf_present` /
    `node_present` are views).  Every absent slot belongs to the library.  With the present set [0, n) the buffers equal
    those of a `Tree` holding n leaves."""

    def __init__(self, arity, height, capacity, engine=None, device=None):
        import numpy as np
        self.engine = engine or default_engine(0 if device is None else int(device))
        self.arity, self.height, self.capacity = int(arity), int(height), int(capacity)
        leaf_slots, node_slots, self.level_offset = self.engine.mtree_layout(self.arity, self.height, self.capacity)
        if device is None:
            self.leaves = np.zeros((leaf_slots, 4), dtype=np.uint64)
            self.nodes = np.zeros((node_slots, 4), dtype=np.uint64)
            self.present = np.zeros((leaf_slots + node_slots,), dtype=np.uint8)
        else:
            import torch
            dev = torch.device("cuda", int(device))
            self.leaves = torch.zeros((leaf_slots, 4), dtype=torch.int64, device=dev)
            self.nodes = torch.zeros((node_slots, 4), dtype=torch.int64, device=dev)
            self.present = torch.zeros((leaf_slots + node_slots,), dtype=torch.uint8, device=dev)
        self.leaf_present = self.present[:leaf_slots]
        self.node_present = self.present[leaf_slots:]
        # all-zero buffers are the empty tree (root 0)

    def apply(self, pos, op, values, async_=False):
        """One batch: op[i] = 0 inserts / overwrites values[i] at pos[i], op[i] = 1 removes pos[i]; the result equals
        applying the operations in batch order."""
        self.engine.smtree_update(self, pos, values=values, op=op, async_=async_)

    def insert(self, pos, values, async_=False):
        """leaves[pos[i]] = values[i], present (the last write to a position wins)."""
        self.engine.smtree_update(self, pos, values=values, async_=async_)

    def remove(self, pos, async_=False):
        """Make the positions `pos` absent (removing an absent position does nothing)."""
        _remove(self.engine.smtree_update, self, self.leaves, pos, async_)

    def build(self, async_=False):
        """Recompute every node from the leaves and `leaf_present` (e.g. after writing them directly)."""
        self.engine.smtree_build(self, async_=async_)

    @property
    def root(self):
        return self.nodes[-1]

    def len(self):
        """Number of present positions."""
        return self.engine.smtree_len(self)

    def __len__(self):
        return self.len()

    def contains(self, pos):
        """Whether position `pos` holds a value."""
        pos = int(pos)
        if pos < 0 or pos >= self.capacity:
            return False
        return bool(int(self.leaf_present[pos]))

    def open(self, pos, async_=False):
        """Openings of the present positions `pos`: (n, height, arity, 4), absent slots zero."""
        return self.engine.smtree_open_batch(self, pos, async_=async_)

    opening = Tree.opening     # poseidon-merkle `Opening` of a present position (host arrays)


class CompactTree:
    """Compact sparse tree of the poseidon-merkle `Tree<T, H, A>` shape at any height (p252_ctree): positions are any
    integers below arity^height (every u64 at arity 2 / height 64 or arity 4 / height 32), and storage is proportional
    to the present leaves, at most `max_leaves` of them.  Presence and the empty-subtree rule are those of `SparseTree`.
    Level l is the sorted list of its present nodes: `keys` (node indices) and `values` (scalars) from slot
    level_offset[l], `count[l]` entries, every later slot zero.  Buffers are numpy arrays (device=None) or CUDA tensors
    on cuda:`device` (int64 tensors hold the indices' bits).  All-zero buffers are the empty tree."""

    def __init__(self, arity, height, max_leaves, engine=None, device=None):
        import numpy as np
        self.engine = engine or default_engine(0 if device is None else int(device))
        self.arity, self.height, self.max_leaves = int(arity), int(height), int(max_leaves)
        total, self.level_offset = self.engine.ctree_layout(self.arity, self.height, self.max_leaves)
        if device is None:
            self.keys = np.zeros((total,), dtype=np.uint64)
            self.values = np.zeros((total, 4), dtype=np.uint64)
            self.count = np.zeros((self.height + 1,), dtype=np.uint64)
        else:
            import torch
            dev = torch.device("cuda", int(device))
            self.keys = torch.zeros((total,), dtype=torch.int64, device=dev)
            self.values = torch.zeros((total, 4), dtype=torch.int64, device=dev)
            self.count = torch.zeros((self.height + 1,), dtype=torch.int64, device=dev)

    def apply(self, pos, op, values, async_=False):
        """One batch: op[i] = 0 inserts / overwrites values[i] at pos[i], op[i] = 1 removes pos[i]; the result equals
        applying the operations in batch order."""
        self.engine.ctree_update(self, pos, values=values, op=op, async_=async_)

    def insert(self, pos, values, async_=False):
        """Position pos[i] holds values[i] (the last write to a position wins)."""
        self.engine.ctree_update(self, pos, values=values, async_=async_)

    def remove(self, pos, async_=False):
        """Make the positions `pos` absent (removing an absent position does nothing)."""
        _remove(self.engine.ctree_update, self, self.values, pos, async_)

    @property
    def root(self):
        return self.values[self.level_offset[self.height]]

    def len(self):
        """Number of present positions (count[0])."""
        return int(self.count[0])

    def __len__(self):
        return self.len()

    def level(self, l):
        """(keys, values) views of the present nodes of level l."""
        c, o = int(self.count[l]), self.level_offset[l]
        return self.keys[o:o + c], self.values[o:o + c]

    def contains(self, pos):
        """Whether position `pos` holds a value: a binary search over level 0's keys."""
        pos = int(pos)
        if pos < 0 or pos >= self.arity ** self.height:
            return False
        keys, _ = self.level(0)
        if _is_torch(keys):
            import torch
            # int64 tensors hold u64 bits: flipping the sign bit turns u64 order into int64 order
            lo = -(1 << 63)
            k = torch.tensor([pos + lo], dtype=torch.int64, device=keys.device)
            j = int(torch.searchsorted(keys ^ lo, k))
            return j < keys.shape[0] and int(keys[j]) ^ lo == int(k)
        import numpy as np
        j = int(np.searchsorted(keys, np.uint64(pos)))
        return j < keys.shape[0] and int(keys[j]) == pos

    def open(self, pos, async_=False):
        """Openings of the present positions `pos`: (n, height, arity, 4), absent slots zero."""
        return self.engine.ctree_open_batch(self, pos, async_=async_)

    def opening(self, i):
        """poseidon-merkle `Opening` of present position i (host arrays)."""
        import numpy as np
        if _is_torch(self.values):
            import torch
            j = int(i) - (1 << 64) if int(i) >= 1 << 63 else int(i)
            branch = self.open(torch.tensor([j], dtype=torch.int64, device=self.values.device))[0]
            branch, root = branch.cpu().numpy().view(np.uint64), self.root.cpu().numpy().view(np.uint64)
        else:
            branch, root = self.open(np.array([int(i)], dtype=np.uint64))[0], self.root
        return Opening(root, branch, int(i), arity=self.arity)
