//! Sparse fixed-height trees with inserts and removals at any position (`p252_smtree`), poseidon-merkle's
//! `Tree::insert(pos, item)` / `Tree::remove(pos)` over the H100 engine.  The `extern "C"` block below holds exactly the
//! `p252_smtree_*` functions; tests/c/smtree_smoke.c calls exactly that set (tests/test_smtree_bindings.py checks both
//! against the header).  It sits in a module of its own so that the three blocks of lib.rs stay as they are.
use core::ffi::c_int;
use core::mem::size_of;
use dusk_bls12_381::BlsScalar;

use super::{as_fr, as_fr_mut, need, p252_ctx, p252_mtree_layout, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_smtree`: a sparse fixed-height tree whose buffers this crate owns (host memory).
#[repr(C)]
pub struct p252_smtree {
    pub struct_size: u32,
    pub arity: i32,
    pub height: i32,
    pub reserved: i32,
    pub capacity: u64,
    pub leaves: *mut Fr,
    pub nodes: *mut Fr,
    pub present: *mut u8,
}

extern "C" {
    fn p252_smtree_build(ctx: *mut p252_ctx, tree: *mut p252_smtree, flags: c_int) -> c_int;
    fn p252_smtree_update(ctx: *mut p252_ctx, tree: *mut p252_smtree, pos: *const u64, op: *const u8, values: *const Fr,
                          n: usize, n_rejected: *mut usize, flags: c_int) -> c_int;
    fn p252_smtree_len(ctx: *mut p252_ctx, tree: *const p252_smtree, n_present: *mut u64, flags: c_int) -> c_int;
    fn p252_smtree_open_batch(ctx: *mut p252_ctx, tree: *const p252_smtree, pos: *const u64, n: usize, paths_out: *mut Fr,
                              flags: c_int) -> c_int;
}

/// Sparse tree of poseidon-merkle's `Tree<T, H, A>` shape: every position in `[0, capacity)` holds a value or is empty;
/// empty leaves and nodes with no value below them are `BlsScalar::zero()` and are never hashed.  Batches of inserts
/// and removals rehash only the touched paths on the GPU.
pub struct SparseTree {
    raw: p252_smtree,
    leaves: Vec<BlsScalar>,
    nodes: Vec<BlsScalar>,
    present: Vec<u8>,
}

impl SparseTree {
    pub fn new(arity: usize, height: usize, capacity: u64) -> Result<Self, BatchError> {
        let (mut ls, mut ns) = (0u64, 0u64);
        status(unsafe { p252_mtree_layout(arity as c_int, height as c_int, capacity, &mut ls, &mut ns, core::ptr::null_mut()) })?;
        let raw = p252_smtree {
            struct_size: size_of::<p252_smtree>() as u32, arity: arity as i32, height: height as i32, reserved: 0, capacity,
            leaves: core::ptr::null_mut(), nodes: core::ptr::null_mut(), present: core::ptr::null_mut(),
        };
        Ok(Self {
            raw,
            leaves: vec![BlsScalar::zero(); ls as usize],
            nodes: vec![BlsScalar::zero(); ns as usize],
            present: vec![0u8; (ls + ns) as usize],
        })
    }

    fn bind(&mut self) -> *mut p252_smtree {
        self.raw.leaves = as_fr_mut(&mut self.leaves);
        self.raw.nodes = as_fr_mut(&mut self.nodes);
        self.raw.present = self.present.as_mut_ptr();
        &mut self.raw
    }

    pub fn root(&self) -> BlsScalar { self.nodes[self.nodes.len() - 1] }
    pub fn contains(&self, pos: u64) -> bool { pos < self.raw.capacity && self.present[pos as usize] != 0 }
    /// Number of present positions.
    pub fn len(&mut self, engine: &Engine) -> Result<u64, BatchError> {
        let mut n = 0u64;
        let t = self.bind();
        status(unsafe { p252_smtree_len(engine.0, t, &mut n, P252_MEM_HOST) })?;
        Ok(n)
    }

    /// One batch: `ops[i] == 0` inserts / overwrites `values[i]` at `pos[i]`, `ops[i] == 1` removes `pos[i]`; the same as
    /// applying them one after another.
    pub fn apply(&mut self, engine: &Engine, pos: &[u64], ops: &[u8], values: &[BlsScalar]) -> Result<(), BatchError> {
        need(pos.len() == ops.len() && pos.len() == values.len(), "pos, ops and values must have equal lengths")?;
        let t = self.bind();
        status(unsafe { p252_smtree_update(engine.0, t, pos.as_ptr(), ops.as_ptr(), as_fr(values), pos.len(),
                                           core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// `Tree::insert(pos[i], values[i])` for every i (the last write to a position wins).
    pub fn insert(&mut self, engine: &Engine, pos: &[u64], values: &[BlsScalar]) -> Result<(), BatchError> {
        need(pos.len() == values.len(), "pos.len() must equal values.len()")?;
        let t = self.bind();
        status(unsafe { p252_smtree_update(engine.0, t, pos.as_ptr(), core::ptr::null(), as_fr(values), pos.len(),
                                           core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// `Tree::remove(pos[i])` for every i.
    pub fn remove(&mut self, engine: &Engine, pos: &[u64]) -> Result<(), BatchError> {
        let ops = vec![1u8; pos.len()];
        let zeros = vec![BlsScalar::zero(); pos.len()];
        self.apply(engine, pos, &ops, &zeros)
    }
    /// Recompute every node from the leaves and their presence.
    pub fn rebuild(&mut self, engine: &Engine) -> Result<(), BatchError> {
        let t = self.bind();
        status(unsafe { p252_smtree_build(engine.0, t, P252_MEM_HOST) })
    }
    /// `branch` of the poseidon-merkle `Opening` of every present position in `pos`: height x arity scalars each.
    pub fn open_batch(&mut self, engine: &Engine, pos: &[u64]) -> Result<Vec<BlsScalar>, BatchError> {
        let per = (self.raw.height as usize) * (self.raw.arity as usize);
        let mut paths = vec![BlsScalar::zero(); pos.len() * per];
        let t = self.bind();
        status(unsafe { p252_smtree_open_batch(engine.0, t, pos.as_ptr(), pos.len(), as_fr_mut(&mut paths), P252_MEM_HOST) })?;
        Ok(paths)
    }
}
