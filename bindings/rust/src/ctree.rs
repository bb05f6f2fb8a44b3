//! Compact sparse trees (`p252_ctree`): poseidon-merkle's `Tree<T, H, A>` at any height, positions anywhere below
//! `A^H` (every `u64` at `A = 2, H = 64` or `A = 4, H = 32`), storage proportional to the present leaves.  The
//! `extern "C"` block below holds exactly the `p252_ctree_*` functions; tests/c/ctree_smoke.c calls exactly that set
//! (tests/test_ctree_bindings.py checks both against the header).  It sits in a module of its own so that the three
//! blocks of lib.rs stay as they are.
use core::ffi::c_int;
use core::mem::size_of;
use dusk_bls12_381::BlsScalar;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_ctree`: a compact sparse tree whose buffers this crate owns (host memory).
#[repr(C)]
pub struct p252_ctree {
    pub struct_size: u32,
    pub arity: i32,
    pub height: i32,
    pub reserved: i32,
    pub max_leaves: u64,
    pub keys: *mut u64,
    pub values: *mut Fr,
    pub count: *mut u64,
}

extern "C" {
    fn p252_ctree_layout(arity: c_int, height: c_int, max_leaves: u64, total_slots: *mut u64, level_offset: *mut u64) -> c_int;
    fn p252_ctree_update(ctx: *mut p252_ctx, tree: *mut p252_ctree, pos: *const u64, op: *const u8, values: *const Fr,
                         n: usize, n_rejected: *mut usize, flags: c_int) -> c_int;
    fn p252_ctree_open_batch(ctx: *mut p252_ctx, tree: *const p252_ctree, pos: *const u64, n: usize, paths_out: *mut Fr,
                             flags: c_int) -> c_int;
}

/// Sparse tree of poseidon-merkle's `Tree<T, H, A>` shape at any height: every position below `A^H` holds a value or is
/// empty; empty leaves and nodes with no value below them are `BlsScalar::zero()` and are never hashed.  Each level is
/// the sorted list of its present nodes; batches of inserts and removals run on the GPU.
pub struct CompactTree {
    raw: p252_ctree,
    keys: Vec<u64>,
    values: Vec<BlsScalar>,
    count: Vec<u64>,
    offset: Vec<u64>,
}

impl CompactTree {
    pub fn new(arity: usize, height: usize, max_leaves: u64) -> Result<Self, BatchError> {
        need(height >= 1 && height <= 64, "height must be 1..64")?;
        let mut total = 0u64;
        let mut offset = vec![0u64; height + 1];
        status(unsafe { p252_ctree_layout(arity as c_int, height as c_int, max_leaves, &mut total, offset.as_mut_ptr()) })?;
        let raw = p252_ctree {
            struct_size: size_of::<p252_ctree>() as u32, arity: arity as i32, height: height as i32, reserved: 0, max_leaves,
            keys: core::ptr::null_mut(), values: core::ptr::null_mut(), count: core::ptr::null_mut(),
        };
        Ok(Self {
            raw,
            keys: vec![0u64; total as usize],
            values: vec![BlsScalar::zero(); total as usize],
            count: vec![0u64; height + 1],
            offset,
        })
    }

    fn bind(&mut self) -> *mut p252_ctree {
        self.raw.keys = self.keys.as_mut_ptr();
        self.raw.values = as_fr_mut(&mut self.values);
        self.raw.count = self.count.as_mut_ptr();
        &mut self.raw
    }

    pub fn root(&self) -> BlsScalar { self.values[self.offset[self.raw.height as usize] as usize] }
    /// Number of present positions.
    pub fn len(&self) -> u64 { self.count[0] }
    pub fn contains(&self, pos: u64) -> bool { self.keys[..self.count[0] as usize].binary_search(&pos).is_ok() }

    /// One batch: `ops[i] == 0` inserts / overwrites `values[i]` at `pos[i]`, `ops[i] == 1` removes `pos[i]`; the same as
    /// applying them one after another.
    pub fn apply(&mut self, engine: &Engine, pos: &[u64], ops: &[u8], values: &[BlsScalar]) -> Result<(), BatchError> {
        need(pos.len() == ops.len() && pos.len() == values.len(), "pos, ops and values must have equal lengths")?;
        let t = self.bind();
        status(unsafe { p252_ctree_update(engine.0, t, pos.as_ptr(), ops.as_ptr(), as_fr(values), pos.len(),
                                          core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// `Tree::insert(pos[i], values[i])` for every i (the last write to a position wins).
    pub fn insert(&mut self, engine: &Engine, pos: &[u64], values: &[BlsScalar]) -> Result<(), BatchError> {
        need(pos.len() == values.len(), "pos.len() must equal values.len()")?;
        let t = self.bind();
        status(unsafe { p252_ctree_update(engine.0, t, pos.as_ptr(), core::ptr::null(), as_fr(values), pos.len(),
                                          core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// `Tree::remove(pos[i])` for every i.
    pub fn remove(&mut self, engine: &Engine, pos: &[u64]) -> Result<(), BatchError> {
        let ops = vec![1u8; pos.len()];
        let zeros = vec![BlsScalar::zero(); pos.len()];
        self.apply(engine, pos, &ops, &zeros)
    }
    /// `branch` of the poseidon-merkle `Opening` of every present position in `pos`: height x arity scalars each.
    pub fn open_batch(&mut self, engine: &Engine, pos: &[u64]) -> Result<Vec<BlsScalar>, BatchError> {
        let per = (self.raw.height as usize) * (self.raw.arity as usize);
        let mut paths = vec![BlsScalar::zero(); pos.len() * per];
        let t = self.bind();
        status(unsafe { p252_ctree_open_batch(engine.0, t, pos.as_ptr(), pos.len(), as_fr_mut(&mut paths), P252_MEM_HOST) })?;
        Ok(paths)
    }
}
