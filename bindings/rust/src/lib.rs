//! SOURCE ONLY -- never compiled in this repository's image (no cargo/rustc).  Batch entry points for
//! `dusk_poseidon` over the H100 engine: `Hash::digest_batch`, `hades::permute_batch`,
//! `encrypt_batch`, `decrypt_batch`, `merkle4_build`, Merkle openings, fixed-height trees with batched updates
//! (`Tree`), sparse fixed-height trees with inserts and removals at any position (`SparseTree`, in smtree.rs),
//! compact sparse trees at any height (`CompactTree`, in ctree.rs),
//! variable-length digest batches (`Engine::digest_batch_varlen`), bound to include/poseidon252_b200.h.
//! The `extern "C"` block below is checked mechanically against the header by tests/test_abi.py
//! (same symbol set, same parameter counts) and its exact call set is exercised by tests/c/abi_smoke.c.
//!
//! Layout contract: the C side reads every scalar as `p252_fr { uint64_t l[4]; }` = `BlsScalar.0`
//! (Montgomery limbs; the reference reads `.0` directly at src/hash.rs:180).  `BlsScalar` is a one-field tuple
//! struct `Scalar(pub [u64; 4])`; Rust does not promise `repr(transparent)` for it, so the assumptions this file
//! relies on are asserted at compile time below, and every pointer handed to C is derived from the `.0` array
//! (`as_fr` / `as_fr_mut`), never from a cast of `*const BlsScalar` itself.
#![allow(non_camel_case_types)]

use core::ffi::{c_char, c_int};
use core::mem::{align_of, size_of};
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::JubJubAffine;
use dusk_poseidon::{Domain, Error};

/// `p252_fr`
pub type Fr = [u64; 4];

// A slice of BlsScalar must be a dense array of 32-byte, 8-aligned limb quadruples.
const _: () = assert!(size_of::<BlsScalar>() == 32 && align_of::<BlsScalar>() == 8);
const _: () = assert!(size_of::<[BlsScalar; 5]>() == 160);
const _: () = assert!(size_of::<Fr>() == 32 && align_of::<Fr>() == 8);

#[inline]
fn as_fr(s: &[BlsScalar]) -> *const Fr {
    // `.0` of element 0 is at offset 0 of the slice (single-field struct, size == size of the field)
    if s.is_empty() { core::ptr::NonNull::<Fr>::dangling().as_ptr() } else { &s[0].0 as *const Fr }
}
#[inline]
fn as_fr_mut(s: &mut [BlsScalar]) -> *mut Fr {
    if s.is_empty() { core::ptr::NonNull::<Fr>::dangling().as_ptr() } else { &mut s[0].0 as *mut Fr }
}

#[repr(C)]
pub struct p252_ctx {
    _private: [u8; 0],
}

pub const P252_MEM_HOST: c_int = 0;

extern "C" {
    fn p252_create(device: c_int, out: *mut *mut p252_ctx) -> c_int;
    fn p252_destroy(ctx: *mut p252_ctx);
    fn p252_strerror(status: c_int) -> *const c_char;
    fn p252_permute_batch(ctx: *mut p252_ctx, states: *mut Fr, n: usize, flags: c_int) -> c_int;
    fn p252_hash_batch(ctx: *mut p252_ctx, domain: c_int, input: *const Fr, n: usize, in_len: usize,
                       out: *mut Fr, out_len: usize, flags: c_int) -> c_int;
    fn p252_hash_batch_truncated(ctx: *mut p252_ctx, domain: c_int, input: *const Fr, n: usize, in_len: usize,
                                 out_raw: *mut Fr, out_len: usize, flags: c_int) -> c_int;
    fn p252_encrypt_batch(ctx: *mut p252_ctx, msg: *const Fr, n: usize, l: usize,
                          secret_uv: *const Fr, nonce: *const Fr, cipher: *mut Fr,
                          flags: c_int) -> c_int;
    fn p252_decrypt_batch(ctx: *mut p252_ctx, cipher: *const Fr, n: usize, l: usize,
                          secret_uv: *const Fr, nonce: *const Fr, msg: *mut Fr,
                          ok: *mut u8, n_failed: *mut usize, flags: c_int) -> c_int;
    fn p252_merkle_tree_nodes(arity: c_int, n_leaves: usize, n_internal: *mut usize, n_levels: *mut c_int) -> c_int;
    fn p252_merkle_build(ctx: *mut p252_ctx, arity: c_int, leaves: *const Fr, n_leaves: usize,
                         nodes_out: *mut Fr, flags: c_int) -> c_int;
    fn p252_merkle_open_batch(ctx: *mut p252_ctx, arity: c_int, leaves: *const Fr, n_leaves: usize, nodes: *const Fr,
                              leaf_idx: *const u64, n: usize, paths_out: *mut Fr, flags: c_int) -> c_int;
    fn p252_merkle_verify_batch(ctx: *mut p252_ctx, arity: c_int, depth: c_int, leaf_items: *const Fr,
                                leaf_idx: *const u64, paths: *const Fr, root: *const Fr, n: usize, ok: *mut u8,
                                n_failed: *mut usize, flags: c_int) -> c_int;
}

/// `p252_mtree`: a fixed-height tree whose buffers this crate owns (host memory).
#[repr(C)]
pub struct p252_mtree {
    pub struct_size: u32,
    pub arity: i32,
    pub height: i32,
    pub reserved: i32,
    pub capacity: u64,
    pub n_leaves: u64,
    pub leaves: *mut Fr,
    pub nodes: *mut Fr,
}

// Fixed-height trees.  A block of its own: its exact call set is exercised by tests/c/mtree_smoke.c
// (tests/test_mtree_bindings.py checks both against the header), as the block above is by tests/c/abi_smoke.c.
extern "C" {
    fn p252_mtree_layout(arity: c_int, height: c_int, capacity: u64, leaf_slots: *mut u64, node_slots: *mut u64,
                         level_offset: *mut u64) -> c_int;
    fn p252_mtree_build(ctx: *mut p252_ctx, tree: *mut p252_mtree, flags: c_int) -> c_int;
    fn p252_mtree_update(ctx: *mut p252_ctx, tree: *mut p252_mtree, idx: *const u64, values: *const Fr, n_upd: usize,
                         append: *const Fr, n_append: usize, n_rejected: *mut usize, flags: c_int) -> c_int;
    fn p252_mtree_open_batch(ctx: *mut p252_ctx, tree: *const p252_mtree, leaf_idx: *const u64, n: usize,
                             paths_out: *mut Fr, flags: c_int) -> c_int;
}

// Variable-length digest batches.  A block of its own holding exactly this function: tests/c/varlen_smoke.c calls it
// (tests/test_varlen_bindings.py checks both against the header).
extern "C" {
    fn p252_hash_batch_varlen(ctx: *mut p252_ctx, domain: c_int, input: *const Fr, n_scalars: usize, offsets: *const u64,
                              n: usize, max_len: usize, out: *mut Fr, out_len: usize, n_rejected: *mut usize,
                              flags: c_int) -> c_int;
}

// Sparse fixed-height trees (inserts and removals at any position): their own `extern "C"` block in smtree.rs.
mod smtree;
pub use smtree::{p252_smtree, SparseTree};

// Encrypt / decrypt batches over messages of different lengths: their own `extern "C"` block in crypt_varlen.rs (methods
// on Engine).
mod crypt_varlen;

// Compact sparse trees (positions anywhere below arity^height, storage proportional to the present leaves): their own
// `extern "C"` block in ctree.rs.
mod ctree;
pub use ctree::{p252_ctree, CompactTree};

// JubJub key exchange and encrypt / decrypt with the shared secret derived on the device: their own `extern "C"` block in
// dhke.rs (methods on Engine).
mod dhke;

// Fixed-base scalar multiplication ([s] G for public and ephemeral keys) and the sender's encrypt batch: their own
// `extern "C"` block in fixed_base.rs (methods on Engine).
mod fixed_base;

// Stealth addresses (the sender's note keys and a view key's ownership scan): their own `extern "C"` block in stealth.rs
// (methods on Engine).
mod stealth;

// Schnorr signatures over JubJub (signing and verification with the Poseidon challenge): their own `extern "C"` block in
// schnorr.rs (methods on Engine).
mod schnorr;

// JubJub point compression (JubJubAffine::from_bytes / to_bytes over a batch): their own `extern "C"` block in points.rs
// (methods on Engine).
mod points;

// JubJub multi-scalar multiplication and all-or-nothing Schnorr batch verification: their own `extern "C"` block in
// msm.rs (methods on Engine).
mod msm;

// Phoenix note nullifiers (which owned notes are spent): their own `extern "C"` block in nullifier.rs (methods on Engine).
mod nullifier;

// Double-key Schnorr signatures over G and G' and spending a note under its note secret key: their own `extern "C"`
// block in schnorr_double.rs (methods on Engine).
mod schnorr_double;

// Phoenix note values (commitments, creating obfuscated notes and their checked opening): their own `extern "C"` block in
// notes.rs (methods on Engine).
mod notes;

// Multi-key wallet scans (owner, nullifier, checked opening and per-key totals of every note): their own `extern "C"` block
// in wallet.rs (methods on Engine).
mod wallet;

// All-or-nothing batch verification of double-key Schnorr signatures (one MSM over G and G'): its own `extern "C"` block
// in verify_double_all.rs (a method on Engine).
mod verify_double_all;

// JubJub ElGamal and the encrypted sender of a Phoenix note: their own `extern "C"` block in elgamal.rs (methods on
// Engine).
mod elgamal;
pub use elgamal::SenderEncryption;

// BlsScalar::hash_to_scalar of many byte strings and BlsScalar::from_bytes_wide: their own `extern "C"` block in
// hash_to_scalar.rs (methods on Engine).
mod hash_to_scalar;
pub use hash_to_scalar::HASH_TO_SCALAR_MAX_LEN;

// Mixed digest batches (items of any domains, input and output lengths, finalized or truncated): their own `extern "C"`
// block in hash_mixed.rs (a method on Engine).
mod hash_mixed;
pub use hash_mixed::{MixedItem, MIXED_TRUNCATED};

/// Engine failures that have no dusk_poseidon::Error counterpart.
#[derive(Debug)]
pub enum BatchError {
    Poseidon(Error),
    /// a slice whose length does not match the batch shape (checked before anything reaches C)
    Shape(&'static str),
    Engine(c_int, &'static str),
}

fn status(rc: c_int) -> Result<(), BatchError> {
    // positive codes are dusk_poseidon::Error in declaration order (src/error.rs:11-32)
    match rc {
        0 => Ok(()),
        1 => Err(BatchError::Poseidon(Error::IOPatternViolation)),
        2 => Err(BatchError::Poseidon(Error::InvalidIOPattern)),
        3 => Err(BatchError::Poseidon(Error::TooFewInputElements)),
        4 => Err(BatchError::Poseidon(Error::EncryptionFailed)),
        5 => Err(BatchError::Poseidon(Error::DecryptionFailed)),
        6 => Err(BatchError::Poseidon(Error::InvalidPoint)),
        e => Err(BatchError::Engine(e, unsafe { core::ffi::CStr::from_ptr(p252_strerror(e)).to_str().unwrap_or("?") })),
    }
}

fn domain_code(d: Domain) -> c_int {
    match d {
        Domain::Merkle4 => 0,
        Domain::Merkle2 => 1,
        Domain::Encryption => 2,
        Domain::Other => 3,
    }
}

fn need(cond: bool, what: &'static str) -> Result<(), BatchError> {
    if cond { Ok(()) } else { Err(BatchError::Shape(what)) }
}

/// One CUDA device + stream.  Calls on one engine serialise inside the library (context mutex).
pub struct Engine(*mut p252_ctx);
unsafe impl Send for Engine {}

impl Engine {
    pub fn new(device: i32) -> Result<Self, BatchError> {
        let mut ctx = core::ptr::null_mut();
        status(unsafe { p252_create(device, &mut ctx) })?;
        Ok(Self(ctx))
    }

    /// `hades::permute_batch`: n independent `ScalarPermutation::permute` (states: n x 5, in place).
    pub fn permute_batch(&self, states: &mut [[BlsScalar; 5]]) -> Result<(), BatchError> {
        let n = states.len();
        let p = if n == 0 { core::ptr::NonNull::<Fr>::dangling().as_ptr() } else { &mut states[0][0].0 as *mut Fr };
        status(unsafe { p252_permute_batch(self.0, p, n, P252_MEM_HOST) })
    }

    /// `Hash::digest_batch`: `inputs.len() / in_len` independent `Hash::digest(domain, chunk)`.
    pub fn digest_batch(&self, domain: Domain, inputs: &[BlsScalar], in_len: usize, output_len: usize)
                        -> Result<Vec<BlsScalar>, BatchError> {
        need(in_len > 0 && inputs.len() % in_len == 0, "inputs.len() must be a multiple of in_len")?;
        let n = inputs.len() / in_len;
        let ol = if domain == Domain::Other && output_len > 0 { output_len } else { 1 };
        let mut out = vec![BlsScalar::zero(); n * ol];
        status(unsafe {
            p252_hash_batch(self.0, domain_code(domain), as_fr(inputs), n, in_len, as_fr_mut(&mut out), ol, P252_MEM_HOST)
        })?;
        Ok(out)
    }

    /// `Hash::digest(domain, inputs[i])` for inputs of any lengths in one call (`output_len` as `Hash::output_len`).
    pub fn digest_batch_varlen(&self, domain: Domain, inputs: &[&[BlsScalar]], output_len: usize)
                               -> Result<Vec<Vec<BlsScalar>>, BatchError> {
        let ol = if domain == Domain::Other && output_len > 0 { output_len } else { 1 };
        let data: Vec<BlsScalar> = inputs.iter().flat_map(|s| s.iter().copied()).collect();
        let mut offsets = Vec::with_capacity(inputs.len() + 1);
        offsets.push(0u64);
        for s in inputs {
            offsets.push(offsets[offsets.len() - 1] + s.len() as u64);
        }
        let longest = inputs.iter().map(|s| s.len()).max().unwrap_or(1).max(1);
        let mut out = vec![BlsScalar::zero(); inputs.len() * ol];
        status(unsafe {
            p252_hash_batch_varlen(self.0, domain_code(domain), as_fr(&data), data.len(), offsets.as_ptr(), inputs.len(),
                                   longest, as_fr_mut(&mut out), ol, core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok(out.chunks(ol).map(|c| c.to_vec()).collect())
    }

    /// `Hash::digest_truncated` batch: raw limbs for `JubJubScalar::from_raw` (src/hash.rs:164-183).
    pub fn digest_truncated_batch(&self, domain: Domain, inputs: &[BlsScalar], in_len: usize)
                                  -> Result<Vec<[u64; 4]>, BatchError> {
        need(in_len > 0 && inputs.len() % in_len == 0, "inputs.len() must be a multiple of in_len")?;
        let n = inputs.len() / in_len;
        let mut out = vec![[0u64; 4]; n];
        status(unsafe {
            p252_hash_batch_truncated(self.0, domain_code(domain), as_fr(inputs), n, in_len, out.as_mut_ptr(), 1, P252_MEM_HOST)
        })?;
        Ok(out)
    }

    /// `encrypt_batch`: messages n x L, one shared secret point and nonce per message.
    pub fn encrypt_batch(&self, messages: &[BlsScalar], l: usize, secrets: &[JubJubAffine], nonces: &[BlsScalar])
                         -> Result<Vec<BlsScalar>, BatchError> {
        let n = secrets.len();
        need(messages.len() == n * l, "messages.len() must be secrets.len() * l")?;
        need(nonces.len() == n, "nonces.len() must equal secrets.len()")?;
        let uv: Vec<BlsScalar> = secrets.iter().flat_map(|p| [p.get_u(), p.get_v()]).collect();
        let mut cipher = vec![BlsScalar::zero(); n * (l + 1)];
        status(unsafe {
            p252_encrypt_batch(self.0, as_fr(messages), n, l, as_fr(&uv), as_fr(nonces), as_fr_mut(&mut cipher),
                               P252_MEM_HOST)
        })?;
        Ok(cipher)
    }

    /// `decrypt_batch`: per-item `Result` like `dusk_poseidon::decrypt`.
    pub fn decrypt_batch(&self, ciphers: &[BlsScalar], l: usize, secrets: &[JubJubAffine], nonces: &[BlsScalar])
                         -> Result<Vec<Result<Vec<BlsScalar>, Error>>, BatchError> {
        let n = secrets.len();
        need(ciphers.len() == n * (l + 1), "ciphers.len() must be secrets.len() * (l + 1)")?;
        need(nonces.len() == n, "nonces.len() must equal secrets.len()")?;
        let uv: Vec<BlsScalar> = secrets.iter().flat_map(|p| [p.get_u(), p.get_v()]).collect();
        let mut msg = vec![BlsScalar::zero(); n * l];
        let mut ok = vec![0u8; n];
        let mut failed = 0usize;
        status(unsafe {
            p252_decrypt_batch(self.0, as_fr(ciphers), n, l, as_fr(&uv), as_fr(nonces), as_fr_mut(&mut msg),
                               ok.as_mut_ptr(), &mut failed, P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok(msg[i * l..(i + 1) * l].to_vec()) } else { Err(Error::DecryptionFailed) })
            .collect())
    }

    /// Tree of `Domain::Merkle4` / `Merkle2` digests (arity 4 / 2): internal levels bottom-up, root last.
    pub fn merkle_build(&self, arity: usize, leaves: &[BlsScalar]) -> Result<Vec<BlsScalar>, BatchError> {
        let mut n_internal = 0usize;
        status(unsafe { p252_merkle_tree_nodes(arity as c_int, leaves.len(), &mut n_internal, core::ptr::null_mut()) })?;
        let mut nodes = vec![BlsScalar::zero(); n_internal];
        status(unsafe {
            p252_merkle_build(self.0, arity as c_int, as_fr(leaves), leaves.len(), as_fr_mut(&mut nodes), P252_MEM_HOST)
        })?;
        Ok(nodes)
    }

    /// Openings (`branch` of a poseidon-merkle `Opening`): per leaf index, depth x arity scalars, level 0 first.
    pub fn merkle_open_batch(&self, arity: usize, leaves: &[BlsScalar], nodes: &[BlsScalar], leaf_idx: &[u64])
                             -> Result<Vec<BlsScalar>, BatchError> {
        let (mut n_internal, mut depth) = (0usize, 0 as c_int);
        status(unsafe { p252_merkle_tree_nodes(arity as c_int, leaves.len(), &mut n_internal, &mut depth) })?;
        need(nodes.len() == n_internal, "nodes.len() must be (n_leaves - 1) / (arity - 1)")?;
        let mut paths = vec![BlsScalar::zero(); leaf_idx.len() * depth as usize * arity];
        status(unsafe {
            p252_merkle_open_batch(self.0, arity as c_int, as_fr(leaves), leaves.len(), as_fr(nodes), leaf_idx.as_ptr(),
                                   leaf_idx.len(), as_fr_mut(&mut paths), P252_MEM_HOST)
        })?;
        Ok(paths)
    }

    /// n x `Opening::verify`: `true` where the opening proves `leaf_items[i]` under `root`.
    pub fn merkle_verify_batch(&self, arity: usize, depth: usize, leaf_items: &[BlsScalar], leaf_idx: &[u64],
                               paths: &[BlsScalar], root: &BlsScalar) -> Result<Vec<bool>, BatchError> {
        let n = leaf_items.len();
        need(leaf_idx.len() == n, "leaf_idx.len() must equal leaf_items.len()")?;
        need(paths.len() == n * depth * arity, "paths.len() must be n * depth * arity")?;
        let mut ok = vec![0u8; n];
        let mut failed = 0usize;
        status(unsafe {
            p252_merkle_verify_batch(self.0, arity as c_int, depth as c_int, as_fr(leaf_items), leaf_idx.as_ptr(),
                                     as_fr(paths), &root.0 as *const Fr, n, ok.as_mut_ptr(), &mut failed, P252_MEM_HOST)
        })?;
        Ok(ok.into_iter().map(|b| b != 0).collect())
    }
}

/// Fixed-height tree of poseidon-merkle's `Tree<T, H, A>` shape: room for `capacity <= arity^height` leaves, empty
/// slots and empty subtrees are `BlsScalar::zero()`.  `extend` / `update` rehash only the touched paths on the GPU.
pub struct Tree {
    raw: p252_mtree,
    leaves: Vec<BlsScalar>,
    nodes: Vec<BlsScalar>,
}

impl Tree {
    pub fn new(arity: usize, height: usize, capacity: u64) -> Result<Self, BatchError> {
        let (mut ls, mut ns) = (0u64, 0u64);
        status(unsafe { p252_mtree_layout(arity as c_int, height as c_int, capacity, &mut ls, &mut ns, core::ptr::null_mut()) })?;
        let raw = p252_mtree {
            struct_size: size_of::<p252_mtree>() as u32, arity: arity as i32, height: height as i32, reserved: 0,
            capacity, n_leaves: 0, leaves: core::ptr::null_mut(), nodes: core::ptr::null_mut(),
        };
        Ok(Self { raw, leaves: vec![BlsScalar::zero(); ls as usize], nodes: vec![BlsScalar::zero(); ns as usize] })
    }

    fn bind(&mut self) -> *mut p252_mtree {
        self.raw.leaves = as_fr_mut(&mut self.leaves);
        self.raw.nodes = as_fr_mut(&mut self.nodes);
        &mut self.raw
    }

    pub fn len(&self) -> u64 { self.raw.n_leaves }
    pub fn root(&self) -> BlsScalar { self.nodes[self.nodes.len() - 1] }

    /// Append `values` at `[len, len + values.len())`.
    pub fn extend(&mut self, engine: &Engine, values: &[BlsScalar]) -> Result<(), BatchError> {
        let t = self.bind();
        status(unsafe { p252_mtree_update(engine.0, t, core::ptr::null(), core::ptr::null(), 0, as_fr(values), values.len(),
                                          core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// `leaves[idx[i]] = values[i]` for indices below `len` (the last write to a leaf wins).
    pub fn update(&mut self, engine: &Engine, idx: &[u64], values: &[BlsScalar]) -> Result<(), BatchError> {
        need(idx.len() == values.len(), "idx.len() must equal values.len()")?;
        let t = self.bind();
        status(unsafe { p252_mtree_update(engine.0, t, idx.as_ptr(), as_fr(values), idx.len(), core::ptr::null(), 0,
                                          core::ptr::null_mut(), P252_MEM_HOST) })
    }
    /// Recompute every node from the leaf prefix.
    pub fn rebuild(&mut self, engine: &Engine) -> Result<(), BatchError> {
        let t = self.bind();
        status(unsafe { p252_mtree_build(engine.0, t, P252_MEM_HOST) })
    }
    /// `branch` of the poseidon-merkle `Opening` of every leaf in `leaf_idx`: height x arity scalars each, level 0 first.
    pub fn open_batch(&mut self, engine: &Engine, leaf_idx: &[u64]) -> Result<Vec<BlsScalar>, BatchError> {
        let per = (self.raw.height as usize) * (self.raw.arity as usize);
        let mut paths = vec![BlsScalar::zero(); leaf_idx.len() * per];
        let t = self.bind();
        status(unsafe { p252_mtree_open_batch(engine.0, t, leaf_idx.as_ptr(), leaf_idx.len(), as_fr_mut(&mut paths), P252_MEM_HOST) })?;
        Ok(paths)
    }
}

impl Drop for Engine {
    fn drop(&mut self) {
        unsafe { p252_destroy(self.0) }
    }
}
