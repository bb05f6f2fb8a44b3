//! `BlsScalar::hash_to_scalar` of many byte strings on the GPU (`p252_hash_to_scalar_batch`) and
//! `BlsScalar::from_bytes_wide` on its own (`p252_scalars_from_bytes_wide`):
//!
//! ```text
//! hash_to_scalar(bytes) = from_bytes_wide(BLAKE2b-512(bytes))
//! from_bytes_wide(w)    = (w[0..32] + w[32..64] * 2^256) mod p      (little-endian)
//! ```
//!
//! A Phoenix payload hash `BlsScalar::hash_to_scalar(&payload.to_hash_input_bytes())` is the message every spend's
//! `SignatureDouble` signs; `hash_to_scalar_batch` computes a whole block's worth in one call.  The `extern "C"` block
//! below holds exactly these two functions; tests/c/hash_to_scalar_smoke.c calls exactly that block
//! (tests/test_hash_to_scalar_cpu.py checks both against the header).  It sits in a module of its own so that the
//! blocks of lib.rs stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;

use super::{as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `P252_HASH_TO_SCALAR_MAX_LEN`: the longest message, in bytes
pub const HASH_TO_SCALAR_MAX_LEN: usize = 1 << 20;

extern "C" {
    fn p252_hash_to_scalar_batch(ctx: *mut p252_ctx, bytes: *const u8, n_bytes: usize, offsets: *const u64, n: usize,
                                 max_len: usize, out: *mut Fr, n_rejected: *mut usize, flags: c_int) -> c_int;
    fn p252_scalars_from_bytes_wide(ctx: *mut p252_ctx, bytes: *const u8, n: usize, out: *mut Fr, flags: c_int) -> c_int;
}

impl Engine {
    /// `BlsScalar::hash_to_scalar(messages[i])` for every message, of any lengths up to `HASH_TO_SCALAR_MAX_LEN` bytes
    /// (empty ones included), in one device call.
    pub fn hash_to_scalar_batch(&self, messages: &[&[u8]]) -> Result<Vec<BlsScalar>, BatchError> {
        let longest = messages.iter().map(|m| m.len()).max().unwrap_or(0);
        need(longest <= HASH_TO_SCALAR_MAX_LEN, "a message is longer than HASH_TO_SCALAR_MAX_LEN")?;
        let mut data = Vec::with_capacity(messages.iter().map(|m| m.len()).sum());
        let mut offsets = Vec::with_capacity(messages.len() + 1);
        offsets.push(0u64);
        for m in messages {
            data.extend_from_slice(m);
            offsets.push(data.len() as u64);
        }
        let mut out = vec![BlsScalar::zero(); messages.len()];
        status(unsafe {
            p252_hash_to_scalar_batch(self.0, data.as_ptr(), data.len(), offsets.as_ptr(), messages.len(), longest,
                                      as_fr_mut(&mut out), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok(out)
    }

    /// `BlsScalar::from_bytes_wide(&wide[i])` for every 64-byte row.
    pub fn scalars_from_bytes_wide(&self, wide: &[[u8; 64]]) -> Result<Vec<BlsScalar>, BatchError> {
        let mut out = vec![BlsScalar::zero(); wide.len()];
        status(unsafe {
            p252_scalars_from_bytes_wide(self.0, wide.as_ptr() as *const u8, wide.len(), as_fr_mut(&mut out), P252_MEM_HOST)
        })?;
        Ok(out)
    }
}
