//! Mixed digest batches (`p252_hash_batch_mixed`): every `Hash` the reference can build, of any domains, input and
//! output lengths, finalized or truncated, in one device call:
//!
//! ```text
//! item i = Hash::new(domain_i); update(input_i); output_len(output_len_i); finalize() or finalize_truncated()
//! ```
//!
//! The chunk layout of `update()` never changes a digest, so one concatenated input per item describes it.  The
//! `extern "C"` block below holds exactly this function; tests/c/hash_mixed_smoke.c calls exactly that block
//! (tests/test_hash_mixed_cpu.py checks both against the header).  It sits in a module of its own so that the blocks of
//! lib.rs stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_poseidon::Domain;

use super::{as_fr, domain_code, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `P252_MIXED_TRUNCATED`: the mode bit of an item that ends with `finalize_truncated()`
pub const MIXED_TRUNCATED: u8 = 0x80;

extern "C" {
    fn p252_hash_batch_mixed(ctx: *mut p252_ctx, mode: *const u8, input: *const Fr, n_scalars: usize, offsets: *const u64,
                             n: usize, max_len: usize, out: *mut Fr, n_out: usize, out_offsets: *const u64,
                             max_out_len: usize, n_rejected: *mut usize, flags: c_int) -> c_int;
}

/// One `Hash` of a mixed batch: `Hash::new(domain)`, `update(input)`, `output_len(output_len)` (honoured for
/// `Domain::Other` only, as the reference does), then `finalize()` or, with `truncated`, `finalize_truncated()`.
pub struct MixedItem<'a> {
    pub domain: Domain,
    pub input: &'a [BlsScalar],
    pub output_len: usize,
    pub truncated: bool,
}

impl Engine {
    /// The outputs of every item, in item order: `BlsScalar.0` limbs of `finalize()`, or for a truncated item the raw
    /// limbs `finalize_truncated()` hands to `JubJubScalar::from_raw`.  An invalid item (a Merkle arity violation, an
    /// empty input, an input or output longer than `P252_VARLEN_MAX_LEN`) fails the whole call with nothing computed.
    pub fn digest_batch_mixed(&self, items: &[MixedItem]) -> Result<Vec<Vec<Fr>>, BatchError> {
        let mut mode = Vec::with_capacity(items.len());
        let mut data: Vec<BlsScalar> = Vec::new();
        let mut offsets = vec![0u64];
        let mut out_offsets = vec![0u64];
        for it in items {
            let ol = if it.domain == Domain::Other && it.output_len > 0 { it.output_len } else { 1 };
            mode.push(domain_code(it.domain) as u8 | if it.truncated { MIXED_TRUNCATED } else { 0 });
            data.extend_from_slice(it.input);
            offsets.push(data.len() as u64);
            out_offsets.push(out_offsets[out_offsets.len() - 1] + ol as u64);
        }
        let longest = items.iter().map(|it| it.input.len()).max().unwrap_or(1).max(1);
        let longest_out = out_offsets.windows(2).map(|w| (w[1] - w[0]) as usize).max().unwrap_or(1);
        let n_out = out_offsets[items.len()] as usize;
        need(n_out < usize::MAX / 32, "too many output rows")?;
        let mut out = vec![[0u64; 4]; n_out.max(1)];
        status(unsafe {
            p252_hash_batch_mixed(self.0, mode.as_ptr(), as_fr(&data), data.len(), offsets.as_ptr(), items.len(), longest,
                                  out.as_mut_ptr(), n_out, out_offsets.as_ptr(), longest_out, core::ptr::null_mut(),
                                  P252_MEM_HOST)
        })?;
        Ok(out_offsets.windows(2).map(|w| out[w[0] as usize..w[1] as usize].to_vec()).collect())
    }
}
