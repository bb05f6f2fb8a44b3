//! Encrypt / decrypt batches over messages of different lengths (`p252_encrypt_batch_varlen` /
//! `p252_decrypt_batch_varlen`): `dusk_poseidon::{encrypt, decrypt}` on slices of any length, one GPU call for the whole
//! batch.  The `extern "C"` block below holds exactly these two functions; tests/c/crypt_varlen_smoke.c calls exactly
//! that block (tests/test_crypt_varlen_bindings.py checks both against the header).  It sits in a module of its own so
//! that the three blocks of lib.rs stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::JubJubAffine;
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

extern "C" {
    fn p252_encrypt_batch_varlen(ctx: *mut p252_ctx, msg: *const Fr, n_scalars: usize, offsets: *const u64, n: usize,
                                 max_len: usize, secret_uv: *const Fr, nonce: *const Fr, cipher: *mut Fr,
                                 n_rejected: *mut usize, flags: c_int) -> c_int;
    fn p252_decrypt_batch_varlen(ctx: *mut p252_ctx, cipher: *const Fr, n_scalars: usize, offsets: *const u64, n: usize,
                                 max_len: usize, secret_uv: *const Fr, nonce: *const Fr, msg: *mut Fr, ok: *mut u8,
                                 n_failed: *mut usize, n_rejected: *mut usize, flags: c_int) -> c_int;
}

/// The slices back to back plus their n + 1 offsets and the longest length.
fn pack(items: &[&[BlsScalar]]) -> (Vec<BlsScalar>, Vec<u64>, usize) {
    let data: Vec<BlsScalar> = items.iter().flat_map(|s| s.iter().copied()).collect();
    let mut offsets = Vec::with_capacity(items.len() + 1);
    offsets.push(0u64);
    for s in items {
        offsets.push(offsets[offsets.len() - 1] + s.len() as u64);
    }
    (data, offsets, items.iter().map(|s| s.len()).max().unwrap_or(0))
}

impl Engine {
    /// `encrypt(messages[i], secrets[i], nonces[i])` for messages of any lengths, one call; cipher i has
    /// `messages[i].len() + 1` scalars.  An empty message fails the whole batch (nothing is computed).
    pub fn encrypt_batch_varlen(&self, messages: &[&[BlsScalar]], secrets: &[JubJubAffine], nonces: &[BlsScalar])
                                -> Result<Vec<Vec<BlsScalar>>, BatchError> {
        let n = messages.len();
        need(secrets.len() == n, "secrets.len() must equal messages.len()")?;
        need(nonces.len() == n, "nonces.len() must equal messages.len()")?;
        let (data, offsets, longest) = pack(messages);
        let uv: Vec<BlsScalar> = secrets.iter().flat_map(|p| [p.get_u(), p.get_v()]).collect();
        let mut cipher = vec![BlsScalar::zero(); data.len() + n];
        status(unsafe {
            p252_encrypt_batch_varlen(self.0, as_fr(&data), data.len(), offsets.as_ptr(), n, longest.max(1), as_fr(&uv),
                                      as_fr(nonces), as_fr_mut(&mut cipher), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n).map(|i| cipher[offsets[i] as usize + i..offsets[i + 1] as usize + i + 1].to_vec()).collect())
    }

    /// `decrypt(ciphers[i], secrets[i], nonces[i])` for ciphers of any lengths, one call: a per-item `Result` like
    /// `dusk_poseidon::decrypt`.  A cipher shorter than 2 scalars fails the whole batch (nothing is computed).
    pub fn decrypt_batch_varlen(&self, ciphers: &[&[BlsScalar]], secrets: &[JubJubAffine], nonces: &[BlsScalar])
                                -> Result<Vec<Result<Vec<BlsScalar>, Error>>, BatchError> {
        let n = ciphers.len();
        need(secrets.len() == n, "secrets.len() must equal ciphers.len()")?;
        need(nonces.len() == n, "nonces.len() must equal ciphers.len()")?;
        let (data, offsets, longest) = pack(ciphers);
        let uv: Vec<BlsScalar> = secrets.iter().flat_map(|p| [p.get_u(), p.get_v()]).collect();
        let mut msg = vec![BlsScalar::zero(); data.len().saturating_sub(n)];
        let mut ok = vec![0u8; n];
        let mut failed = 0usize;
        status(unsafe {
            p252_decrypt_batch_varlen(self.0, as_fr(&data), data.len(), offsets.as_ptr(), n, longest.saturating_sub(1).max(1),
                                      as_fr(&uv), as_fr(nonces), as_fr_mut(&mut msg), ok.as_mut_ptr(), &mut failed,
                                      core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok(msg[offsets[i] as usize - i..offsets[i + 1] as usize - i - 1].to_vec())
                } else {
                    Err(Error::DecryptionFailed)
                }
            })
            .collect())
    }
}
