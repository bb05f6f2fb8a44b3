//! JubJub key exchange on the GPU (`p252_dhke_batch`) and encrypt / decrypt batches that derive their shared secret
//! with it (`p252_encrypt_batch_dhke` / `p252_decrypt_batch_dhke`): `dusk_poseidon::{encrypt, decrypt}` with
//! `shared_secret = dhke(secret, public)` (src/encryption.rs:11-43), the shared secret never leaving the device.  The
//! `extern "C"` block below holds exactly these three functions; tests/c/dhke_smoke.c calls exactly that block
//! (tests/test_jubjub_cpu.py checks both against the header).  It sits in a module of its own so that the three blocks of
//! lib.rs stay as they are.
//!
//! Secrets cross the boundary as `p252_jscalar`: the canonical little-endian integer of `JubJubScalar::to_bytes()` (not
//! the crate's internal limbs); points as `(get_u().0, get_v().0)`.  `secrets` and `publics` each hold 1 (broadcast) or
//! n items.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
pub type JScalar = [u64; 4];

extern "C" {
    fn p252_dhke_batch(ctx: *mut p252_ctx, secret: *const JScalar, n_secret: usize, public_uv: *const Fr, n_public: usize,
                       n: usize, shared_uv: *mut Fr, ok: *mut u8, n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_encrypt_batch_dhke(ctx: *mut p252_ctx, msg: *const Fr, n: usize, l: usize, secret: *const JScalar,
                               n_secret: usize, public_uv: *const Fr, n_public: usize, nonce: *const Fr, cipher: *mut Fr,
                               ok: *mut u8, n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_decrypt_batch_dhke(ctx: *mut p252_ctx, cipher: *const Fr, n: usize, l: usize, secret: *const JScalar,
                               n_secret: usize, public_uv: *const Fr, n_public: usize, nonce: *const Fr, msg: *mut Fr,
                               ok: *mut u8, n_failed: *mut usize, flags: c_int) -> c_int;
}

fn jscalars(secrets: &[JubJubScalar]) -> Vec<JScalar> {
    secrets
        .iter()
        .map(|s| {
            let b = s.to_bytes();
            let mut l = [0u64; 4];
            for (k, w) in l.iter_mut().enumerate() {
                *w = u64::from_le_bytes(b[8 * k..8 * k + 8].try_into().unwrap());
            }
            l
        })
        .collect()
}

fn points(publics: &[JubJubAffine]) -> Vec<BlsScalar> {
    publics.iter().flat_map(|p| [p.get_u(), p.get_v()]).collect()
}

/// the batch size of a (secrets, publics) pair: each is 1 or n
fn shape(n_secret: usize, n_public: usize, n: Option<usize>) -> Result<usize, BatchError> {
    let n = n.unwrap_or(if n_secret == 1 { n_public } else { n_secret });
    need(n_secret == 1 || n_secret == n, "secrets must hold 1 or n items")?;
    need(n_public == 1 || n_public == n, "publics must hold 1 or n items")?;
    Ok(n)
}

impl Engine {
    /// `dhke(secrets[i], publics[i])` for every item (either slice may hold one item, used by all): a per-item `Result`,
    /// `Err(Error::InvalidPoint)` where the point is not on the curve.
    pub fn dhke_batch(&self, secrets: &[JubJubScalar], publics: &[JubJubAffine])
                      -> Result<Vec<Result<JubJubAffine, Error>>, BatchError> {
        let n = shape(secrets.len(), publics.len(), None)?;
        let (s, p) = (jscalars(secrets), points(publics));
        let mut out = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_dhke_batch(self.0, s.as_ptr(), s.len(), as_fr(&p), publics.len(), n, as_fr_mut(&mut out), ok.as_mut_ptr(),
                            core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok(JubJubAffine::from_raw_unchecked(out[2 * i], out[2 * i + 1])) } else { Err(Error::InvalidPoint) })
            .collect())
    }

    /// `encrypt(messages[i], &dhke(secrets[i], publics[i]), &nonces[i])`, messages of one length L, one call; cipher i is
    /// `Err(Error::InvalidPoint)` where the key exchange was invalid.
    pub fn encrypt_batch_dhke(&self, messages: &[&[BlsScalar]], secrets: &[JubJubScalar], publics: &[JubJubAffine],
                              nonces: &[BlsScalar]) -> Result<Vec<Result<Vec<BlsScalar>, Error>>, BatchError> {
        let n = shape(secrets.len(), publics.len(), Some(messages.len()))?;
        need(nonces.len() == n, "nonces.len() must equal messages.len()")?;
        let l = messages.first().map_or(1, |m| m.len());
        need(messages.iter().all(|m| m.len() == l), "messages must have one length")?;
        let data: Vec<BlsScalar> = messages.iter().flat_map(|m| m.iter().copied()).collect();
        let (s, p) = (jscalars(secrets), points(publics));
        let mut cipher = vec![BlsScalar::zero(); n * (l + 1)];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_encrypt_batch_dhke(self.0, as_fr(&data), n, l, s.as_ptr(), s.len(), as_fr(&p), publics.len(), as_fr(nonces),
                                    as_fr_mut(&mut cipher), ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok(cipher[i * (l + 1)..(i + 1) * (l + 1)].to_vec()) } else { Err(Error::InvalidPoint) })
            .collect())
    }

    /// `decrypt(ciphers[i], &dhke(secrets[i], publics[i]), &nonces[i])`, ciphers of one length, one call -- the wallet scan
    /// passes one view key in `secrets`.  A failed item is `Err(Error::DecryptionFailed)`, whether authentication failed
    /// or the key exchange was invalid.
    pub fn decrypt_batch_dhke(&self, ciphers: &[&[BlsScalar]], secrets: &[JubJubScalar], publics: &[JubJubAffine],
                              nonces: &[BlsScalar]) -> Result<Vec<Result<Vec<BlsScalar>, Error>>, BatchError> {
        let n = shape(secrets.len(), publics.len(), Some(ciphers.len()))?;
        need(nonces.len() == n, "nonces.len() must equal ciphers.len()")?;
        let c = ciphers.first().map_or(2, |m| m.len());
        need(c >= 2 && ciphers.iter().all(|m| m.len() == c), "ciphers must have one length of at least 2")?;
        let data: Vec<BlsScalar> = ciphers.iter().flat_map(|m| m.iter().copied()).collect();
        let (s, p) = (jscalars(secrets), points(publics));
        let mut msg = vec![BlsScalar::zero(); n * (c - 1)];
        let mut ok = vec![0u8; n];
        let mut failed = 0usize;
        status(unsafe {
            p252_decrypt_batch_dhke(self.0, as_fr(&data), n, c - 1, s.as_ptr(), s.len(), as_fr(&p), publics.len(),
                                    as_fr(nonces), as_fr_mut(&mut msg), ok.as_mut_ptr(), &mut failed, P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok(msg[i * (c - 1)..(i + 1) * (c - 1)].to_vec()) } else { Err(Error::DecryptionFailed) })
            .collect())
    }
}
