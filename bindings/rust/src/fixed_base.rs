//! Fixed-base JubJub scalar multiplication on the GPU (`p252_fixed_base_batch`) and the sender's side of the key
//! exchange as one call (`p252_encrypt_batch_ephemeral`): `GENERATOR_EXTENDED * &r` for every note, plus
//! `dusk_poseidon::encrypt(msg, &dhke(&r, &pk), &nonce)` with the shared secret never leaving the device
//! (src/encryption.rs:22-42).  The `extern "C"` block below holds exactly these two functions; tests/c/fixed_base_smoke.c
//! calls exactly that block (tests/test_fixed_base_cpu.py checks both against the header).  It sits in a module of its
//! own so that the three blocks of lib.rs stay as they are.
//!
//! The base is always the caller's: pass `dusk_jubjub::GENERATOR` for public keys and ephemeral keys.  It is read on the
//! host; a base off the curve fails the whole call with `BatchError::Poseidon(Error::InvalidPoint)`.  Secrets cross the
//! boundary as `p252_jscalar` (the canonical little-endian integer of `JubJubScalar::to_bytes()`).
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_fixed_base_batch(ctx: *mut p252_ctx, base_uv: *const Fr, secret: *const JScalar, n: usize, out_uv: *mut Fr,
                             ok: *mut u8, n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_encrypt_batch_ephemeral(ctx: *mut p252_ctx, msg: *const Fr, n: usize, l: usize, r: *const JScalar,
                                    base_uv: *const Fr, public_uv: *const Fr, n_public: usize, nonce: *const Fr,
                                    cipher: *mut Fr, r_uv: *mut Fr, ok: *mut u8, n_invalid: *mut usize, flags: c_int)
                                    -> c_int;
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

fn point(p: &JubJubAffine) -> [BlsScalar; 2] {
    [p.get_u(), p.get_v()]
}

impl Engine {
    /// `base * secrets[i]` for every item, one base for the batch (e.g. `GENERATOR` for public or ephemeral keys): a
    /// per-item `Result`, `Err(Error::InvalidPoint)` where the secret is not a canonical scalar.
    pub fn fixed_base_batch(&self, base: &JubJubAffine, secrets: &[JubJubScalar])
                            -> Result<Vec<Result<JubJubAffine, Error>>, BatchError> {
        let n = secrets.len();
        let (s, b) = (jscalars(secrets), point(base));
        let mut out = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_fixed_base_batch(self.0, as_fr(&b), s.as_ptr(), n, as_fr_mut(&mut out), ok.as_mut_ptr(),
                                  core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok(JubJubAffine::from_raw_unchecked(out[2 * i], out[2 * i + 1])) } else { Err(Error::InvalidPoint) })
            .collect())
    }

    /// The sender, one note per item: `R_i = base * r_i` and `encrypt(messages[i], &dhke(&r_i, &publics[i]), &nonces[i])`,
    /// messages of one length L; `publics` holds one receiver key for all notes or one per note.  Item i is
    /// `Ok((cipher, R))`, or `Err(Error::InvalidPoint)` where `r_i` or the receiver key was invalid.
    pub fn encrypt_batch_ephemeral(&self, messages: &[&[BlsScalar]], r: &[JubJubScalar], base: &JubJubAffine,
                                   publics: &[JubJubAffine], nonces: &[BlsScalar])
                                   -> Result<Vec<Result<(Vec<BlsScalar>, JubJubAffine), Error>>, BatchError> {
        let n = messages.len();
        need(r.len() == n, "r.len() must equal messages.len()")?;
        need(publics.len() == 1 || publics.len() == n, "publics must hold 1 or n items")?;
        need(nonces.len() == n, "nonces.len() must equal messages.len()")?;
        let l = messages.first().map_or(1, |m| m.len());
        need(messages.iter().all(|m| m.len() == l), "messages must have one length")?;
        let data: Vec<BlsScalar> = messages.iter().flat_map(|m| m.iter().copied()).collect();
        let p: Vec<BlsScalar> = publics.iter().flat_map(point).collect();
        let (s, b) = (jscalars(r), point(base));
        let mut cipher = vec![BlsScalar::zero(); n * (l + 1)];
        let mut eph = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_encrypt_batch_ephemeral(self.0, as_fr(&data), n, l, s.as_ptr(), as_fr(&b), as_fr(&p), publics.len(),
                                         as_fr(nonces), as_fr_mut(&mut cipher), as_fr_mut(&mut eph), ok.as_mut_ptr(),
                                         core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok((cipher[i * (l + 1)..(i + 1) * (l + 1)].to_vec(),
                        JubJubAffine::from_raw_unchecked(eph[2 * i], eph[2 * i + 1])))
                } else {
                    Err(Error::InvalidPoint)
                }
            })
            .collect())
    }
}
