//! Schnorr signatures over JubJub on the GPU: jubjub-schnorr's `SecretKey::sign` (`p252_schnorr_sign_batch`) and
//! `PublicKey::verify` (`p252_schnorr_verify_batch`), with
//! `challenge(R, m) = Hash::digest_truncated(Domain::Other, &[R.u, R.v, m])[0]`:
//!
//! ```text
//! sign   (sk, r; m):        R = G * r,  u = r - challenge(R, m) * sk  (mod r_J)
//! verify (PK; (u, R), m):   G * u + PK * challenge(R, m) == R
//! ```
//!
//! The `extern "C"` block below holds exactly these two functions; tests/c/schnorr_smoke.c calls exactly that block
//! (tests/test_schnorr_cpu.py checks both against the header).  It sits in a module of its own so that the three blocks
//! of lib.rs stay as they are.  The base G is read on the host; a G off the curve fails the whole call with
//! `BatchError::Poseidon(Error::InvalidPoint)`.  The nonce r must be secret, uniformly random and never reused: two
//! signatures with one key and one nonce reveal the key.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_schnorr_sign_batch(ctx: *mut p252_ctx, sk: *const JScalar, n_secret: usize, r: *const JScalar, msg: *const Fr,
                               n: usize, base_uv: *const Fr, u_out: *mut JScalar, r_uv: *mut Fr, ok: *mut u8,
                               n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_schnorr_verify_batch(ctx: *mut p252_ctx, pk_uv: *const Fr, n_public: usize, u: *const JScalar, r_uv: *const Fr,
                                 msg: *const Fr, n: usize, base_uv: *const Fr, verified: *mut u8, n_verified: *mut usize,
                                 n_invalid: *mut usize, flags: c_int) -> c_int;
}

fn jscalar(s: &JubJubScalar) -> JScalar {
    let b = s.to_bytes();
    let mut l = [0u64; 4];
    for (k, w) in l.iter_mut().enumerate() {
        *w = u64::from_le_bytes(b[8 * k..8 * k + 8].try_into().unwrap());
    }
    l
}

fn from_jscalar(l: &JScalar) -> JubJubScalar {
    let mut b = [0u8; 32];
    for (k, w) in l.iter().enumerate() {
        b[8 * k..8 * k + 8].copy_from_slice(&w.to_le_bytes());
    }
    JubJubScalar::from_bytes(&b).unwrap()
}

fn points(p: &[JubJubAffine]) -> Vec<BlsScalar> {
    p.iter().flat_map(|q| [q.get_u(), q.get_v()]).collect()
}

impl Engine {
    /// One signature per message with the secret keys `sk` (one key for all messages or one per message) and one fresh
    /// nonce `r[i]` per message: item i is `Ok((u, R))`, or `Err(Error::InvalidPoint)` where a scalar is not canonical.
    pub fn schnorr_sign_batch(&self, base: &JubJubAffine, sk: &[JubJubScalar], r: &[JubJubScalar], msgs: &[BlsScalar])
                              -> Result<Vec<Result<(JubJubScalar, JubJubAffine), Error>>, BatchError> {
        let n = r.len();
        need(sk.len() == 1 || sk.len() == n, "sk must hold 1 or n keys")?;
        need(msgs.len() == n, "msgs.len() must equal r.len()")?;
        let k: Vec<JScalar> = sk.iter().map(jscalar).collect();
        let s: Vec<JScalar> = r.iter().map(jscalar).collect();
        let g = points(core::slice::from_ref(base));
        let mut u = vec![[0u64; 4]; n];
        let mut rr = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_schnorr_sign_batch(self.0, k.as_ptr(), sk.len(), s.as_ptr(), as_fr(msgs), n, as_fr(&g), u.as_mut_ptr(),
                                    as_fr_mut(&mut rr), ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok((from_jscalar(&u[i]), JubJubAffine::from_raw_unchecked(rr[2 * i], rr[2 * i + 1])))
                } else {
                    Err(Error::InvalidPoint)
                }
            })
            .collect())
    }

    /// `PublicKey::verify` over the signatures `(u[i], R[i])` of `msgs[i]` under `keys` (one key for all or one per
    /// signature): `(verified, n_invalid)`.  `verified[i]` is false for a signature that does not verify and for an
    /// invalid item (R with a coordinate not canonical, a key off the curve); `n_invalid` counts the invalid ones.
    pub fn schnorr_verify_batch(&self, base: &JubJubAffine, keys: &[JubJubAffine], u: &[JubJubScalar], r_keys: &[JubJubAffine],
                                msgs: &[BlsScalar]) -> Result<(Vec<bool>, usize), BatchError> {
        let n = u.len();
        need(keys.len() == 1 || keys.len() == n, "keys must hold 1 or n points")?;
        need(r_keys.len() == n && msgs.len() == n, "r_keys and msgs must hold u.len() items")?;
        let s: Vec<JScalar> = u.iter().map(jscalar).collect();
        let (g, pk, rk) = (points(core::slice::from_ref(base)), points(keys), points(r_keys));
        let mut verified = vec![0u8; n];
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_schnorr_verify_batch(self.0, as_fr(&pk), keys.len(), s.as_ptr(), as_fr(&rk), as_fr(msgs), n, as_fr(&g),
                                      verified.as_mut_ptr(), core::ptr::null_mut(), &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((verified.into_iter().map(|o| o != 0).collect(), n_invalid))
    }
}
