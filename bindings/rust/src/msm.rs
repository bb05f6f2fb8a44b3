//! JubJub multi-scalar multiplication (`p252_jubjub_msm`) and all-or-nothing Schnorr batch verification
//! (`p252_schnorr_verify_all`) on the GPU:
//!
//! ```text
//! msm(s, P):          sum [s_i] P_i                                         (the identity for no items)
//! verify_all(...):    [8] ([sum z u] G + sum [z c] PK - sum [z] R) == O,     c = challenge(R, msg), z the caller's weights
//! ```
//!
//! Both calls are VARIABLE TIME (scalar bits become bucket indexes on the device): public data only.  The weights must be
//! uniformly random, unpredictable to the signers and nonzero; the library draws none.  The check is cofactored: an R
//! shifted by a small-order point passes it and fails `schnorr_verify_batch`.  The `extern "C"` block below holds exactly
//! these two functions; it sits in a module of its own so that the three blocks of lib.rs stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_jubjub_msm(ctx: *mut p252_ctx, scalars: *const JScalar, points_uv: *const Fr, n: usize, out_uv: *mut Fr,
                       n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_schnorr_verify_all(ctx: *mut p252_ctx, pk_uv: *const Fr, n_public: usize, u: *const JScalar, r_uv: *const Fr,
                               msg: *const Fr, weight: *const JScalar, n: usize, base_uv: *const Fr, all_verified: *mut u8,
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

fn points(p: &[JubJubAffine]) -> Vec<BlsScalar> {
    p.iter().flat_map(|q| [q.get_u(), q.get_v()]).collect()
}

impl Engine {
    /// `sum [scalars[i]] points[i]` (public scalars only): `(sum, n_invalid)`.
    pub fn jubjub_msm(&self, scalars: &[JubJubScalar], pts: &[JubJubAffine]) -> Result<(JubJubAffine, usize), BatchError> {
        let n = scalars.len();
        need(pts.len() == n, "points.len() must equal scalars.len()")?;
        let s: Vec<JScalar> = scalars.iter().map(jscalar).collect();
        let p = points(pts);
        let mut out = vec![BlsScalar::zero(); 2];
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_jubjub_msm(self.0, s.as_ptr(), as_fr(&p), n, as_fr_mut(&mut out), &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((JubJubAffine::from_raw_unchecked(out[0], out[1]), n_invalid))
    }

    /// One answer for the signatures `(u[i], R[i])` of `msgs[i]` under `keys` (one key for all or one per signature) with
    /// the caller's random weights: `(all_verified, n_invalid)`.
    pub fn schnorr_verify_all(&self, base: &JubJubAffine, keys: &[JubJubAffine], u: &[JubJubScalar], r_keys: &[JubJubAffine],
                              msgs: &[BlsScalar], weights: &[JubJubScalar]) -> Result<(bool, usize), BatchError> {
        let n = u.len();
        need(keys.len() == 1 || keys.len() == n, "keys must hold 1 or n points")?;
        need(r_keys.len() == n && msgs.len() == n && weights.len() == n, "r_keys, msgs and weights must hold u.len() items")?;
        let (s, z) = (u.iter().map(jscalar).collect::<Vec<_>>(), weights.iter().map(jscalar).collect::<Vec<_>>());
        let (g, pk, rk) = (points(core::slice::from_ref(base)), points(keys), points(r_keys));
        let mut all = 0u8;
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_schnorr_verify_all(self.0, as_fr(&pk), keys.len(), s.as_ptr(), as_fr(&rk), as_fr(msgs), z.as_ptr(), n,
                                    as_fr(&g), &mut all, &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((all != 0, n_invalid))
    }
}
