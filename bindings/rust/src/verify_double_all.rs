//! All-or-nothing batch verification of double-key Schnorr signatures (`p252_schnorr_verify_double_all`) on the GPU:
//!
//! ```text
//! verify_double_all(...):  [8] ([sum z u] G + [sum z' u] G' + sum [z c] PK + sum [z' c] PK' - sum [z] R - sum [z'] R') == O
//!                          c = challenge2(R, R', msg),  z and z' the caller's two independent arrays of weights
//! ```
//!
//! The call is VARIABLE TIME (scalar bits become bucket indexes on the device): public data only.  Both weight arrays
//! must be uniformly random, unpredictable to the signers, nonzero and drawn independently of each other: with equal
//! weights only the sum of an item's two equations is checked, and a signer can make them fail by amounts that cancel.
//! The library draws no randomness.  The check is cofactored: an R shifted by a small-order point passes it and fails
//! `schnorr_verify_double_batch`.  The `extern "C"` block below holds exactly this function; tests/c/verify_double_all_smoke.c
//! calls exactly that block.  It sits in a module of its own so that the blocks of lib.rs, msm.rs and schnorr_double.rs
//! stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};

use super::{as_fr, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_schnorr_verify_double_all(ctx: *mut p252_ctx, pk_uv: *const Fr, pkp_uv: *const Fr, n_public: usize,
                                      u: *const JScalar, r_uv: *const Fr, rp_uv: *const Fr, msg: *const Fr,
                                      weight: *const JScalar, weight_p: *const JScalar, n: usize, g_uv: *const Fr,
                                      gp_uv: *const Fr, all_verified: *mut u8, n_invalid: *mut usize,
                                      flags: c_int) -> c_int;
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
    /// One answer for the double-key signatures `(u[i], R[i], R'[i])` of `msgs[i]` under `keys` / `keys_p` (one pair for
    /// all or one per signature) with the caller's two independent arrays of random weights: `(all_verified, n_invalid)`.
    #[allow(clippy::too_many_arguments)]
    pub fn schnorr_verify_double_all(&self, base: &JubJubAffine, base_p: &JubJubAffine, keys: &[JubJubAffine],
                                     keys_p: &[JubJubAffine], u: &[JubJubScalar], r_keys: &[JubJubAffine],
                                     rp_keys: &[JubJubAffine], msgs: &[BlsScalar], weights: &[JubJubScalar],
                                     weights_p: &[JubJubScalar]) -> Result<(bool, usize), BatchError> {
        let n = u.len();
        need(keys.len() == 1 || keys.len() == n, "keys must hold 1 or n points")?;
        need(keys_p.len() == keys.len(), "keys_p must hold as many points as keys")?;
        need(r_keys.len() == n && rp_keys.len() == n && msgs.len() == n, "r_keys, rp_keys and msgs must hold u.len() items")?;
        need(weights.len() == n && weights_p.len() == n, "weights and weights_p must hold u.len() items")?;
        let s: Vec<JScalar> = u.iter().map(jscalar).collect();
        let (z, zp): (Vec<JScalar>, Vec<JScalar>) = (weights.iter().map(jscalar).collect(), weights_p.iter().map(jscalar).collect());
        let (g, gp) = (points(core::slice::from_ref(base)), points(core::slice::from_ref(base_p)));
        let (pk, pkp, rk, rpk) = (points(keys), points(keys_p), points(r_keys), points(rp_keys));
        let mut all = 0u8;
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_schnorr_verify_double_all(self.0, as_fr(&pk), as_fr(&pkp), keys.len(), s.as_ptr(), as_fr(&rk), as_fr(&rpk),
                                           as_fr(msgs), z.as_ptr(), zp.as_ptr(), n, as_fr(&g), as_fr(&gp), &mut all,
                                           &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((all != 0, n_invalid))
    }
}
