//! Stealth addresses on the GPU: the sender's `PublicKey::gen_stealth_address` (`p252_stealth_address_batch`) and a
//! wallet's `ViewKey::owns` scan (`p252_stealth_owns_batch`), with
//! `hash(P) = Hash::digest_truncated(Domain::Other, &[P.u, P.v])[0]`:
//!
//! ```text
//! sender   (r; A, B):             R = G * r,  note_pk = G * hash(A * r) + B
//! receiver (a, B; R, note_pk):    owns  <=>  note_pk == G * hash(R * a) + B
//! ```
//!
//! The shared points and their hashes never leave the device.  The `extern "C"` block below holds exactly these two
//! functions; tests/c/stealth_smoke.c calls exactly that block (tests/test_stealth_cpu.py checks both against the header).
//! It sits in a module of its own so that the three blocks of lib.rs stay as they are.  The base G and the receiver's
//! spend key B of the scan are read on the host; either one off the curve fails the whole call with
//! `BatchError::Poseidon(Error::InvalidPoint)`.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_stealth_address_batch(ctx: *mut p252_ctx, r: *const JScalar, n: usize, base_uv: *const Fr, a_uv: *const Fr,
                                  b_uv: *const Fr, n_public: usize, r_uv: *mut Fr, note_pk_uv: *mut Fr, ok: *mut u8,
                                  n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_stealth_owns_batch(ctx: *mut p252_ctx, view_a: *const JScalar, spend_b_uv: *const Fr, base_uv: *const Fr,
                               r_uv: *const Fr, note_pk_uv: *const Fr, n: usize, owned: *mut u8, n_owned: *mut usize,
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
    /// One stealth address per `r[i]` for the receiver key `(a_keys, b_keys)` (one key for all notes or one per note):
    /// item i is `Ok((R, note_pk))`, or `Err(Error::InvalidPoint)` where `r_i` is not canonical or a key is off the curve.
    pub fn stealth_address_batch(&self, base: &JubJubAffine, r: &[JubJubScalar], a_keys: &[JubJubAffine],
                                 b_keys: &[JubJubAffine])
                                 -> Result<Vec<Result<(JubJubAffine, JubJubAffine), Error>>, BatchError> {
        let n = r.len();
        need(a_keys.len() == 1 || a_keys.len() == n, "a_keys must hold 1 or n items")?;
        need(b_keys.len() == a_keys.len(), "b_keys.len() must equal a_keys.len()")?;
        let s: Vec<JScalar> = r.iter().map(jscalar).collect();
        let (g, a, b) = (points(core::slice::from_ref(base)), points(a_keys), points(b_keys));
        let mut eph = vec![BlsScalar::zero(); 2 * n];
        let mut pk = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_stealth_address_batch(self.0, s.as_ptr(), n, as_fr(&g), as_fr(&a), as_fr(&b), a_keys.len(),
                                       as_fr_mut(&mut eph), as_fr_mut(&mut pk), ok.as_mut_ptr(), core::ptr::null_mut(),
                                       P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok((JubJubAffine::from_raw_unchecked(eph[2 * i], eph[2 * i + 1]),
                        JubJubAffine::from_raw_unchecked(pk[2 * i], pk[2 * i + 1])))
                } else {
                    Err(Error::InvalidPoint)
                }
            })
            .collect())
    }

    /// `ViewKey::owns` over the notes `(r_keys[i], note_keys[i])` with view key `view_a` and spend key `spend_b`:
    /// `(owned, n_invalid)`.  `owned[i]` is false for someone else's note and for an invalid one (view key not canonical,
    /// `R` off the curve, a `note_pk` coordinate not canonical); `n_invalid` counts the invalid ones.
    pub fn stealth_owns_batch(&self, base: &JubJubAffine, view_a: &JubJubScalar, spend_b: &JubJubAffine,
                              r_keys: &[JubJubAffine], note_keys: &[JubJubAffine])
                              -> Result<(Vec<bool>, usize), BatchError> {
        let n = r_keys.len();
        need(note_keys.len() == n, "note_keys.len() must equal r_keys.len()")?;
        let a = jscalar(view_a);
        let (g, b) = (points(core::slice::from_ref(base)), points(core::slice::from_ref(spend_b)));
        let (rk, pk) = (points(r_keys), points(note_keys));
        let mut owned = vec![0u8; n];
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_stealth_owns_batch(self.0, &a, as_fr(&b), as_fr(&g), as_fr(&rk), as_fr(&pk), n, owned.as_mut_ptr(),
                                    core::ptr::null_mut(), &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((owned.into_iter().map(|o| o != 0).collect(), n_invalid))
    }
}
