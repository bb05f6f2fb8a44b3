//! Phoenix note nullifiers on the GPU (`p252_nullifier_batch`): phoenix-core's `SecretKey::gen_note_sk` and
//! `Note::gen_nullifier` over a batch of owned notes, with `hash(P) = Hash::digest_truncated(Domain::Other, &[P.u, P.v])[0]`:
//!
//! ```text
//! note_sk   = hash(R * a) + b                                  (mod r_J)
//! nullifier = Hash::digest(Domain::Other, &[pk'.u, pk'.v, BlsScalar::from(pos)])[0],   pk' = G' * note_sk
//! ```
//!
//! The shared points, note_sk and pk' never leave the device.  The `extern "C"` block below holds exactly this function;
//! tests/c/nullifier_smoke.c calls exactly that block (tests/test_nullifier_cpu.py checks both against the header).  It
//! sits in a module of its own so that the three blocks of lib.rs stay as they are.  G' (`GENERATOR_NUMS`) is read on the
//! host; off the curve it fails the whole call with `BatchError::Poseidon(Error::InvalidPoint)`.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_nullifier_batch(ctx: *mut p252_ctx, a: *const JScalar, b: *const JScalar, n_secret: usize, base_uv: *const Fr,
                            r_uv: *const Fr, pos: *const u64, n: usize, nullifier: *mut Fr, ok: *mut u8,
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
    /// The nullifier of every note `(r_keys[i], positions[i])` for the secret key `(a[k], b[k])` (one key for all notes
    /// or one per note) and the second generator `g_nums`: item i is `Ok(nullifier)`, or `Err(Error::InvalidPoint)` where
    /// `a` or `b` is not canonical or `R` is off the curve.
    pub fn nullifier_batch(&self, g_nums: &JubJubAffine, a: &[JubJubScalar], b: &[JubJubScalar], r_keys: &[JubJubAffine],
                           positions: &[u64]) -> Result<Vec<Result<BlsScalar, Error>>, BatchError> {
        let n = r_keys.len();
        need(a.len() == 1 || a.len() == n, "a must hold 1 or n items")?;
        need(b.len() == a.len(), "b.len() must equal a.len()")?;
        need(positions.len() == n, "positions.len() must equal r_keys.len()")?;
        let (sa, sb): (Vec<JScalar>, Vec<JScalar>) = (a.iter().map(jscalar).collect(), b.iter().map(jscalar).collect());
        let (g, rk) = (points(core::slice::from_ref(g_nums)), points(r_keys));
        let mut out = vec![BlsScalar::zero(); n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_nullifier_batch(self.0, sa.as_ptr(), sb.as_ptr(), a.len(), as_fr(&g), as_fr(&rk), positions.as_ptr(), n,
                                 as_fr_mut(&mut out), ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n).map(|i| if ok[i] != 0 { Ok(out[i]) } else { Err(Error::InvalidPoint) }).collect())
    }
}
