//! Double-key Schnorr signatures over JubJub on the GPU: jubjub-schnorr's `SecretKey::sign_double`
//! (`p252_schnorr_sign_double_batch`) and `SignatureDouble::verify` (`p252_schnorr_verify_double_batch`), and the spend
//! signature of a Phoenix note under its note secret key (`p252_note_sign_double_batch`), with
//! `challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, &[R.u, R.v, R'.u, R'.v, m])[0]`:
//!
//! ```text
//! sign_double   (sk, r; m):                 R = G * r,  R' = G' * r,  u = r - challenge2(R, R', m) * sk  (mod r_J)
//! verify_double ((PK, PK'); (u, R, R'), m):  G * u + PK * c == R  and  G' * u + PK' * c == R'
//! note_sk = hash(R_note * a) + b  (mod r_J),   pk' = G' * note_sk
//! ```
//!
//! The `extern "C"` block below holds exactly these three functions; tests/c/schnorr_double_smoke.c calls exactly that
//! block (tests/test_schnorr_double_cpu.py checks both against the header).  It sits in a module of its own so that the
//! three blocks of lib.rs and the two functions of schnorr.rs stay as they are.  G and G' (`GENERATOR_NUMS`) are read on
//! the host; either off the curve fails the whole call with `BatchError::Poseidon(Error::InvalidPoint)`.  note_sk never
//! leaves the device; pk', returned as the spend proof's witness, links the spend to the note and must stay private.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_schnorr_sign_double_batch(ctx: *mut p252_ctx, sk: *const JScalar, n_secret: usize, r: *const JScalar,
                                      msg: *const Fr, n: usize, g_uv: *const Fr, gp_uv: *const Fr, u: *mut JScalar,
                                      r_uv: *mut Fr, rp_uv: *mut Fr, ok: *mut u8, n_invalid: *mut usize,
                                      flags: c_int) -> c_int;
    fn p252_schnorr_verify_double_batch(ctx: *mut p252_ctx, pk_uv: *const Fr, pkp_uv: *const Fr, n_public: usize,
                                        u: *const JScalar, r_uv: *const Fr, rp_uv: *const Fr, msg: *const Fr, n: usize,
                                        g_uv: *const Fr, gp_uv: *const Fr, verified: *mut u8, n_verified: *mut usize,
                                        n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_note_sign_double_batch(ctx: *mut p252_ctx, a: *const JScalar, b: *const JScalar, n_secret: usize,
                                   note_r_uv: *const Fr, r: *const JScalar, msg: *const Fr, n: usize, g_uv: *const Fr,
                                   gp_uv: *const Fr, u: *mut JScalar, r_uv: *mut Fr, rp_uv: *mut Fr, pkp_uv: *mut Fr,
                                   ok: *mut u8, n_invalid: *mut usize, flags: c_int) -> c_int;
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

fn point(s: &[BlsScalar], i: usize) -> JubJubAffine {
    JubJubAffine::from_raw_unchecked(s[2 * i], s[2 * i + 1])
}

/// A double-key signature `(u, R, R')`.
pub type SignatureDouble = (JubJubScalar, JubJubAffine, JubJubAffine);

impl Engine {
    /// One double-key signature per message with the secret keys `sk` (one key for all messages or one per message) and
    /// one fresh nonce `r[i]` per message, over the generators `g` and `g_nums`: item i is `Ok((u, R, R'))`, or
    /// `Err(Error::InvalidPoint)` where a scalar is not canonical.
    pub fn schnorr_sign_double_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, sk: &[JubJubScalar],
                                     r: &[JubJubScalar], msgs: &[BlsScalar])
                                     -> Result<Vec<Result<SignatureDouble, Error>>, BatchError> {
        let n = r.len();
        need(sk.len() == 1 || sk.len() == n, "sk must hold 1 or n keys")?;
        need(msgs.len() == n, "msgs.len() must equal r.len()")?;
        let k: Vec<JScalar> = sk.iter().map(jscalar).collect();
        let s: Vec<JScalar> = r.iter().map(jscalar).collect();
        let (gg, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let mut u = vec![[0u64; 4]; n];
        let (mut rr, mut rp) = (vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n]);
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_schnorr_sign_double_batch(self.0, k.as_ptr(), sk.len(), s.as_ptr(), as_fr(msgs), n, as_fr(&gg), as_fr(&gp),
                                           u.as_mut_ptr(), as_fr_mut(&mut rr), as_fr_mut(&mut rp), ok.as_mut_ptr(),
                                           core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok((from_jscalar(&u[i]), point(&rr, i), point(&rp, i))) } else { Err(Error::InvalidPoint) })
            .collect())
    }

    /// `SignatureDouble::verify` over the signatures `sigs[i]` of `msgs[i]` under the key pairs `(keys[k], keys_nums[k])`
    /// (one pair for all or one per signature): `(verified, n_invalid)`.  `verified[i]` is false for a signature that does
    /// not verify and for an invalid item (R or R' with a coordinate not canonical, a key off the curve); `n_invalid`
    /// counts the invalid ones.
    pub fn schnorr_verify_double_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, keys: &[JubJubAffine],
                                       keys_nums: &[JubJubAffine], sigs: &[SignatureDouble], msgs: &[BlsScalar])
                                       -> Result<(Vec<bool>, usize), BatchError> {
        let n = sigs.len();
        need(keys.len() == 1 || keys.len() == n, "keys must hold 1 or n points")?;
        need(keys_nums.len() == keys.len(), "keys_nums.len() must equal keys.len()")?;
        need(msgs.len() == n, "msgs.len() must equal sigs.len()")?;
        let s: Vec<JScalar> = sigs.iter().map(|q| jscalar(&q.0)).collect();
        let rr: Vec<JubJubAffine> = sigs.iter().map(|q| q.1).collect();
        let rp: Vec<JubJubAffine> = sigs.iter().map(|q| q.2).collect();
        let (gg, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let (pk, pkp, rr, rp) = (points(keys), points(keys_nums), points(&rr), points(&rp));
        let mut verified = vec![0u8; n];
        let mut n_invalid = 0usize;
        status(unsafe {
            p252_schnorr_verify_double_batch(self.0, as_fr(&pk), as_fr(&pkp), keys.len(), s.as_ptr(), as_fr(&rr), as_fr(&rp),
                                             as_fr(msgs), n, as_fr(&gg), as_fr(&gp), verified.as_mut_ptr(),
                                             core::ptr::null_mut(), &mut n_invalid, P252_MEM_HOST)
        })?;
        Ok((verified.into_iter().map(|o| o != 0).collect(), n_invalid))
    }

    /// The spend signature of every note `r_keys[i]` under its note secret key `hash(r_keys[i] * a) + b` for the wallet
    /// key `(a[k], b[k])` (one key for all notes or one per note), with one fresh nonce `r[i]` per note: item i is
    /// `Ok(((u, R, R'), pk'))`, or `Err(Error::InvalidPoint)` where a scalar is not canonical or the note's R is off the
    /// curve.  pk' links the spend to the note: keep it as private as the note.
    pub fn note_sign_double_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, a: &[JubJubScalar], b: &[JubJubScalar],
                                  r_keys: &[JubJubAffine], r: &[JubJubScalar], msgs: &[BlsScalar])
                                  -> Result<Vec<Result<(SignatureDouble, JubJubAffine), Error>>, BatchError> {
        let n = r.len();
        need(a.len() == 1 || a.len() == n, "a must hold 1 or n items")?;
        need(b.len() == a.len(), "b.len() must equal a.len()")?;
        need(r_keys.len() == n && msgs.len() == n, "r_keys and msgs must hold r.len() items")?;
        let (sa, sb): (Vec<JScalar>, Vec<JScalar>) = (a.iter().map(jscalar).collect(), b.iter().map(jscalar).collect());
        let s: Vec<JScalar> = r.iter().map(jscalar).collect();
        let (gg, gp, rk) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)), points(r_keys));
        let mut u = vec![[0u64; 4]; n];
        let (mut rr, mut rp, mut pkp) =
            (vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n]);
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_note_sign_double_batch(self.0, sa.as_ptr(), sb.as_ptr(), a.len(), as_fr(&rk), s.as_ptr(), as_fr(msgs), n,
                                        as_fr(&gg), as_fr(&gp), u.as_mut_ptr(), as_fr_mut(&mut rr), as_fr_mut(&mut rp),
                                        as_fr_mut(&mut pkp), ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok(((from_jscalar(&u[i]), point(&rr, i), point(&rp, i)), point(&pkp, i)))
                } else {
                    Err(Error::InvalidPoint)
                }
            })
            .collect())
    }
}
