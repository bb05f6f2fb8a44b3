//! Phoenix note values on the GPU: the Pedersen value commitment (`p252_value_commit_batch`), the sender's obfuscated
//! notes (`p252_note_create_batch`) and the wallet's checked opening (`p252_note_open_batch`), phoenix-core's
//! `Note::new` and `Note::value` / `value_blinder` as recalled, with
//! `hash(P) = Hash::digest_truncated(Domain::Other, &[P.u, P.v])[0]`:
//!
//! ```text
//! commit(v, blinder) = G * v + G' * blinder                                        (v a u64, blinder < r_J)
//! create:  R = G * r,  S = A * r,  note_pk = G * hash(S) + B,  C = commit(v, blinder),
//!          cipher = encrypt(&[BlsScalar::from(v), BlsScalar::from(blinder)], S, nonce)
//! open:    (m0, m1) = decrypt(cipher, R * a, nonce); opens iff m0 < 2^64, m1 < r_J and commit(m0, m1) == C
//! ```
//!
//! The `extern "C"` block below holds exactly these three functions; tests/c/notes_smoke.c calls exactly that block
//! (tests/test_notes_cpu.py checks both against the header).  It sits in a module of its own so that the three blocks of
//! lib.rs stay as they are.  G and G' (`GENERATOR_NUMS`) are read on the host; either off the curve fails the whole call
//! with `BatchError::Poseidon(Error::InvalidPoint)`.  S and hash(S) never leave the device; the opening (v, blinder) is
//! returned because the spend proof takes it as a witness.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_value_commit_batch(ctx: *mut p252_ctx, value: *const u64, blinder: *const JScalar, n: usize, g_uv: *const Fr,
                               gp_uv: *const Fr, commitment_uv: *mut Fr, ok: *mut u8, n_invalid: *mut usize,
                               flags: c_int) -> c_int;
    fn p252_note_create_batch(ctx: *mut p252_ctx, r: *const JScalar, value: *const u64, blinder: *const JScalar,
                              nonce: *const Fr, n: usize, g_uv: *const Fr, gp_uv: *const Fr, a_uv: *const Fr,
                              b_uv: *const Fr, n_public: usize, r_uv: *mut Fr, note_pk_uv: *mut Fr,
                              commitment_uv: *mut Fr, cipher: *mut Fr, ok: *mut u8, n_invalid: *mut usize,
                              flags: c_int) -> c_int;
    fn p252_note_open_batch(ctx: *mut p252_ctx, a: *const JScalar, n_secret: usize, r_uv: *const Fr, nonce: *const Fr,
                            cipher: *const Fr, commitment_uv: *const Fr, n: usize, g_uv: *const Fr, gp_uv: *const Fr,
                            value: *mut u64, blinder: *mut JScalar, ok: *mut u8, n_failed: *mut usize,
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

fn affine(uv: &[BlsScalar]) -> JubJubAffine {
    JubJubAffine::from_raw_unchecked(uv[0], uv[1])
}

/// One obfuscated note as `p252_note_create_batch` writes it.
pub struct CreatedNote {
    pub r_key: JubJubAffine,
    pub note_pk: JubJubAffine,
    pub commitment: JubJubAffine,
    pub cipher: [BlsScalar; 3],
}

impl Engine {
    /// `G * values[i] + G' * blinders[i]`: item i is `Ok(commitment)`, or `Err(Error::InvalidPoint)` where the blinder
    /// is not canonical.
    pub fn value_commit_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, values: &[u64], blinders: &[JubJubScalar])
                              -> Result<Vec<Result<JubJubAffine, Error>>, BatchError> {
        let n = values.len();
        need(blinders.len() == n, "blinders.len() must equal values.len()")?;
        let sb: Vec<JScalar> = blinders.iter().map(jscalar).collect();
        let (g, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let mut c = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_value_commit_batch(self.0, values.as_ptr(), sb.as_ptr(), n, as_fr(&g), as_fr(&gp), as_fr_mut(&mut c),
                                    ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n).map(|i| if ok[i] != 0 { Ok(affine(&c[2 * i..])) } else { Err(Error::InvalidPoint) }).collect())
    }

    /// Obfuscated notes of `values[i]` with `blinders[i]` for the receiver `(a_keys[k], b_keys[k])` (one key for all
    /// notes or one per note), nonce `r[i]` and cipher nonce `nonces[i]`: item i is `Ok(note)`, or
    /// `Err(Error::InvalidPoint)` where `r` or the blinder is not canonical or a receiver key is off the curve.
    pub fn note_create_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, r: &[JubJubScalar], values: &[u64],
                             blinders: &[JubJubScalar], nonces: &[BlsScalar], a_keys: &[JubJubAffine],
                             b_keys: &[JubJubAffine]) -> Result<Vec<Result<CreatedNote, Error>>, BatchError> {
        let n = r.len();
        need(values.len() == n && blinders.len() == n && nonces.len() == n, "values, blinders and nonces need r.len() items")?;
        need(a_keys.len() == 1 || a_keys.len() == n, "a_keys must hold 1 or n items")?;
        need(b_keys.len() == a_keys.len(), "b_keys.len() must equal a_keys.len()")?;
        let (sr, sb): (Vec<JScalar>, Vec<JScalar>) = (r.iter().map(jscalar).collect(), blinders.iter().map(jscalar).collect());
        let (g, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let (ak, bk) = (points(a_keys), points(b_keys));
        let (mut rk, mut pk, mut c) = (vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n]);
        let mut cipher = vec![BlsScalar::zero(); 3 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_note_create_batch(self.0, sr.as_ptr(), values.as_ptr(), sb.as_ptr(), as_fr(nonces), n, as_fr(&g), as_fr(&gp),
                                   as_fr(&ak), as_fr(&bk), a_keys.len(), as_fr_mut(&mut rk), as_fr_mut(&mut pk),
                                   as_fr_mut(&mut c), as_fr_mut(&mut cipher), ok.as_mut_ptr(), core::ptr::null_mut(),
                                   P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] == 0 {
                    return Err(Error::InvalidPoint);
                }
                Ok(CreatedNote { r_key: affine(&rk[2 * i..]), note_pk: affine(&pk[2 * i..]), commitment: affine(&c[2 * i..]),
                                 cipher: [cipher[3 * i], cipher[3 * i + 1], cipher[3 * i + 2]] })
            })
            .collect())
    }

    /// The checked openings of notes `(r_keys[i], nonces[i], ciphers[i], commitments[i])` under the view key `a[k]` (one
    /// key for all notes or one per note): item i is `Ok((value, blinder))`, or `Err(Error::DecryptionFailed)` where the
    /// note does not open or the item is invalid (`a` not canonical, `R` off the curve).
    pub fn note_open_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, a: &[JubJubScalar], r_keys: &[JubJubAffine],
                           nonces: &[BlsScalar], ciphers: &[[BlsScalar; 3]], commitments: &[JubJubAffine])
                           -> Result<Vec<Result<(u64, JubJubScalar), Error>>, BatchError> {
        let n = r_keys.len();
        need(a.len() == 1 || a.len() == n, "a must hold 1 or n items")?;
        need(nonces.len() == n && ciphers.len() == n && commitments.len() == n,
             "nonces, ciphers and commitments need r_keys.len() items")?;
        let sa: Vec<JScalar> = a.iter().map(jscalar).collect();
        let (g, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let (rk, ck) = (points(r_keys), points(commitments));
        let cf: Vec<BlsScalar> = ciphers.iter().flatten().copied().collect();
        let mut value = vec![0u64; n];
        let mut blinder = vec![[0u64; 4]; n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_note_open_batch(self.0, sa.as_ptr(), a.len(), as_fr(&rk), as_fr(nonces), as_fr(&cf), as_fr(&ck), n, as_fr(&g),
                                 as_fr(&gp), value.as_mut_ptr(), blinder.as_mut_ptr(), ok.as_mut_ptr(),
                                 core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok((value[i], from_jscalar(&blinder[i]))) } else { Err(Error::DecryptionFailed) })
            .collect())
    }
}
