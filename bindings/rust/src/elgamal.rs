//! JubJub ElGamal on the GPU (`p252_elgamal_encrypt_batch`, `p252_elgamal_decrypt_batch`) and the encrypted sender of a
//! Phoenix note (`p252_note_sender_encrypt_batch`, `p252_note_sender_decrypt_batch`), phoenix-core's `elgamal::encrypt` /
//! `decrypt` and `Sender::Encryption` as recalled, with `hash(P) = Hash::digest_truncated(Domain::Other, &[P.u, P.v])[0]`:
//!
//! ```text
//! encrypt(PK, M; r)   = (c1, c2) = (G * r, M + PK * r)
//! decrypt(sk; c1, c2) = c2 - c1 * sk
//! sender:  [encrypt(note_pk, A; r_A), encrypt(note_pk, B; r_B)],  opened under note_sk = hash(R * a) + b  (mod r_J)
//!          only where G * note_sk == note_pk
//! ```
//!
//! ElGamal is not authenticated: `elgamal_decrypt_batch` under a wrong key returns some other point.  The sender call
//! checks ownership first and reports a note it does not own as `Err(Error::DecryptionFailed)`.  The `extern "C"` block
//! below holds exactly these four functions; tests/c/elgamal_smoke.c calls exactly that block (tests/test_elgamal_cpu.py
//! checks both against the header).  It sits in a module of its own so that the three blocks of lib.rs stay as they are.
//! G is read on the host; off the curve it fails the whole call with `BatchError::Poseidon(Error::InvalidPoint)`.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

extern "C" {
    fn p252_elgamal_encrypt_batch(ctx: *mut p252_ctx, pk_uv: *const Fr, n_public: usize, msg_uv: *const Fr,
                                  r: *const JScalar, n: usize, g_uv: *const Fr, c1_uv: *mut Fr, c2_uv: *mut Fr,
                                  ok: *mut u8, n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_elgamal_decrypt_batch(ctx: *mut p252_ctx, sk: *const JScalar, n_secret: usize, c1_uv: *const Fr,
                                  c2_uv: *const Fr, n: usize, msg_uv: *mut Fr, ok: *mut u8, n_invalid: *mut usize,
                                  flags: c_int) -> c_int;
    fn p252_note_sender_encrypt_batch(ctx: *mut p252_ctx, note_pk_uv: *const Fr, sender_a_uv: *const Fr,
                                      sender_b_uv: *const Fr, n_sender: usize, blinder: *const JScalar, n: usize,
                                      g_uv: *const Fr, sender_enc: *mut Fr, ok: *mut u8, n_invalid: *mut usize,
                                      flags: c_int) -> c_int;
    fn p252_note_sender_decrypt_batch(ctx: *mut p252_ctx, a: *const JScalar, b: *const JScalar, n_secret: usize,
                                      r_uv: *const Fr, note_pk_uv: *const Fr, sender_enc: *const Fr, n: usize,
                                      g_uv: *const Fr, sender_a_uv: *mut Fr, sender_b_uv: *mut Fr, ok: *mut u8,
                                      n_failed: *mut usize, flags: c_int) -> c_int;
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

fn affine(uv: &[BlsScalar]) -> JubJubAffine {
    JubJubAffine::from_raw_unchecked(uv[0], uv[1])
}

/// A note's encrypted sender as `p252_note_sender_encrypt_batch` writes it: `[(c1_A, c2_A), (c1_B, c2_B)]`.
pub struct SenderEncryption(pub [(JubJubAffine, JubJubAffine); 2]);

impl Engine {
    /// `(G * r[i], msgs[i] + pks[k] * r[i])` for one public key or one per message; never reuse `r` under one key.  Item i
    /// is `Ok((c1, c2))`, or `Err(Error::InvalidPoint)` where `r` is not canonical or the key or message is off the curve.
    pub fn elgamal_encrypt_batch(&self, g: &JubJubAffine, pks: &[JubJubAffine], msgs: &[JubJubAffine], r: &[JubJubScalar])
                                 -> Result<Vec<Result<(JubJubAffine, JubJubAffine), Error>>, BatchError> {
        let n = msgs.len();
        need(pks.len() == 1 || pks.len() == n, "pks must hold 1 or n items")?;
        need(r.len() == n, "r.len() must equal msgs.len()")?;
        let sr: Vec<JScalar> = r.iter().map(jscalar).collect();
        let (g, pk, m) = (points(core::slice::from_ref(g)), points(pks), points(msgs));
        let (mut c1, mut c2) = (vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n]);
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_elgamal_encrypt_batch(self.0, as_fr(&pk), pks.len(), as_fr(&m), sr.as_ptr(), n, as_fr(&g),
                                       as_fr_mut(&mut c1), as_fr_mut(&mut c2), ok.as_mut_ptr(), core::ptr::null_mut(),
                                       P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| if ok[i] != 0 { Ok((affine(&c1[2 * i..]), affine(&c2[2 * i..]))) } else { Err(Error::InvalidPoint) })
            .collect())
    }

    /// `c2[i] - c1[i] * sk[k]` for one key or one per ciphertext.  Not authenticated: a wrong key gives another point.
    /// Item i is `Ok(message)`, or `Err(Error::InvalidPoint)` where `sk` is not canonical or a point is off the curve.
    pub fn elgamal_decrypt_batch(&self, sk: &[JubJubScalar], c1: &[JubJubAffine], c2: &[JubJubAffine])
                                 -> Result<Vec<Result<JubJubAffine, Error>>, BatchError> {
        let n = c1.len();
        need(sk.len() == 1 || sk.len() == n, "sk must hold 1 or n items")?;
        need(c2.len() == n, "c2.len() must equal c1.len()")?;
        let ss: Vec<JScalar> = sk.iter().map(jscalar).collect();
        let (p1, p2) = (points(c1), points(c2));
        let mut m = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_elgamal_decrypt_batch(self.0, ss.as_ptr(), sk.len(), as_fr(&p1), as_fr(&p2), n, as_fr_mut(&mut m),
                                       ok.as_mut_ptr(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n).map(|i| if ok[i] != 0 { Ok(affine(&m[2 * i..])) } else { Err(Error::InvalidPoint) }).collect())
    }

    /// The encrypted sender `(a_keys[k], b_keys[k])` (one sender for all notes or one per note) of every note under its
    /// `note_pks[i]`, with the blinders `blinders[i] = [r_A, r_B]`: item i is `Ok(encryption)`, or
    /// `Err(Error::InvalidPoint)` where a blinder is not canonical or a point is off the curve.
    pub fn note_sender_encrypt_batch(&self, g: &JubJubAffine, note_pks: &[JubJubAffine], a_keys: &[JubJubAffine],
                                     b_keys: &[JubJubAffine], blinders: &[[JubJubScalar; 2]])
                                     -> Result<Vec<Result<SenderEncryption, Error>>, BatchError> {
        let n = note_pks.len();
        need(a_keys.len() == 1 || a_keys.len() == n, "a_keys must hold 1 or n items")?;
        need(b_keys.len() == a_keys.len(), "b_keys.len() must equal a_keys.len()")?;
        need(blinders.len() == n, "blinders.len() must equal note_pks.len()")?;
        let sb: Vec<JScalar> = blinders.iter().flatten().map(jscalar).collect();
        let (g, pk, ak, bk) = (points(core::slice::from_ref(g)), points(note_pks), points(a_keys), points(b_keys));
        let mut enc = vec![BlsScalar::zero(); 8 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_note_sender_encrypt_batch(self.0, as_fr(&pk), as_fr(&ak), as_fr(&bk), a_keys.len(), sb.as_ptr(), n,
                                           as_fr(&g), as_fr_mut(&mut enc), ok.as_mut_ptr(), core::ptr::null_mut(),
                                           P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] == 0 {
                    return Err(Error::InvalidPoint);
                }
                let e = &enc[8 * i..];
                Ok(SenderEncryption([(affine(&e[0..]), affine(&e[2..])), (affine(&e[4..]), affine(&e[6..]))]))
            })
            .collect())
    }

    /// The sender `(A, B)` of every note `(r_keys[i], note_pks[i], encs[i])` under the secret key `(a[k], b[k])` (one key
    /// for all notes or one per note): item i is `Ok((A, B))`, or `Err(Error::DecryptionFailed)` where the key does not own
    /// the note or the item is invalid.
    pub fn note_sender_decrypt_batch(&self, g: &JubJubAffine, a: &[JubJubScalar], b: &[JubJubScalar],
                                     r_keys: &[JubJubAffine], note_pks: &[JubJubAffine], encs: &[SenderEncryption])
                                     -> Result<Vec<Result<(JubJubAffine, JubJubAffine), Error>>, BatchError> {
        let n = r_keys.len();
        need(a.len() == 1 || a.len() == n, "a must hold 1 or n items")?;
        need(b.len() == a.len(), "b.len() must equal a.len()")?;
        need(note_pks.len() == n && encs.len() == n, "note_pks and encs need r_keys.len() items")?;
        let (sa, sb): (Vec<JScalar>, Vec<JScalar>) = (a.iter().map(jscalar).collect(), b.iter().map(jscalar).collect());
        let (g, rk, pk) = (points(core::slice::from_ref(g)), points(r_keys), points(note_pks));
        let ef: Vec<BlsScalar> =
            encs.iter().flat_map(|e| points(&[e.0[0].0, e.0[0].1, e.0[1].0, e.0[1].1])).collect();
        let (mut sa_out, mut sb_out) = (vec![BlsScalar::zero(); 2 * n], vec![BlsScalar::zero(); 2 * n]);
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_note_sender_decrypt_batch(self.0, sa.as_ptr(), sb.as_ptr(), a.len(), as_fr(&rk), as_fr(&pk), as_fr(&ef), n,
                                           as_fr(&g), as_fr_mut(&mut sa_out), as_fr_mut(&mut sb_out), ok.as_mut_ptr(),
                                           core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 { Ok((affine(&sa_out[2 * i..]), affine(&sb_out[2 * i..]))) } else { Err(Error::DecryptionFailed) }
            })
            .collect())
    }
}
