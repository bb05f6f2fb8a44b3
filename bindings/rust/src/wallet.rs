//! Phoenix wallet scans on the GPU (`p252_wallet_scan_batch`): which of several keys owns each note, and for the owned
//! notes their nullifier and checked opening, with per-key totals, in one call.  wallet-core's `map_owned(keys, notes)`
//! and its balance, as recalled, with `hash(P) = Hash::digest_truncated(Domain::Other, &[P.u, P.v])[0]`:
//!
//! ```text
//! owner(i)     = the smallest j with note_pk == G * hash(R * a_j) + G * b_j, or none
//! nullifier(i) = Hash::digest(Domain::Other, &[pk'.u, pk'.v, pos])[0],  pk' = G' * (hash(R * a_j) + b_j)
//! opening(i)   = (m0, m1) = decrypt(cipher, R * a_j, nonce); opens iff m0 < 2^64, m1 < r_J and G * m0 + G' * m1 == C
//! ```
//!
//! The `extern "C"` block below holds exactly this function; tests/c/wallet_smoke.c calls exactly that block
//! (tests/test_wallet_cpu.py checks both against the header).  G and G' (`GENERATOR_NUMS`) are read on the host; either
//! off the curve fails the whole call with `BatchError::Poseidon(Error::InvalidPoint)`.  The keys and the shared points
//! never leave the device; the openings are returned because the spend proof takes them as witnesses.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::{JubJubAffine, JubJubScalar};

use super::{as_fr, as_fr_mut, need, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

/// `p252_jscalar`
type JScalar = [u64; 4];

/// `P252_WALLET_MAX_KEYS`
pub const WALLET_MAX_KEYS: usize = 256;

extern "C" {
    fn p252_wallet_scan_batch(ctx: *mut p252_ctx, a: *const JScalar, b: *const JScalar, n_keys: usize, r_uv: *const Fr,
                              note_pk_uv: *const Fr, pos: *const u64, nonce: *const Fr, cipher: *const Fr,
                              commitment_uv: *const Fr, n: usize, g_uv: *const Fr, gp_uv: *const Fr, owner: *mut i32,
                              nullifier: *mut Fr, value: *mut u64, blinder: *mut JScalar, opened: *mut u8,
                              key_totals: *mut u64, n_invalid: *mut usize, n_bad_keys: *mut usize, flags: c_int) -> c_int;
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

/// One note as the wallet scan sees it.
pub struct ScanNote {
    pub r_key: JubJubAffine,
    pub note_pk: JubJubAffine,
    pub pos: u64,
    pub nonce: BlsScalar,
    pub cipher: [BlsScalar; 3],
    pub commitment: JubJubAffine,
}

/// An owned note: the owning key's index, the nullifier, and the opening `(value, blinder)` if the note opens.
pub struct OwnedNote {
    pub key: usize,
    pub nullifier: BlsScalar,
    pub opening: Option<(u64, JubJubScalar)>,
}

/// Per-key totals: the 128-bit sum of the opened values, the owned and the opened notes.
pub struct KeyTotals {
    pub value: u128,
    pub n_owned: u64,
    pub n_opened: u64,
}

impl Engine {
    /// Scans `notes` with the keys `(a[j], G * b[j])`: item i is `Some(owned)` for the smallest key that owns note i, or
    /// `None` (also for an invalid note).  Keys with `a` or `b` not canonical own nothing.
    pub fn wallet_scan_batch(&self, g: &JubJubAffine, g_nums: &JubJubAffine, a: &[JubJubScalar], b: &[JubJubScalar],
                             notes: &[ScanNote]) -> Result<(Vec<Option<OwnedNote>>, Vec<KeyTotals>), BatchError> {
        let (k, n) = (a.len(), notes.len());
        need((1..=WALLET_MAX_KEYS).contains(&k), "a must hold 1 to WALLET_MAX_KEYS keys")?;
        need(b.len() == k, "b.len() must equal a.len()")?;
        let (sa, sb): (Vec<JScalar>, Vec<JScalar>) = (a.iter().map(jscalar).collect(), b.iter().map(jscalar).collect());
        let (g, gp) = (points(core::slice::from_ref(g)), points(core::slice::from_ref(g_nums)));
        let rk: Vec<BlsScalar> = notes.iter().flat_map(|x| [x.r_key.get_u(), x.r_key.get_v()]).collect();
        let pk: Vec<BlsScalar> = notes.iter().flat_map(|x| [x.note_pk.get_u(), x.note_pk.get_v()]).collect();
        let ck: Vec<BlsScalar> = notes.iter().flat_map(|x| [x.commitment.get_u(), x.commitment.get_v()]).collect();
        let pos: Vec<u64> = notes.iter().map(|x| x.pos).collect();
        let nonce: Vec<BlsScalar> = notes.iter().map(|x| x.nonce).collect();
        let cf: Vec<BlsScalar> = notes.iter().flat_map(|x| x.cipher).collect();
        let mut owner = vec![-1i32; n];
        let mut nul = vec![BlsScalar::zero(); n];
        let mut value = vec![0u64; n];
        let mut blinder = vec![[0u64; 4]; n];
        let mut opened = vec![0u8; n];
        let mut totals = vec![0u64; 4 * k];
        status(unsafe {
            p252_wallet_scan_batch(self.0, sa.as_ptr(), sb.as_ptr(), k, as_fr(&rk), as_fr(&pk), pos.as_ptr(), as_fr(&nonce),
                                   as_fr(&cf), as_fr(&ck), n, as_fr(&g), as_fr(&gp), owner.as_mut_ptr(), as_fr_mut(&mut nul),
                                   value.as_mut_ptr(), blinder.as_mut_ptr(), opened.as_mut_ptr(), totals.as_mut_ptr(),
                                   core::ptr::null_mut(), core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        let rows = (0..n)
            .map(|i| {
                (owner[i] >= 0).then(|| OwnedNote {
                    key: owner[i] as usize,
                    nullifier: nul[i],
                    opening: (opened[i] != 0).then(|| (value[i], from_jscalar(&blinder[i]))),
                })
            })
            .collect();
        let sums = totals
            .chunks(4)
            .map(|t| KeyTotals { value: (t[1] as u128) << 64 | t[0] as u128, n_owned: t[2], n_opened: t[3] })
            .collect();
        Ok((rows, sums))
    }
}
