//! JubJub point compression on the GPU: dusk-jubjub's `JubJubAffine::from_bytes` (`p252_points_from_bytes`) and
//! `JubJubAffine::to_bytes` (`p252_points_to_bytes`) over a batch:
//!
//! ```text
//! to_bytes(u, v):   the 32 little-endian bytes of canonical v, bit 255 = the low bit of canonical u
//! from_bytes(b):    v = b without bit 255 (< p), u^2 = (v^2 - 1) / (1 + d v^2) a square, u the root with that low bit
//! ```
//!
//! A set sign bit with u = 0 is accepted (pre-ZIP-216).  The `extern "C"` block below holds exactly these two functions;
//! tests/c/points_smoke.c calls exactly that block (tests/test_points_cpu.py checks both against the header).  It sits in a
//! module of its own so that the three blocks of lib.rs stay as they are.
use core::ffi::c_int;
use dusk_bls12_381::BlsScalar;
use dusk_jubjub::JubJubAffine;
use dusk_poseidon::Error;

use super::{as_fr, as_fr_mut, p252_ctx, status, BatchError, Engine, Fr, P252_MEM_HOST};

extern "C" {
    fn p252_points_from_bytes(ctx: *mut p252_ctx, bytes: *const u8, n: usize, out_uv: *mut Fr, ok: *mut u8,
                              n_invalid: *mut usize, flags: c_int) -> c_int;
    fn p252_points_to_bytes(ctx: *mut p252_ctx, uv: *const Fr, n: usize, bytes: *mut u8, ok: *mut u8, n_invalid: *mut usize,
                            flags: c_int) -> c_int;
}

impl Engine {
    /// `JubJubAffine::from_bytes` per encoding: item i is `Ok(point)`, or `Err(Error::InvalidPoint)` where v is not
    /// canonical or u^2 is not a square.
    pub fn points_from_bytes_batch(&self, bytes: &[[u8; 32]]) -> Result<Vec<Result<JubJubAffine, Error>>, BatchError> {
        let n = bytes.len();
        let mut uv = vec![BlsScalar::zero(); 2 * n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_points_from_bytes(self.0, bytes.as_ptr() as *const u8, n, as_fr_mut(&mut uv), ok.as_mut_ptr(),
                                   core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok((0..n)
            .map(|i| {
                if ok[i] != 0 {
                    Ok(JubJubAffine::from_raw_unchecked(uv[2 * i], uv[2 * i + 1]))
                } else {
                    Err(Error::InvalidPoint)
                }
            })
            .collect())
    }

    /// `JubJubAffine::to_bytes` per point: item i is `Ok(bytes)`, or `Err(Error::InvalidPoint)` for a point off the curve
    /// (e.g. one built with `from_raw_unchecked`).
    pub fn points_to_bytes_batch(&self, points: &[JubJubAffine]) -> Result<Vec<Result<[u8; 32], Error>>, BatchError> {
        let n = points.len();
        let uv: Vec<BlsScalar> = points.iter().flat_map(|q| [q.get_u(), q.get_v()]).collect();
        let mut bytes = vec![[0u8; 32]; n];
        let mut ok = vec![0u8; n];
        status(unsafe {
            p252_points_to_bytes(self.0, as_fr(&uv), n, bytes.as_mut_ptr() as *mut u8, ok.as_mut_ptr(),
                                 core::ptr::null_mut(), P252_MEM_HOST)
        })?;
        Ok(bytes.into_iter().zip(ok).map(|(b, o)| if o != 0 { Ok(b) } else { Err(Error::InvalidPoint) }).collect())
    }
}
