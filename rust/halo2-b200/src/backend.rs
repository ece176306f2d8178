//! Safe wrappers over `ffi` with the argument meaning of the halo2-axiom functions they replace.
//! halo2curves `Fr` / `Fq` are `#[repr(transparent)] struct([u64; 4])` in Montgomery form and `G1Affine {x, y}`,
//! `G1 {x, y, z}` are plain structs of those, so slices are passed as `*const u64` without copying — the `[u64; 4]`
//! little-endian limb contract halo2-base itself relies on (halo2-base/src/utils/mod.rs:332-377).
use crate::ffi::*;
use crate::plonk::Assigned;  // the fork's own `Assigned` (halo2-axiom 0.5.3 plonk/assigned.rs), outside this directory
use halo2curves::bn256::{Fr, G1Affine, G1};
use once_cell::sync::OnceCell;
use std::ffi::CStr;

pub struct Backend { ctx: *mut H2bCtx }
unsafe impl Send for Backend {}
unsafe impl Sync for Backend {}   // the library serialises calls on one context with its own mutex (include/h2b200.h)

static BACKEND: OnceCell<Backend> = OnceCell::new();

pub fn check(ctx: *mut H2bCtx, rc: i32) {
    if rc != H2B_OK {
        let msg = unsafe { CStr::from_ptr(h2b_last_error(ctx)) }.to_string_lossy().into_owned();
        match rc {
            // where the Rust loop panics: single_phase.rs:279-286 / :304 (out of columns, missing break points)
            H2B_ERR_LAYOUT => panic!("assign_witnesses: {msg}"),
            _ => panic!("h2b200: {msg} (code {rc})"),
        }
    }
}

/// SRS handle: replaces the `g` / `g_lagrange` vectors of `ParamsKZG<Bn256>` on the device.
pub struct Srs { h: *mut H2bSrs, pub k: u32 }

/// `h2b_poly`: a column / polynomial that stays in HBM between the phases of one proof.
pub struct Poly { h: *mut H2bPoly, pub len: usize }

impl Backend {
    /// device index from `H2B200_DEVICE` (default 0); one process per GPU for multi-GPU runs
    pub fn global() -> &'static Backend {
        BACKEND.get_or_init(|| {
            let dev = std::env::var("H2B200_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
            let mut ctx = std::ptr::null_mut();
            let rc = unsafe { h2b_ctx_create(dev, &mut ctx) };
            if rc != H2B_OK {
                let msg = unsafe { CStr::from_ptr(h2b_last_error(std::ptr::null())) }.to_string_lossy().into_owned();
                panic!("h2b200: no CUDA device, and there is no CPU fallback: {msg}");
            }
            Backend { ctx }
        })
    }

    /// `ParamsKZG::setup` / `ParamsKZG::read` call this once (reference call sites halo2-base/src/utils/mod.rs:401-443)
    pub fn upload_srs(&self, g: &[G1Affine], g_lagrange: &[G1Affine], k: u32) -> Srs {
        assert_eq!(g.len(), 1 << k);
        assert_eq!(g_lagrange.len(), 1 << k);
        let mut h = std::ptr::null_mut();
        check(self.ctx, unsafe {
            h2b_srs_upload(self.ctx, g.as_ptr() as *const u64, g_lagrange.as_ptr() as *const u64, k, 0, g.len(), &mut h)
        });
        Srs { h, k }
    }

    /// `ParamsKZG::commit_lagrange` (basis = H2B_BASIS_LAGRANGE) / `commit` (H2B_BASIS_MONOMIAL): `best_multiexp(&poly, &bases)`
    pub fn commit(&self, srs: &Srs, basis: i32, poly: &[Fr]) -> G1 {
        let mut out = G1::default();
        check(self.ctx, unsafe {
            h2b_msm_g1(self.ctx, srs.h, basis, poly.as_ptr() as *const u64, poly.len(), &mut out as *mut G1 as *mut u64)
        });
        out
    }

    /// all commitments of one prover phase (advice columns, the permuted pair, the h pieces ...)
    pub fn commit_batch(&self, srs: &Srs, basis: &[i32], polys: &[&[Fr]]) -> Vec<G1> {
        let n = polys.first().map_or(0, |p| p.len());
        let ptrs: Vec<*const u64> = polys.iter().map(|p| { assert_eq!(p.len(), n); p.as_ptr() as *const u64 }).collect();
        let mut out = vec![G1::default(); polys.len()];
        check(self.ctx, unsafe {
            h2b_msm_g1_batch(self.ctx, srs.h, basis.as_ptr(), ptrs.as_ptr(), polys.len(), n, out.as_mut_ptr() as *mut u64)
        });
        out
    }

    /// `arithmetic::best_fft(a, omega, log_n)`
    pub fn best_fft(&self, a: &mut [Fr], omega: Fr, log_n: u32) {
        assert_eq!(a.len(), 1 << log_n);
        check(self.ctx, unsafe { h2b_ntt_fr(self.ctx, a.as_mut_ptr() as *mut u64, log_n, &omega as *const Fr as *const u64, 0) });
    }
    /// `EvaluationDomain::lagrange_to_coeff`
    pub fn lagrange_to_coeff(&self, a: &mut [Fr], k: u32) {
        check(self.ctx, unsafe { h2b_lagrange_to_coeff(self.ctx, a.as_mut_ptr() as *mut u64, k) });
    }
    /// `EvaluationDomain::coeff_to_extended`
    pub fn coeff_to_extended(&self, coeffs: &[Fr], extended_k: u32) -> Vec<Fr> {
        let mut out = vec![Fr::zero(); 1 << extended_k];
        check(self.ctx, unsafe {
            h2b_coeff_to_extended(self.ctx, coeffs.as_ptr() as *const u64, coeffs.len(), extended_k, out.as_mut_ptr() as *mut u64)
        });
        out
    }
    /// `EvaluationDomain::extended_to_coeff` (the caller truncates to n * (degree - 1))
    pub fn extended_to_coeff(&self, a: &mut [Fr], extended_k: u32) {
        check(self.ctx, unsafe { h2b_extended_to_coeff(self.ctx, a.as_mut_ptr() as *mut u64, extended_k) });
    }

    /// The prover branch of `SinglePhaseCoreManager::assign_raw`
    /// (halo2-base/src/gates/flex_gate/threads/single_phase.rs:152-156 -> :273-312): `vcol` is the
    /// concatenation of `ctx.advice` over `self.threads` in order (parallelize.rs:8-29 fixes that order), as
    /// [`AssignedCell`] records straight from `Vec<Assigned<Fr>>`; `break_points` is the pinned `ThreadBreakPoints`
    /// of the phase (builder.rs:181-204).  Returns `ncols` columns of 2^k rows.
    pub fn assign_witnesses(&self, vcol: &[AssignedCell], break_points: &[usize], k: u32, ncols: usize) -> Vec<Fr> {
        let bp: Vec<u64> = break_points.iter().map(|&b| b as u64).collect();
        let mut cols = vec![Fr::zero(); ncols << k];
        check(self.ctx, unsafe {
            h2b_assign_columns_assigned(self.ctx, vcol.as_ptr() as *const u64, vcol.len(), bp.as_ptr(), bp.len(), k, ncols,
                                        cols.as_mut_ptr() as *mut u64)
        });
        cols
    }

    /// halo2-base's own witness form for the resident prover (`h2b_apply_rational_dev`, `h2b_assign_lookups_indexed_dev`),
    /// built in one walk with no inversion: `threads` = (context_id, `ctx.advice`) of every thread in order (their
    /// concatenation is the virtual column); `lookups` = (context_id, offset) of every `ContextCell` that
    /// `LookupAnyManager::assign_raw` copies (virtual_region/lookups.rs:130-155), in its order.
    pub fn assigned_witness(&self, threads: &[(usize, &[Assigned<Fr>])], lookups: &[(usize, usize)]) -> AssignedWitness {
        let mut start = std::collections::HashMap::new();
        let mut w = AssignedWitness::default();
        for (id, advice) in threads {
            start.insert(*id, w.values.len() as u64);
            for a in advice.iter() {
                match a {
                    Assigned::Zero => w.values.push(Fr::zero()),
                    Assigned::Trivial(x) => w.values.push(*x),
                    Assigned::Rational(n, d) => {
                        w.rational_index.push(w.values.len() as u64);
                        w.rational_den.push(*d);
                        w.values.push(*n);
                    }
                }
            }
        }
        w.lookup_index = lookups.iter().map(|(id, off)| start[id] + *off as u64).collect();
        w
    }

    pub fn poly(&self, len: usize) -> Poly {
        let mut h = std::ptr::null_mut();
        check(self.ctx, unsafe { h2b_poly_alloc(self.ctx, len, &mut h) });
        Poly { h, len }
    }
    pub fn raw(&self) -> *mut H2bCtx { self.ctx }
}

/// `#[repr(C)]` staging record of one `Assigned<Fr>` (halo2-base/src/lib.rs:157-188 re-exports the prover crate's
/// `Assigned::{Zero, Trivial(F), Rational(F, F)}`): tag 0 = Zero, 1 = Trivial(num), 2 = Rational(num, den).
/// 72 bytes, the layout `h2b_assign_columns_assigned` consumes; the kernel batch-inverts the denominators itself.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct AssignedCell { pub tag: u64, pub num: [u64; 4], pub den: [u64; 4] }

/// halo2-base's own witness form (include/h2b200.h): `values` holds n for every `Rational(n, d)` cell;
/// (`rational_index[i]`, `rational_den[i]`) are those cells, indices strictly increasing; `lookup_index` names the
/// looked-up cells in the virtual column.  Upload the three arrays to `h2b_poly` buffers and call
/// `h2b_apply_rational_dev`, `h2b_assign_columns_dev`, `h2b_assign_lookups_indexed_dev` (INTEGRATION.md §3b).
#[derive(Default)]
pub struct AssignedWitness { pub values: Vec<Fr>, pub rational_index: Vec<u64>, pub rational_den: Vec<Fr>, pub lookup_index: Vec<u64> }

impl Poly {
    pub fn device_ptr(&self) -> *mut std::os::raw::c_void { unsafe { h2b_poly_device_ptr(self.h) } }
    pub fn upload(&self, b: &Backend, offset: usize, data: &[Fr]) {
        check(b.raw(), unsafe { h2b_poly_upload(b.raw(), self.h, offset, data.as_ptr() as *const u64, data.len()) });
    }
    pub fn download(&self, b: &Backend, offset: usize, out: &mut [Fr]) {
        check(b.raw(), unsafe { h2b_poly_download(b.raw(), self.h, offset, out.as_mut_ptr() as *mut u64, out.len()) });
    }
}
impl Drop for Srs { fn drop(&mut self) { unsafe { h2b_srs_destroy(Backend::global().raw(), self.h) } } }
impl Drop for Poly { fn drop(&mut self) { unsafe { h2b_poly_free(Backend::global().raw(), self.h) } } }
