//! `extern "C"` surface of `libspectre_b200.so` (include/spectre_b200.h) and the thin safe layer the patched halo2_proofs
//! call sites use. One declaration per C entry point the fork binds; the C header cites, for each of them, the upstream
//! item it replaces. Nothing in this file changes a halo2 signature: `arithmetic.rs`, `poly/domain.rs`,
//! `poly/kzg/commitment.rs`, `plonk/evaluation.rs` keep their public items and call in here (see ../patches/).
//!
//! Error policy (SURVEY.md 8b): every wrapper returns `Option` / `Result`; on `None` the caller runs its untouched upstream
//! CPU body, so a failing device can make a proof slower but never wrong and never aborts the prover.
//!
//! Layout contract, checked at compile time below: halo2curves keeps `Fr` / `Fq` as `[u64; 4]` Montgomery limbs and
//! `G1Affine` as `{x, y}`, `G1` as `{x, y, z}` -- byte for byte the library's `spb_fr`, `spb_g1_affine`, `spb_g1`.
#![allow(non_camel_case_types, dead_code)]

use halo2curves::bn256::{Fr, G1Affine, G1};
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};
use std::sync::OnceLock;

#[repr(C)]
pub struct spb_ctx {
    _p: [u8; 0],
}
#[repr(C)]
pub struct spb_srs {
    _p: [u8; 0],
}
#[repr(C)]
pub struct spb_domain {
    _p: [u8; 0],
}
#[repr(C)]
pub struct spb_shplonk {
    _p: [u8; 0],
}

/// `spb_graph`: the flat GraphEvaluator encoding (see `plonk/evaluation_b200.rs` for the producer).
#[repr(C)]
pub struct spb_graph {
    pub program: *const u32,
    pub program_words: usize,
    pub num_calculations: u32,
    pub num_intermediates: u32,
    pub constants: *const Fr,
    pub num_constants: u32,
    pub rotations: *const i32,
    pub num_rotations: u32,
}

/// `spb_rotation_set`: one set of `construct_intermediate_sets` (multiopen/shplonk.rs).
#[repr(C)]
pub struct spb_rotation_set {
    pub points: *const Fr,
    pub n_points: u32,
    pub d_polys: *const *const Fr,
    pub n_polys: u32,
    pub evals: *const Fr,
}

pub const SPB_BASIS_G: c_int = 0;
pub const SPB_BASIS_G_LAGRANGE: c_int = 1;
pub const SPB_ERR_CONSTRAINT: c_int = -5;
pub const SPB_ERR_DATA: c_int = -6;
pub const SPB_SERDE_RAW_BYTES: c_int = 1;
pub const SPB_SERDE_RAW_BYTES_UNCHECKED: c_int = 2;

// compile-time layout checks (the Rust side of the C header's static_assert in csrc/capi.cu)
const _: () = assert!(std::mem::size_of::<Fr>() == 32 && std::mem::align_of::<Fr>() <= 16);
const _: () = assert!(std::mem::size_of::<G1Affine>() == 64);
const _: () = assert!(std::mem::size_of::<G1>() == 96);

extern "C" {
    // ---- context ----
    pub fn spb_init(device_ids: *const c_int, n_dev: c_int) -> *mut spb_ctx;
    pub fn spb_shutdown(ctx: *mut spb_ctx);
    pub fn spb_last_error(ctx: *mut spb_ctx) -> *const c_char;
    pub fn spb_device_count() -> c_int;
    pub fn spb_stream(ctx: *mut spb_ctx, dev_index: c_int) -> *mut c_void;
    pub fn spb_host_register(ctx: *mut spb_ctx, ptr: *mut c_void, bytes: usize) -> c_int;
    pub fn spb_host_unregister(ctx: *mut spb_ctx, ptr: *mut c_void) -> c_int;
    // ---- ParamsKZG ----
    pub fn spb_srs_upload(ctx: *mut spb_ctx, k: u32, g: *const G1Affine, g_lagrange: *const G1Affine, out: *mut *mut spb_srs) -> c_int;
    pub fn spb_srs_read_file(ctx: *mut spb_ctx, path: *const c_char, out: *mut *mut spb_srs) -> c_int;
    /// `format`: SPB_SERDE_RAW_BYTES (checked, upstream's `ParamsKZG::read`) or SPB_SERDE_RAW_BYTES_UNCHECKED
    pub fn spb_srs_read_file_custom(ctx: *mut spb_ctx, path: *const c_char, format: c_int, out: *mut *mut spb_srs) -> c_int;
    pub fn spb_srs_write_file(ctx: *mut spb_ctx, srs: *const spb_srs, path: *const c_char) -> c_int;
    pub fn spb_srs_download(ctx: *mut spb_ctx, srs: *const spb_srs, basis: c_int, start: usize, count: usize, out: *mut G1Affine) -> c_int;
    pub fn spb_srs_downsize(ctx: *mut spb_ctx, srs: *const spb_srs, k: u32, out: *mut *mut spb_srs) -> c_int;
    pub fn spb_srs_precompute(ctx: *mut spb_ctx, srs: *mut spb_srs) -> c_int;
    pub fn spb_srs_free(ctx: *mut spb_ctx, srs: *mut spb_srs);
    pub fn spb_srs_k(srs: *const spb_srs) -> u32;
    // ---- MSM ----
    pub fn spb_msm_raw(ctx: *mut spb_ctx, scalars: *const Fr, bases: *const G1Affine, n: usize, out: *mut G1) -> c_int;
    /// bases of any length kept resident (an SRS handle with only basis G set): `spb_msm(handle, SPB_BASIS_G, ..)` then moves the scalars only
    pub fn spb_bases_upload(ctx: *mut spb_ctx, bases: *const G1Affine, n: usize, out: *mut *mut spb_srs) -> c_int;
    pub fn spb_msm(ctx: *mut spb_ctx, srs: *const spb_srs, basis: c_int, scalars: *const Fr, n: usize, out: *mut G1) -> c_int;
    pub fn spb_msm_batch(ctx: *mut spb_ctx, srs: *const spb_srs, basis: c_int, scalars: *const *const Fr, n: usize, count: usize, out: *mut G1) -> c_int;
    pub fn spb_msm_dev(ctx: *mut spb_ctx, srs: *const spb_srs, basis: c_int, d_scalars: *const Fr, n: usize, out: *mut G1) -> c_int;
    pub fn spb_msm_batch_dev(ctx: *mut spb_ctx, srs: *const spb_srs, basis: c_int, d_scalars: *const *const Fr, n: usize, count: usize, out: *mut G1) -> c_int;
    // ---- NTT / EvaluationDomain ----
    pub fn spb_ntt(ctx: *mut spb_ctx, a: *mut Fr, log_n: u32, omega: *const Fr) -> c_int;
    pub fn spb_domain_new(ctx: *mut spb_ctx, j: u32, k: u32, out: *mut *mut spb_domain) -> c_int;
    pub fn spb_domain_free(ctx: *mut spb_ctx, d: *mut spb_domain);
    pub fn spb_lagrange_to_coeff(ctx: *mut spb_ctx, d: *const spb_domain, a: *mut Fr) -> c_int;
    pub fn spb_coeff_to_extended(ctx: *mut spb_ctx, d: *const spb_domain, inp: *const Fr, out: *mut Fr) -> c_int;
    pub fn spb_extended_to_coeff(ctx: *mut spb_ctx, d: *const spb_domain, inp: *const Fr, out: *mut Fr) -> c_int;
    pub fn spb_divide_by_vanishing(ctx: *mut spb_ctx, d: *const spb_domain, a: *mut Fr) -> c_int;
    pub fn spb_lagrange_to_coeff_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_a: *mut Fr) -> c_int;
    pub fn spb_lagrange_to_coeff_batch_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_a: *const *mut Fr, count: usize) -> c_int;
    pub fn spb_coeff_to_extended_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_in: *const Fr, d_out: *mut Fr) -> c_int;
    pub fn spb_coeff_to_extended_batch_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_in: *const *const Fr, d_out: *const *mut Fr, count: usize) -> c_int;
    pub fn spb_extended_to_coeff_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_in: *const Fr, d_out: *mut Fr) -> c_int;
    pub fn spb_divide_by_vanishing_dev(ctx: *mut spb_ctx, d: *const spb_domain, d_a: *mut Fr) -> c_int;
    // ---- batch polynomial arithmetic ----
    pub fn spb_batch_invert(ctx: *mut spb_ctx, a: *mut Fr, n: usize) -> c_int;
    pub fn spb_eval_polynomial(ctx: *mut spb_ctx, poly: *const Fr, n: usize, point: *const Fr, out: *mut Fr) -> c_int;
    pub fn spb_kate_division(ctx: *mut spb_ctx, a: *const Fr, n: usize, b: *const Fr, q: *mut Fr) -> c_int;
    pub fn spb_eval_polynomial_dev(ctx: *mut spb_ctx, d_poly: *const Fr, n: usize, point: *const Fr, out: *mut Fr) -> c_int;
    pub fn spb_lincomb_dev(ctx: *mut spb_ctx, d_polys: *const *const Fr, count: usize, y: *const Fr, d_out: *mut Fr, n: usize) -> c_int;
    /// d_out[i] = draw number first + i of `Fr::random(&mut ChaCha20Rng::from_seed(seed))`, generated in device memory (the
    /// vanishing argument's random polynomial of a device-resident create_proof)
    pub fn spb_fr_random_chacha_dev(ctx: *mut spb_ctx, seed: *const u8, first: u64, d_out: *mut Fr, n: usize) -> c_int;
    // ---- evaluate_h ----
    pub fn spb_graph_evaluate_dev(
        ctx: *mut spb_ctx, g: *const spb_graph, d_fixed: *const *const Fr, n_fixed: u32, d_advice: *const *const Fr, n_advice: u32,
        d_instance: *const *const Fr, n_instance: u32, challenges: *const Fr, n_challenges: u32, beta: *const Fr, gamma: *const Fr,
        theta: *const Fr, y: *const Fr, d_values: *mut Fr, size: u64, rot_scale: i32,
    ) -> c_int;
    pub fn spb_permutation_constraints_dev(
        ctx: *mut spb_ctx, d_values: *mut Fr, size: u64, rot_scale: i32, last_rotation: i32, n_sets: u32, chunk_len: u32, d_z: *const *const Fr,
        n_cols: u32, d_col_values: *const *const Fr, d_sigma: *const *const Fr, d_l0: *const Fr, d_l_last: *const Fr, d_l_active: *const Fr,
        beta: *const Fr, gamma: *const Fr, y: *const Fr, extended_omega: *const Fr,
    ) -> c_int;
    pub fn spb_lookup_constraints_dev(
        ctx: *mut spb_ctx, d_values: *mut Fr, size: u64, rot_scale: i32, d_product: *const Fr, d_permuted_input: *const Fr, d_permuted_table: *const Fr,
        d_table_value: *const Fr, d_l0: *const Fr, d_l_last: *const Fr, d_l_active: *const Fr, beta: *const Fr, gamma: *const Fr, y: *const Fr,
    ) -> c_int;
    // ---- argument provers ----
    pub fn spb_permute_expression_pair_dev(ctx: *mut spb_ctx, d_input: *const Fr, d_table: *const Fr, usable: usize, d_pi: *mut Fr, d_pt: *mut Fr) -> c_int;
    pub fn spb_permutation_product_dev(
        ctx: *mut spb_ctx, k: u32, d_values: *const *const Fr, d_sigma: *const *const Fr, n_cols: u32, first_col: u32, beta: *const Fr, gamma: *const Fr,
        blinds: *const Fr, n_blinds: u32, last_z: *mut Fr, d_z: *mut Fr,
    ) -> c_int;
    pub fn spb_lookup_product_dev(
        ctx: *mut spb_ctx, n: usize, d_ci: *const Fr, d_ct: *const Fr, d_pi: *const Fr, d_pt: *const Fr, beta: *const Fr, gamma: *const Fr,
        blinds: *const Fr, n_blinds: u32, d_z: *mut Fr,
    ) -> c_int;
    // ---- SHPLONK ----
    pub fn spb_shplonk_begin_dev(
        ctx: *mut spb_ctx, srs: *const spb_srs, n: usize, sets: *const spb_rotation_set, n_sets: u32, y: *const Fr, v: *const Fr, h: *mut G1,
        out: *mut *mut spb_shplonk,
    ) -> c_int;
    pub fn spb_shplonk_finish_dev(ctx: *mut spb_ctx, s: *mut spb_shplonk, u: *const Fr, out: *mut G1) -> c_int;
    pub fn spb_shplonk_abort(ctx: *mut spb_ctx, s: *mut spb_shplonk);
    // ---- proving-key check (ProvingKey::read in SerdeFormat::RawBytes; sigma as Assembly builds it) ----
    /// `*first_out` = the first element of `d` whose stored limbs are not below r, or `n`
    pub fn spb_fr_first_noncanonical_dev(ctx: *mut spb_ctx, d: *const Fr, n: usize, first_out: *mut u64) -> c_int;
    /// per column c and kind q (0 label, 1 blinding, 2 unlabelled): `totals_out[3c + q]`, first rows at `rows_out[(3c + q) cap ..]`
    pub fn spb_sigma_check_dev(
        ctx: *mut spb_ctx, k: u32, d_sigma: *const *const Fr, n_cols: u32, usable: usize, cap: u32, rows_out: *mut u32, totals_out: *mut u64,
    ) -> c_int;
}

/// The process-wide context. `SPECTRE_B200_GPUS=N` (default 1) makes it drive N devices: SRS bases are sharded by point
/// range at upload, MSMs are split over the devices, the quotient kernels over row ranges, batches of NTTs over polynomials.
/// `SPECTRE_B200=0` disables the backend (every wrapper returns `None`, the CPU bodies run).
pub struct Ctx(pub *mut spb_ctx);
unsafe impl Send for Ctx {}
unsafe impl Sync for Ctx {} // the library serialises the calls of one context on its own lock

static CTX: OnceLock<Option<Ctx>> = OnceLock::new();

pub fn ctx() -> Option<*mut spb_ctx> {
    CTX.get_or_init(|| {
        if std::env::var("SPECTRE_B200").map(|v| v == "0").unwrap_or(false) {
            return None;
        }
        let n: c_int = std::env::var("SPECTRE_B200_GPUS").ok().and_then(|s| s.parse().ok()).unwrap_or(1);
        let p = unsafe { spb_init(std::ptr::null(), n) };
        if p.is_null() {
            log::warn!("spectre_b200: no usable CUDA device, halo2_proofs runs on the CPU");
            None
        } else {
            Some(Ctx(p))
        }
    })
    .as_ref()
    .map(|c| c.0)
}

/// A second, independent context on the same devices: what one of `--concurrency N` simultaneous proofs should use
/// (prover/src/prover.rs:114). Contexts share nothing but the GPU; a `spb_srs` may be used from any of them.
pub fn new_context() -> Option<Ctx> {
    let n: c_int = std::env::var("SPECTRE_B200_GPUS").ok().and_then(|s| s.parse().ok()).unwrap_or(1);
    let p = unsafe { spb_init(std::ptr::null(), n) };
    if p.is_null() { None } else { Some(Ctx(p)) }
}

pub fn last_error(ctx: *mut spb_ctx) -> String {
    unsafe { CStr::from_ptr(spb_last_error(ctx)).to_string_lossy().into_owned() }
}

fn ok(ctx: *mut spb_ctx, rc: c_int, what: &str) -> Option<()> {
    if rc == 0 {
        Some(())
    } else {
        log::warn!("spectre_b200: {what} failed ({rc}): {}; falling back to the CPU path", last_error(ctx));
        None
    }
}

/// `best_multiexp` front door for BN254: exact upstream semantics, bases uploaded per call.
pub fn msm_raw(coeffs: &[Fr], bases: &[G1Affine]) -> Option<G1> {
    let ctx = ctx()?;
    let mut out = std::mem::MaybeUninit::<G1>::uninit();
    let rc = unsafe { spb_msm_raw(ctx, coeffs.as_ptr(), bases.as_ptr(), coeffs.len(), out.as_mut_ptr()) };
    ok(ctx, rc, "spb_msm_raw")?;
    Some(unsafe { out.assume_init() })
}

/// `best_fft` front door for `Fr` vectors (natural order in and out, no scaling).
pub fn ntt(a: &mut [Fr], omega: Fr, log_n: u32) -> Option<()> {
    let ctx = ctx()?;
    let rc = unsafe { spb_ntt(ctx, a.as_mut_ptr(), log_n, &omega) };
    ok(ctx, rc, "spb_ntt")
}

/// Device-resident `ParamsKZG` bases (uploaded once; `ParamsKZG` holds one in a `OnceLock`, see poly/kzg/commitment_b200.rs).
pub struct GpuSrs {
    pub ctx: *mut spb_ctx,
    pub h: *mut spb_srs,
    pub k: u32,
}
unsafe impl Send for GpuSrs {}
unsafe impl Sync for GpuSrs {}

impl GpuSrs {
    pub fn upload(k: u32, g: &[G1Affine], g_lagrange: &[G1Affine]) -> Option<Self> {
        let ctx = ctx()?;
        assert_eq!(g.len(), 1usize << k);
        assert_eq!(g_lagrange.len(), 1usize << k);
        let mut h = std::ptr::null_mut();
        let rc = unsafe { spb_srs_upload(ctx, k, g.as_ptr(), g_lagrange.as_ptr(), &mut h) };
        ok(ctx, rc, "spb_srs_upload")?;
        // one-time window tables: W x the basis memory, ~20 % fewer point additions per commitment (DESIGN.md 4.3)
        if std::env::var("SPECTRE_B200_TABLES").map(|v| v != "0").unwrap_or(true) {
            let rc = unsafe { spb_srs_precompute(ctx, h) };
            if rc != 0 {
                log::warn!("spectre_b200: window tables not built ({}); commitments run without them", last_error(ctx));
            }
        }
        Some(GpuSrs { ctx, h, k })
    }

    /// Bases of any length kept resident for repeated `best_multiexp` calls against the same slice (e.g. a caller-held
    /// generator vector): `commit(SPB_BASIS_G, coeffs)` on the result is `best_multiexp(coeffs, &bases[..coeffs.len()])` and moves
    /// 32 B per pair instead of the 96 B of `msm_raw`. The caller owns the association between the slice and the handle.
    pub fn from_bases(bases: &[G1Affine]) -> Option<Self> {
        let ctx = ctx()?;
        let mut h = std::ptr::null_mut();
        let rc = unsafe { spb_bases_upload(ctx, bases.as_ptr(), bases.len(), &mut h) };
        ok(ctx, rc, "spb_bases_upload")?;
        Some(GpuSrs { ctx, h, k: usize::BITS - bases.len().saturating_sub(1).leading_zeros() })
    }

    /// `Params::commit` (basis = SPB_BASIS_G) / `commit_lagrange` (SPB_BASIS_G_LAGRANGE) of host scalars.
    pub fn commit(&self, basis: c_int, scalars: &[Fr]) -> Option<G1> {
        let mut out = std::mem::MaybeUninit::<G1>::uninit();
        let rc = unsafe { spb_msm(self.ctx, self.h, basis, scalars.as_ptr(), scalars.len(), out.as_mut_ptr()) };
        ok(self.ctx, rc, "spb_msm")?;
        Some(unsafe { out.assume_init() })
    }

    /// Several columns against the same basis in one call (create_proof commits its advice columns back to back): two
    /// stream lanes overlap one MSM's reduction tail with the next one's sort and accumulation.
    pub fn commit_batch(&self, basis: c_int, columns: &[&[Fr]]) -> Option<Vec<G1>> {
        if columns.is_empty() {
            return Some(vec![]);
        }
        let n = columns[0].len();
        assert!(columns.iter().all(|c| c.len() == n));
        let ptrs: Vec<*const Fr> = columns.iter().map(|c| c.as_ptr()).collect();
        let mut out = Vec::<G1>::with_capacity(columns.len());
        let rc = unsafe { spb_msm_batch(self.ctx, self.h, basis, ptrs.as_ptr(), n, columns.len(), out.as_mut_ptr()) };
        ok(self.ctx, rc, "spb_msm_batch")?;
        unsafe { out.set_len(columns.len()) };
        Some(out)
    }
}

impl Drop for GpuSrs {
    fn drop(&mut self) {
        unsafe { spb_srs_free(self.ctx, self.h) }
    }
}

/// Device constants of one `EvaluationDomain<Fr>` (`EvaluationDomain::new(j, k)` creates it next to the host fields).
pub struct GpuDomain {
    pub ctx: *mut spb_ctx,
    pub h: *mut spb_domain,
}
unsafe impl Send for GpuDomain {}
unsafe impl Sync for GpuDomain {}

impl GpuDomain {
    pub fn new(j: u32, k: u32) -> Option<Self> {
        let ctx = ctx()?;
        let mut h = std::ptr::null_mut();
        let rc = unsafe { spb_domain_new(ctx, j, k, &mut h) };
        ok(ctx, rc, "spb_domain_new")?;
        Some(GpuDomain { ctx, h })
    }
    pub fn lagrange_to_coeff(&self, a: &mut [Fr]) -> Option<()> {
        ok(self.ctx, unsafe { spb_lagrange_to_coeff(self.ctx, self.h, a.as_mut_ptr()) }, "spb_lagrange_to_coeff")
    }
    /// `a`: 2^k coefficients, `out`: 2^extended_k evaluations on the zeta-coset (zero padding, coset scaling inside the kernel)
    pub fn coeff_to_extended(&self, a: &[Fr], out: &mut [Fr]) -> Option<()> {
        ok(self.ctx, unsafe { spb_coeff_to_extended(self.ctx, self.h, a.as_ptr(), out.as_mut_ptr()) }, "spb_coeff_to_extended")
    }
    /// `a`: 2^extended_k evaluations, `out`: 2^k * (j - 1) coefficients
    pub fn extended_to_coeff(&self, a: &[Fr], out: &mut [Fr]) -> Option<()> {
        ok(self.ctx, unsafe { spb_extended_to_coeff(self.ctx, self.h, a.as_ptr(), out.as_mut_ptr()) }, "spb_extended_to_coeff")
    }
    pub fn divide_by_vanishing_poly(&self, a: &mut [Fr]) -> Option<()> {
        ok(self.ctx, unsafe { spb_divide_by_vanishing(self.ctx, self.h, a.as_mut_ptr()) }, "spb_divide_by_vanishing")
    }
}

impl Drop for GpuDomain {
    fn drop(&mut self) {
        unsafe { spb_domain_free(self.ctx, self.h) }
    }
}

/// `eval_polynomial`, `kate_division`, `BatchInvert` for long Fr vectors (callers keep n < 2^16 on the CPU).
pub fn eval_polynomial(poly: &[Fr], point: Fr) -> Option<Fr> {
    let ctx = ctx()?;
    let mut out = Fr::zero();
    ok(ctx, unsafe { spb_eval_polynomial(ctx, poly.as_ptr(), poly.len(), &point, &mut out) }, "spb_eval_polynomial")?;
    Some(out)
}
pub fn kate_division(a: &[Fr], b: Fr) -> Option<Vec<Fr>> {
    let ctx = ctx()?;
    let mut q = vec![Fr::zero(); a.len() - 1];
    ok(ctx, unsafe { spb_kate_division(ctx, a.as_ptr(), a.len(), &b, q.as_mut_ptr()) }, "spb_kate_division")?;
    Some(q)
}
pub fn batch_invert(a: &mut [Fr]) -> Option<()> {
    let ctx = ctx()?;
    ok(ctx, unsafe { spb_batch_invert(ctx, a.as_mut_ptr(), a.len()) }, "spb_batch_invert")
}

// ---- monomorphisation helpers used by the patched generic call sites (../patches/*.patch) -------------------------------
// halo2_proofs is generic over the curve / field; the device path exists for BN254 only. Each helper is a TypeId comparison
// (a constant after monomorphisation) followed by a pointer cast between identical types.
use crate::plonk::evaluation::GraphEvaluator;
use crate::poly::kzg::commitment::ParamsKZG;
use crate::poly::{EvaluationDomain, Polynomial};
use halo2curves::bn256::Bn256;
use halo2curves::pairing::Engine;
use std::any::TypeId;

pub(crate) fn as_bn256_params<E: Engine + 'static>(p: &ParamsKZG<E>) -> Option<&ParamsKZG<Bn256>> {
    (TypeId::of::<E>() == TypeId::of::<Bn256>()).then(|| unsafe { &*(p as *const ParamsKZG<E> as *const ParamsKZG<Bn256>) })
}
pub(crate) fn cast_g1<E: Engine + 'static>(p: G1) -> E::G1 {
    debug_assert!(TypeId::of::<E>() == TypeId::of::<Bn256>());
    unsafe { std::mem::transmute_copy::<G1, E::G1>(&p) }
}
pub(crate) fn as_fr_poly<F: 'static, B>(p: &Polynomial<F, B>) -> &Polynomial<Fr, B> {
    debug_assert!(TypeId::of::<F>() == TypeId::of::<Fr>());
    unsafe { &*(p as *const Polynomial<F, B> as *const Polynomial<Fr, B>) }
}
pub(crate) fn as_fr_poly_mut<F: 'static, B>(p: &mut Polynomial<F, B>) -> &mut Polynomial<Fr, B> {
    debug_assert!(TypeId::of::<F>() == TypeId::of::<Fr>());
    unsafe { &mut *(p as *mut Polynomial<F, B> as *mut Polynomial<Fr, B>) }
}
pub(crate) fn as_fr_domain<F: ff::Field + 'static>(d: &EvaluationDomain<F>) -> Option<&EvaluationDomain<Fr>> {
    (TypeId::of::<F>() == TypeId::of::<Fr>()).then(|| unsafe { &*(d as *const EvaluationDomain<F> as *const EvaluationDomain<Fr>) })
}
pub(crate) fn as_bn256_graph<C: halo2curves::CurveAffine + 'static>(g: &GraphEvaluator<C>) -> Option<&GraphEvaluator<G1Affine>> {
    (TypeId::of::<C>() == TypeId::of::<G1Affine>()).then(|| unsafe { &*(g as *const GraphEvaluator<C> as *const GraphEvaluator<G1Affine>) })
}
