//! `ParamsKZG<Bn256>` with device-resident bases ([UPSTREAM] halo2_proofs/src/poly/kzg/commitment.rs; Spectre builds the
//! params in `ProverState::new`, prover/src/prover.rs:55, and through `gen_srs` at prover/src/cli.rs:48,165,191).
//!
//! patches/commitment.patch adds ONE field to the struct,
//!     #[cfg(feature = "b200")] pub(crate) gpu: std::sync::OnceLock<Option<crate::b200::GpuSrs>>,
//! initialises it with `OnceLock::new()` in `setup`, `read_custom`, `from_parts` and `downsize` (a downsized params gets a
//! fresh, empty lock: its bases changed), and routes the two commit methods of `impl Params for ParamsKZG<Bn256>` through
//! the functions below. `g`, `g_lagrange`, `g2`, `s_g2` stay on the host as upstream has them (verifier side, `write`).

use crate::b200::{self, GpuSrs, SPB_BASIS_G, SPB_BASIS_G_LAGRANGE};
use crate::arithmetic::best_multiexp_cpu;
use crate::poly::kzg::commitment::ParamsKZG;
use crate::poly::{Coeff, LagrangeCoeff, Polynomial};
use halo2curves::bn256::{Bn256, Fr, G1};

impl ParamsKZG<Bn256> {
    /// the device copy of (g, g_lagrange), uploaded on first use and kept for the life of the params
    pub(crate) fn gpu_srs(&self) -> Option<&GpuSrs> {
        self.gpu.get_or_init(|| GpuSrs::upload(self.k, &self.g, &self.g_lagrange)).as_ref()
    }

    /// body of `Params::commit_lagrange` (the blind is ignored for KZG, as upstream)
    pub(crate) fn commit_lagrange_b200(&self, poly: &Polynomial<Fr, LagrangeCoeff>) -> G1 {
        let scalars: &[Fr] = &poly.values;
        if let Some(r) = self.gpu_srs().and_then(|h| h.commit(SPB_BASIS_G_LAGRANGE, scalars)) {
            return r;
        }
        best_multiexp_cpu(scalars, &self.g_lagrange[0..scalars.len()])
    }

    /// body of `Params::commit`
    pub(crate) fn commit_b200(&self, poly: &Polynomial<Fr, Coeff>) -> G1 {
        let scalars: &[Fr] = &poly.values;
        if let Some(r) = self.gpu_srs().and_then(|h| h.commit(SPB_BASIS_G, scalars)) {
            return r;
        }
        best_multiexp_cpu(scalars, &self.g[0..scalars.len()])
    }

    /// what create_proof's per-column loops become: all advice (or permutation / lookup product) columns in one call
    pub(crate) fn commit_lagrange_many_b200(&self, polys: &[&Polynomial<Fr, LagrangeCoeff>]) -> Vec<G1> {
        let cols: Vec<&[Fr]> = polys.iter().map(|p| &p.values[..]).collect();
        if let Some(v) = self.gpu_srs().and_then(|h| h.commit_batch(SPB_BASIS_G_LAGRANGE, &cols)) {
            return v;
        }
        cols.iter().map(|c| best_multiexp_cpu(c, &self.g_lagrange[0..c.len()])).collect()
    }
}

/// `ParamsKZG::read` (SerdeFormat::RawBytes, checked) straight into device memory: the 2 GiB `kzg_bn254_24.srs` never has to
/// be materialised as `Vec<G1Affine>` when only the prover needs it (b200::spb_srs_read_file_custom). As upstream's `read`
/// does, it rejects a file with a non-canonical coordinate or a point off its curve; the points are checked on the device.
/// The host vectors are still needed by the verifier / `write`, so the default `read` path is unchanged; this is the opt-in
/// for prover-only processes.
pub fn read_params_to_device(path: &std::path::Path) -> Option<(u32, *mut b200::spb_srs)> {
    let ctx = b200::ctx()?;
    let c = std::ffi::CString::new(path.to_str()?).ok()?;
    let mut h = std::ptr::null_mut();
    let rc = unsafe { b200::spb_srs_read_file_custom(ctx, c.as_ptr(), b200::SPB_SERDE_RAW_BYTES, &mut h) };
    if rc == b200::SPB_ERR_DATA {
        log::warn!("spectre_b200: invalid params file: {}", b200::last_error(ctx));
        return None;
    }
    if rc != 0 {
        log::warn!("spectre_b200: {}", b200::last_error(ctx));
        return None;
    }
    let _ = unsafe { b200::spb_srs_precompute(ctx, h) }; // optional: without tables the MSMs still run
    Some((unsafe { b200::spb_srs_k(h) }, h))
}
