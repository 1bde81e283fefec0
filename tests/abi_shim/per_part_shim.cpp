// TEST INFRASTRUCTURE -- the CPU stand-in of the C ABI (shim.cpp, included whole) plus the three entry points a per-part proof
// calls, restated over the oracle's whole-coset routines so that include/spectre_b200_prover.hpp runs Cosets::PerPart on the
// CPU. Build this file instead of shim.cpp; it is never built into, linked with or loaded by the product.
#include "shim.cpp"

extern "C" {
void orc_fr_mul(fe* o, const fe* a, const fe* b);
void orc_fr_inv(fe* o, const fe* a);
void orc_fr_constants(fe* root_of_unity, fe* zeta, fe* one);

// part j of the coset: the oracle's whole coset, rows j, j + R, ...
int spb_coeff_to_extended_part_batch_dev(spb_ctx* ctx, const spb_domain* d, uint32_t part, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count) {
  const uint32_t R = 1u << (d->ek - d->k);
  if (part >= R) return fail(ctx, SPB_ERR_ARG, "abi shim: coset part out of range");
  std::vector<fe> whole((size_t)1 << d->ek);
  for (size_t i = 0; i < count; i++) {
    orc_coeff_to_extended(d->d, (const fe*)d_in[i], whole.data(), kThreads);
    for (size_t m = 0; m < ((size_t)1 << d->k); m++) memcpy(&d_out[i][m], &whole[part + (size_t)R * m], 32);
  }
  return 0;
}
int spb_extended_part_scatter_dev(spb_ctx* ctx, const spb_domain* d, uint32_t part, const spb_fr* d_part, spb_fr* d_extended) {
  const uint32_t R = 1u << (d->ek - d->k);
  if (part >= R) return fail(ctx, SPB_ERR_ARG, "abi shim: coset part out of range");
  for (size_t m = 0; m < ((size_t)1 << d->k); m++) memcpy(&d_extended[part + (size_t)R * m], &d_part[m], 32);
  return 0;
}
// X = g * omega^idx through the oracle's routine, which reads X as zeta * w^idx: with w = omega, beta' = beta g / zeta and
// sigma' = sigma zeta / g every term is the same field element (beta' X = beta g omega^idx, beta' sigma' = beta sigma)
int spb_permutation_constraints_coset_dev(spb_ctx*, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets,
                                          uint32_t chunk_len, const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values,
                                          const spb_fr* const* d_sigma, const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active,
                                          const spb_fr* beta, const spb_fr* gamma, const spb_fr* y, const spb_fr* coset_generator, const spb_fr* omega) {
  fe root, zeta, one, zeta_inv, g_inv, beta2, ratio, delta;
  orc_fr_constants(&root, &zeta, &one);
  orc_fr_inv(&zeta_inv, &zeta); orc_fr_inv(&g_inv, (const fe*)coset_generator);
  orc_fr_mul(&beta2, (const fe*)beta, (const fe*)coset_generator); orc_fr_mul(&beta2, &beta2, &zeta_inv);
  orc_fr_mul(&ratio, &zeta, &g_inv);
  std::vector<std::vector<fe>> sigma2(n_cols);
  std::vector<const fe*> sp(n_cols);
  for (uint32_t c = 0; c < n_cols; c++) {
    sigma2[c].assign((const fe*)d_sigma[c], (const fe*)d_sigma[c] + size);
    orc_vec_scale(sigma2[c].data(), &ratio, size);
    sp[c] = sigma2[c].data();
  }
  orc_fr_delta(&delta);
  orc_permutation_constraints((fe*)d_values, size, rot_scale, last_rotation, n_sets, chunk_len, (const fe* const*)d_z, n_cols, (const fe* const*)d_col_values,
                              sp.data(), (const fe*)d_l0, (const fe*)d_l_last, (const fe*)d_l_active, &beta2, (const fe*)gamma, (const fe*)y, &delta,
                              (const fe*)omega);
  return 0;
}
}
