// TEST INFRASTRUCTURE -- a CPU stand-in for the part of the C ABI (include/spectre_b200.h) that the proof drivers call,
// backed by the ORACLE (oracle/halo2_oracle.c). "Device pointers" are host pointers. It exists so that the HOST logic above
// the ABI (include/spectre_b200_prover.hpp; protocol order, transcript, RNG use, set bookkeeping, expression flattening) can
// be exercised in the `-m "not gpu"` suite without a GPU. It is never built into, linked with or loaded by the product:
// libspectre_b200.so has no CPU path and fails to initialise without a CUDA device. Commitments are computed with the
// known-tau shortcut of the seed-0 SRS, so spb_srs_setup only accepts that secret.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/spectre_b200.h"

extern "C" {
typedef struct { uint64_t l[4]; } fe;
typedef struct { fe x, y; } g1a;
typedef struct orc_domain orc_domain;
typedef struct { const fe* points; uint32_t n_points; const fe* const* polys; uint32_t n_polys; const fe* evals; } orc_rotation_set;
void orc_init(void);
void orc_chacha20_block(const uint8_t key[32], uint64_t counter, uint8_t out[64]);
void orc_fr_from_u512(fe* o, const uint8_t in[64]);
void orc_g1_generator(g1a* o);
void orc_srs_tau(fe* tau);
void orc_fr_delta(fe* out);
void orc_best_fft(fe* a, const fe* omega, uint32_t log_n, int threads);
orc_domain* orc_domain_new(uint32_t j, uint32_t k);
void orc_domain_free(orc_domain* d);
void orc_domain_describe(const orc_domain* d, uint32_t* extended_k, fe* omega, fe* extended_omega, fe* consts6, fe* t_eval);
void orc_lagrange_to_coeff(const orc_domain* d, fe* a, int threads);
void orc_coeff_to_extended(const orc_domain* d, const fe* in, fe* out, int threads);
void orc_extended_to_coeff(const orc_domain* d, fe* in, fe* out, int threads);
void orc_divide_by_vanishing_poly(const orc_domain* d, fe* a);
void orc_eval_polynomial(fe* out, const fe* poly, size_t n, const fe* point);
void orc_commit_known_tau(const fe* coeffs, size_t n, g1a* out);
void orc_commit_lagrange_known_tau(uint32_t k, const fe* evals, size_t n_used, g1a* out);
void orc_graph_evaluate(const uint32_t* prog, uint32_t ncalc, uint32_t n_inter, const fe* constants, const int32_t* rotations, uint32_t nrot, const fe* const* fixed,
                        const fe* const* advice, const fe* const* instance, const fe* challenges, const fe* bgty, fe* values, uint64_t size, int32_t rot_scale);
void orc_permutation_constraints(fe* values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len, const fe* const* z,
                                 uint32_t n_cols, const fe* const* col_values, const fe* const* sigma, const fe* l0, const fe* l_last, const fe* l_active,
                                 const fe* beta, const fe* gamma, const fe* y, const fe* delta, const fe* extended_omega);
void orc_lookup_constraints(fe* values, uint64_t size, int32_t rot_scale, const fe* product, const fe* permuted_input, const fe* permuted_table,
                            const fe* table_value, const fe* l0, const fe* l_last, const fe* l_active, const fe* beta, const fe* gamma, const fe* y);
int orc_permute_expression_pair(const fe* input, const fe* table, size_t usable, fe* permuted_input, fe* permuted_table);
void orc_permutation_product(uint32_t k, const fe* const* values, const fe* const* sigma, uint32_t n_cols, uint32_t first_col, const fe* beta, const fe* gamma,
                             const fe* blinds, uint32_t n_blinds, fe* last_z, fe* z);
void orc_lookup_product(size_t n, const fe* compressed_input, const fe* compressed_table, const fe* permuted_input, const fe* permuted_table, const fe* beta,
                        const fe* gamma, const fe* blinds, uint32_t n_blinds, fe* z);
void orc_shplonk_quotient(size_t n, const orc_rotation_set* sets, uint32_t n_sets, const fe* y, const fe* v, fe* h_x);
int orc_shplonk_linearisation(size_t n, const orc_rotation_set* sets, uint32_t n_sets, const fe* y, const fe* v, const fe* u, const fe* h_x, fe* out);
void orc_vec_scale(fe* a, const fe* alpha, size_t n);
void orc_vec_fold(const fe* const* polys, size_t count, const fe* y, fe* out, size_t n);
}

struct spb_ctx { std::string last_error; };
struct spb_srs { uint32_t k; };
struct spb_domain { orc_domain* d; uint32_t j, k, ek; fe c[8]; };
struct spb_shplonk {
  size_t n; const spb_srs* srs; fe y, v;
  std::vector<std::vector<fe>> points, evals;
  std::vector<std::vector<const fe*>> polys;
  std::vector<fe> h_x;
  std::vector<orc_rotation_set> sets() const {
    std::vector<orc_rotation_set> out;
    for (size_t i = 0; i < points.size(); i++) out.push_back({points[i].data(), (uint32_t)points[i].size(), polys[i].data(), (uint32_t)polys[i].size(), evals[i].data()});
    return out;
  }
};

static const int kThreads = 4;
static int g_open_shplonk = 0;                        // spb_shplonk handles begun and not yet finished or aborted
static int fail(spb_ctx* ctx, int code, const char* msg) { if (ctx) ctx->last_error = msg; return code; }
static void to_jac(const g1a& a, spb_g1* out) {
  g1a gen; orc_g1_generator(&gen);                       // generator x = 1 in Montgomery form = the Fq "one"
  memcpy(&out->x, &a.x, 32); memcpy(&out->y, &a.y, 32);
  bool ident = true;
  for (int i = 0; i < 4; i++) if (a.x.l[i] | a.y.l[i]) ident = false;
  if (ident) memset(&out->z, 0, 32); else memcpy(&out->z, &gen.x, 32);
}

extern "C" {
spb_ctx* spb_init(const int*, int) { orc_init(); return new spb_ctx(); }
void spb_shutdown(spb_ctx* ctx) { delete ctx; }
const char* spb_last_error(spb_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "no context"; }

int spb_srs_setup(spb_ctx* ctx, uint32_t k, const spb_fr* s, spb_srs** out) {
  fe tau; orc_srs_tau(&tau);
  if (memcmp(&tau, s, 32) != 0) return fail(ctx, SPB_ERR_ARG, "abi shim: only the seed-0 SRS secret is supported (known-tau commitments)");
  *out = new spb_srs{k};
  return 0;
}
void spb_srs_free(spb_ctx*, spb_srs* srs) { delete srs; }
uint32_t spb_srs_k(const spb_srs* srs) { return srs->k; }
int spb_msm_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* d_scalars, size_t n, spb_g1* out) {
  if (n > ((size_t)1 << srs->k)) return fail(ctx, SPB_ERR_ARG, "abi shim: more scalars than the SRS has points");
  g1a a;
  if (basis == SPB_BASIS_G) orc_commit_known_tau((const fe*)d_scalars, n, &a); else orc_commit_lagrange_known_tau(srs->k, (const fe*)d_scalars, n, &a);
  to_jac(a, out);
  return 0;
}
int spb_msm_batch_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* d_scalars, size_t n, size_t count, spb_g1* out) {
  for (size_t i = 0; i < count; i++) { int rc = spb_msm_dev(ctx, srs, basis, d_scalars[i], n, out + i); if (rc) return rc; }
  return 0;
}

int spb_domain_new(spb_ctx*, uint32_t j, uint32_t k, spb_domain** out) {
  spb_domain* d = new spb_domain();
  d->d = orc_domain_new(j, k); d->j = j; d->k = k;
  fe consts6[6];
  orc_domain_describe(d->d, &d->ek, &d->c[0], &d->c[2], consts6, nullptr);
  d->c[1] = consts6[0]; d->c[3] = consts6[1]; d->c[4] = consts6[2]; d->c[5] = consts6[3]; d->c[6] = consts6[4]; d->c[7] = consts6[5];
  *out = d;
  return 0;
}
void spb_domain_free(spb_ctx*, spb_domain* d) { if (d) { orc_domain_free(d->d); delete d; } }
uint32_t spb_domain_extended_k(const spb_domain* d) { return d->ek; }
void spb_domain_constants(const spb_domain* d, spb_fr out[8]) { memcpy(out, d->c, sizeof d->c); }
int spb_lagrange_to_coeff_dev(spb_ctx*, const spb_domain* d, spb_fr* a) { orc_lagrange_to_coeff(d->d, (fe*)a, kThreads); return 0; }
int spb_coeff_to_extended_dev(spb_ctx*, const spb_domain* d, const spb_fr* in, spb_fr* out) { orc_coeff_to_extended(d->d, (const fe*)in, (fe*)out, kThreads); return 0; }
int spb_extended_to_coeff_dev(spb_ctx*, const spb_domain* d, const spb_fr* in, spb_fr* out) {
  std::vector<fe> tmp((size_t)1 << d->ek);
  memcpy(tmp.data(), in, tmp.size() * 32);
  orc_extended_to_coeff(d->d, tmp.data(), (fe*)out, kThreads);
  return 0;
}
int spb_divide_by_vanishing_dev(spb_ctx*, const spb_domain* d, spb_fr* a) { orc_divide_by_vanishing_poly(d->d, (fe*)a); return 0; }
int spb_ntt_dev(spb_ctx*, spb_fr* a, uint32_t log_n, const spb_fr* omega) { orc_best_fft((fe*)a, (const fe*)omega, log_n, kThreads); return 0; }

int spb_graph_evaluate_dev(spb_ctx*, const spb_graph* g, const spb_fr* const* d_fixed, uint32_t, const spb_fr* const* d_advice, uint32_t,
                           const spb_fr* const* d_instance, uint32_t, const spb_fr* challenges, uint32_t, const spb_fr* beta, const spb_fr* gamma,
                           const spb_fr* theta, const spb_fr* y, spb_fr* d_values, uint64_t size, int32_t rot_scale) {
  fe bgty[4]; memcpy(&bgty[0], beta, 32); memcpy(&bgty[1], gamma, 32); memcpy(&bgty[2], theta, 32); memcpy(&bgty[3], y, 32);
  orc_graph_evaluate(g->program, g->num_calculations, g->num_intermediates, (const fe*)g->constants, g->rotations, g->num_rotations, (const fe* const*)d_fixed,
                     (const fe* const*)d_advice, (const fe* const*)d_instance, (const fe*)challenges, bgty, (fe*)d_values, size, rot_scale);
  return 0;
}
int spb_permutation_constraints_dev(spb_ctx*, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len,
                                    const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values, const spb_fr* const* d_sigma, const spb_fr* d_l0,
                                    const spb_fr* d_l_last, const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma, const spb_fr* y,
                                    const spb_fr* extended_omega) {
  fe delta; orc_fr_delta(&delta);
  orc_permutation_constraints((fe*)d_values, size, rot_scale, last_rotation, n_sets, chunk_len, (const fe* const*)d_z, n_cols, (const fe* const*)d_col_values,
                              (const fe* const*)d_sigma, (const fe*)d_l0, (const fe*)d_l_last, (const fe*)d_l_active, (const fe*)beta, (const fe*)gamma, (const fe*)y,
                              &delta, (const fe*)extended_omega);
  return 0;
}
int spb_lookup_constraints_dev(spb_ctx*, spb_fr* d_values, uint64_t size, int32_t rot_scale, const spb_fr* d_product, const spb_fr* d_permuted_input,
                               const spb_fr* d_permuted_table, const spb_fr* d_table_value, const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active,
                               const spb_fr* beta, const spb_fr* gamma, const spb_fr* y) {
  orc_lookup_constraints((fe*)d_values, size, rot_scale, (const fe*)d_product, (const fe*)d_permuted_input, (const fe*)d_permuted_table, (const fe*)d_table_value,
                         (const fe*)d_l0, (const fe*)d_l_last, (const fe*)d_l_active, (const fe*)beta, (const fe*)gamma, (const fe*)y);
  return 0;
}
int spb_permute_expression_pair_dev(spb_ctx* ctx, const spb_fr* d_input, const spb_fr* d_table, size_t usable, spb_fr* d_pi, spb_fr* d_pt) {
  if (orc_permute_expression_pair((const fe*)d_input, (const fe*)d_table, usable, (fe*)d_pi, (fe*)d_pt) != 0)
    return fail(ctx, SPB_ERR_CONSTRAINT, "permute_expression_pair: ConstraintSystemFailure (an input value does not occur in the table)");
  return 0;
}
int spb_permutation_product_dev(spb_ctx*, uint32_t k, const spb_fr* const* d_values, const spb_fr* const* d_sigma, uint32_t n_cols, uint32_t first_col,
                                const spb_fr* beta, const spb_fr* gamma, const spb_fr* blinds, uint32_t n_blinds, spb_fr* last_z, spb_fr* d_z) {
  orc_permutation_product(k, (const fe* const*)d_values, (const fe* const*)d_sigma, n_cols, first_col, (const fe*)beta, (const fe*)gamma, (const fe*)blinds, n_blinds,
                          (fe*)last_z, (fe*)d_z);
  return 0;
}
int spb_lookup_product_dev(spb_ctx*, size_t n, const spb_fr* ci, const spb_fr* ct, const spb_fr* pi, const spb_fr* pt, const spb_fr* beta, const spb_fr* gamma,
                           const spb_fr* blinds, uint32_t n_blinds, spb_fr* d_z) {
  orc_lookup_product(n, (const fe*)ci, (const fe*)ct, (const fe*)pi, (const fe*)pt, (const fe*)beta, (const fe*)gamma, (const fe*)blinds, n_blinds, (fe*)d_z);
  return 0;
}
int spb_eval_polynomial_dev(spb_ctx*, const spb_fr* d_poly, size_t n, const spb_fr* point, spb_fr* out) { orc_eval_polynomial((fe*)out, (const fe*)d_poly, n, (const fe*)point); return 0; }
int spb_lincomb_dev(spb_ctx*, const spb_fr* const* d_polys, size_t count, const spb_fr* y, spb_fr* d_out, size_t n) { orc_vec_fold((const fe* const*)d_polys, count, (const fe*)y, (fe*)d_out, n); return 0; }
int spb_fr_random_chacha_dev(spb_ctx*, const uint8_t seed[32], uint64_t first, spb_fr* d_out, size_t n) {
  for (size_t i = 0; i < n; i++) { uint8_t blk[64]; orc_chacha20_block(seed, first + i, blk); orc_fr_from_u512((fe*)d_out + i, blk); }
  return 0;
}
int spb_vec_scale_dev(spb_ctx*, spb_fr* d_a, const spb_fr* alpha, size_t n) { orc_vec_scale((fe*)d_a, (const fe*)alpha, n); return 0; }

int spb_shplonk_begin_dev(spb_ctx* ctx, const spb_srs* srs, size_t n, const spb_rotation_set* sets, uint32_t n_sets, const spb_fr* y, const spb_fr* v,
                          spb_g1* h_commitment, spb_shplonk** out) {
  spb_shplonk* s = new spb_shplonk();
  s->n = n; s->srs = srs; memcpy(&s->y, y, 32); memcpy(&s->v, v, 32);
  for (uint32_t i = 0; i < n_sets; i++) {
    const spb_rotation_set& rs = sets[i];
    s->points.emplace_back((const fe*)rs.points, (const fe*)rs.points + rs.n_points);
    s->evals.emplace_back((const fe*)rs.evals, (const fe*)rs.evals + (size_t)rs.n_points * rs.n_polys);
    s->polys.emplace_back((const fe* const*)rs.d_polys, (const fe* const*)rs.d_polys + rs.n_polys);
  }
  s->h_x.resize(n);
  auto os = s->sets();
  orc_shplonk_quotient(n, os.data(), n_sets, &s->y, &s->v, s->h_x.data());
  int rc = spb_msm_dev(ctx, srs, SPB_BASIS_G, (const spb_fr*)s->h_x.data(), n, h_commitment);
  if (rc) { delete s; return rc; }
  g_open_shplonk++;
  *out = s;
  return 0;
}
int spb_shplonk_finish_dev(spb_ctx* ctx, spb_shplonk* s, const spb_fr* u, spb_g1* commitment) {
  // the header's contract: the handle is consumed on every return, a null argument included
  if (!s || !u || !commitment) { spb_shplonk_abort(ctx, s); return fail(ctx, SPB_ERR_ARG, "spb_shplonk_finish_dev: null argument"); }
  std::vector<fe> fin(s->n - 1);
  auto os = s->sets();
  int rc = orc_shplonk_linearisation(s->n, os.data(), (uint32_t)os.size(), &s->y, &s->v, (const fe*)u, s->h_x.data(), fin.data());
  if (rc == 0) rc = spb_msm_dev(ctx, s->srs, SPB_BASIS_G, (const spb_fr*)fin.data(), s->n - 1, commitment);
  else rc = fail(ctx, SPB_ERR_ARG, "abi shim: evaluations inconsistent with the polynomials");
  spb_shplonk_abort(ctx, s);
  return rc;
}
void spb_shplonk_abort(spb_ctx*, spb_shplonk* s) {
  if (!s) return;
  g_open_shplonk--;
  delete s;
}
// test hook of the shim alone: the number of spb_shplonk handles begun and not yet consumed
int spb_shim_open_shplonk_handles(void) { return g_open_shplonk; }
}
