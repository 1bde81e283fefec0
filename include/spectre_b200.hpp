// spectre_b200.hpp -- C++17 host-side mirror of the halo2_proofs surface on Spectre's create_proof hot path, over the
// C ABI in spectre_b200.h. The reference is compiled Rust and the image has no cargo, so this header (and the Rust
// `extern "C"` block in INTEGRATION.md) is the compiled-language host side: same item names, argument meaning and
// failure behaviour as the upstream Rust ([UPSTREAM] halo2_proofs/src/{arithmetic.rs, poly/domain.rs,
// poly/kzg/commitment.rs}; reached from lightclient-circuits/src/util/circuit.rs:131,158,177,211,263):
//
//   halo2::arithmetic::best_multiexp(coeffs, bases) -> G1      (panics -> std::invalid_argument on length mismatch)
//   halo2::arithmetic::best_fft(a, omega, log_n)               (in place; a.size() must be 1 << log_n)
//   halo2::poly::EvaluationDomain(j, k)                        lagrange_to_coeff / coeff_to_extended / ...
//   halo2::poly::kzg::ParamsKZG                                from_parts / setup / read_custom / commit / commit_lagrange
//
// Header-only; link with -lspectre_b200. There is no CPU fallback: Backend() throws when spb_init fails.
#pragma once
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "spectre_b200.h"

namespace halo2 {

using Fr = spb_fr;
using G1Affine = spb_g1_affine;
using G1 = spb_g1;

class Backend {
 public:
  explicit Backend(const std::vector<int>& devices = {0}) {
    ctx_ = spb_init(devices.data(), (int)devices.size());
    if (!ctx_) throw std::runtime_error("spectre_b200: spb_init failed (no CUDA device; the library has no CPU fallback)");
  }
  ~Backend() { spb_shutdown(ctx_); }
  Backend(const Backend&) = delete;
  Backend& operator=(const Backend&) = delete;
  spb_ctx* ctx() const { return ctx_; }
  void check(int rc, const char* what) const {
    if (rc != 0) throw std::runtime_error(std::string(what) + " failed: " + spb_last_error(ctx_));
  }

 private:
  spb_ctx* ctx_;
};

namespace arithmetic {

inline G1 best_multiexp(const Backend& be, const std::vector<Fr>& coeffs, const std::vector<G1Affine>& bases) {
  if (coeffs.size() != bases.size()) throw std::invalid_argument("best_multiexp: coeffs.len() != bases.len()");
  G1 out;
  be.check(spb_msm_raw(be.ctx(), coeffs.data(), bases.data(), coeffs.size(), &out), "spb_msm_raw");
  return out;
}

inline void best_fft(const Backend& be, std::vector<Fr>& a, const Fr& omega, uint32_t log_n) {
  if (a.size() != ((size_t)1 << log_n)) throw std::invalid_argument("best_fft: a.len() != 1 << log_n");
  be.check(spb_ntt(be.ctx(), a.data(), log_n, &omega), "spb_ntt");
}

inline Fr eval_polynomial(const Backend& be, const std::vector<Fr>& poly, const Fr& point) {
  Fr out;
  be.check(spb_eval_polynomial(be.ctx(), poly.data(), poly.size(), &point, &out), "spb_eval_polynomial");
  return out;
}

inline std::vector<Fr> kate_division(const Backend& be, const std::vector<Fr>& a, const Fr& b) {
  std::vector<Fr> q(a.size() - 1);
  be.check(spb_kate_division(be.ctx(), a.data(), a.size(), &b, q.data()), "spb_kate_division");
  return q;
}

inline void batch_invert(const Backend& be, std::vector<Fr>& a) { be.check(spb_batch_invert(be.ctx(), a.data(), a.size()), "spb_batch_invert"); }

}  // namespace arithmetic

namespace poly {

class EvaluationDomain {
 public:
  EvaluationDomain(const Backend& be, uint32_t j, uint32_t k) : be_(be), j_(j), k_(k) {
    be.check(spb_domain_new(be.ctx(), j, k, &d_), "spb_domain_new");
    extended_k_ = spb_domain_extended_k(d_);
    Fr c[8];
    spb_domain_constants(d_, c);
    omega_ = c[0]; omega_inv_ = c[1]; extended_omega_ = c[2]; extended_omega_inv_ = c[3];
  }
  ~EvaluationDomain() { spb_domain_free(be_.ctx(), d_); }
  EvaluationDomain(const EvaluationDomain&) = delete;
  uint32_t k() const { return k_; }
  uint32_t extended_k() const { return extended_k_; }
  size_t extended_len() const { return (size_t)1 << extended_k_; }
  const Fr& get_omega() const { return omega_; }
  const Fr& get_omega_inv() const { return omega_inv_; }
  const Fr& get_extended_omega() const { return extended_omega_; }

  void lagrange_to_coeff(std::vector<Fr>& a) const { need(a.size(), (size_t)1 << k_); be_.check(spb_lagrange_to_coeff(be_.ctx(), d_, a.data()), "spb_lagrange_to_coeff"); }
  void coeff_to_lagrange(std::vector<Fr>& a) const { need(a.size(), (size_t)1 << k_); be_.check(spb_coeff_to_lagrange(be_.ctx(), d_, a.data()), "spb_coeff_to_lagrange"); }
  std::vector<Fr> coeff_to_extended(const std::vector<Fr>& a) const {
    need(a.size(), (size_t)1 << k_);
    std::vector<Fr> out(extended_len());
    be_.check(spb_coeff_to_extended(be_.ctx(), d_, a.data(), out.data()), "spb_coeff_to_extended");
    return out;
  }
  std::vector<Fr> extended_to_coeff(const std::vector<Fr>& a) const {
    need(a.size(), extended_len());
    std::vector<Fr> out(((size_t)1 << k_) * (j_ - 1));
    be_.check(spb_extended_to_coeff(be_.ctx(), d_, a.data(), out.data()), "spb_extended_to_coeff");
    return out;
  }
  void divide_by_vanishing_poly(std::vector<Fr>& a) const { need(a.size(), extended_len()); be_.check(spb_divide_by_vanishing(be_.ctx(), d_, a.data()), "spb_divide_by_vanishing"); }

 private:
  static void need(size_t got, size_t want) { if (got != want) throw std::invalid_argument("EvaluationDomain: polynomial has the wrong length"); }
  const Backend& be_;
  spb_domain* d_ = nullptr;
  uint32_t j_, k_, extended_k_ = 0;
  Fr omega_, omega_inv_, extended_omega_, extended_omega_inv_;
};

namespace kzg {

class ParamsKZG {
 public:
  // what ParamsKZG::read yields: both bases, uploaded once
  static ParamsKZG from_parts(const Backend& be, uint32_t k, const std::vector<G1Affine>& g, const std::vector<G1Affine>& g_lagrange) {
    spb_srs* h = nullptr;
    be.check(spb_srs_upload(be.ctx(), k, g.empty() ? nullptr : g.data(), g_lagrange.empty() ? nullptr : g_lagrange.data(), &h), "spb_srs_upload");
    return ParamsKZG(be, k, h);
  }
  // ParamsKZG::setup(k, rng) with the secret the rng would draw
  static ParamsKZG setup(const Backend& be, uint32_t k, const Fr& s) {
    spb_srs* h = nullptr;
    be.check(spb_srs_setup(be.ctx(), k, &s, &h), "spb_srs_setup");
    return ParamsKZG(be, k, h);
  }
  // ParamsKZG::read_custom(reader, format) of a params file: format SPB_SERDE_RAW_BYTES (checked: canonical coordinates, every
  // point on its curve; throws naming the first invalid point) or SPB_SERDE_RAW_BYTES_UNCHECKED
  static ParamsKZG read_custom(const Backend& be, const std::string& path, int format) {
    spb_srs* h = nullptr;
    be.check(spb_srs_read_file_custom(be.ctx(), path.c_str(), format, &h), "spb_srs_read_file_custom");
    return ParamsKZG(be, spb_srs_k(h), h);
  }
  ParamsKZG(ParamsKZG&& o) noexcept : be_(o.be_), k_(o.k_), h_(o.h_) { o.h_ = nullptr; }
  ~ParamsKZG() { if (h_) spb_srs_free(be_.ctx(), h_); }
  uint32_t k() const { return k_; }
  uint64_t n() const { return 1ull << k_; }
  const spb_srs* handle() const { return h_; }
  void precompute() { be_.check(spb_srs_precompute(be_.ctx(), h_), "spb_srs_precompute"); }
  // Params::commit / commit_lagrange (the blind is ignored by the KZG scheme upstream, so it is not taken here)
  G1 commit(const std::vector<Fr>& poly) const { return msm(SPB_BASIS_G, poly); }
  G1 commit_lagrange(const std::vector<Fr>& poly) const { return msm(SPB_BASIS_G_LAGRANGE, poly); }
  std::vector<G1Affine> get_g(int basis = SPB_BASIS_G) const {
    std::vector<G1Affine> out(n());
    be_.check(spb_srs_download(be_.ctx(), h_, basis, 0, out.size(), out.data()), "spb_srs_download");
    return out;
  }

 private:
  ParamsKZG(const Backend& be, uint32_t k, spb_srs* h) : be_(be), k_(k), h_(h) {}
  G1 msm(int basis, const std::vector<Fr>& poly) const {
    if (poly.size() > n()) throw std::invalid_argument("commit: polynomial longer than the SRS");
    G1 out;
    be_.check(spb_msm(be_.ctx(), h_, basis, poly.data(), poly.size(), &out), "spb_msm");
    return out;
  }
  const Backend& be_;
  uint32_t k_;
  spb_srs* h_;
};

}  // namespace kzg

// ProverSHPLONK::create_proof over device-resident polynomials (coefficient form, n each). RotationSet mirrors what
// construct_intermediate_sets yields; open() returns the first commitment, finish(u) the second.
namespace shplonk {

struct RotationSet {
  std::vector<Fr> points;
  std::vector<const Fr*> d_polys;   // device pointers
  std::vector<Fr> evals;            // d_polys.size() x points.size()
};

class Prover {
 public:
  Prover(const Backend& be, const kzg::ParamsKZG& params, size_t n, const std::vector<RotationSet>& sets, const Fr& y, const Fr& v, G1* h_commitment) : be_(be) {
    std::vector<spb_rotation_set> raw;
    for (const RotationSet& rs : sets) {
      if (rs.evals.size() != rs.d_polys.size() * rs.points.size()) throw std::invalid_argument("shplonk: evals must be polys x points");
      raw.push_back(spb_rotation_set{rs.points.data(), (uint32_t)rs.points.size(), rs.d_polys.data(), (uint32_t)rs.d_polys.size(), rs.evals.data()});
    }
    be.check(spb_shplonk_begin_dev(be.ctx(), params.handle(), n, raw.data(), (uint32_t)raw.size(), &y, &v, h_commitment, &s_), "spb_shplonk_begin_dev");
  }
  ~Prover() { if (s_) spb_shplonk_abort(be_.ctx(), s_); }
  Prover(const Prover&) = delete;
  G1 finish(const Fr& u) {
    G1 out;
    spb_shplonk* s = s_;
    s_ = nullptr;                     // consumed by the call, also on error
    be_.check(spb_shplonk_finish_dev(be_.ctx(), s, &u, &out), "spb_shplonk_finish_dev");
    return out;
  }

 private:
  const Backend& be_;
  spb_shplonk* s_ = nullptr;
};

}  // namespace shplonk
}  // namespace poly

// plonk::{permutation,lookup}::prover grand products over device-resident Lagrange columns
namespace plonk {

inline Fr permutation_product(const Backend& be, uint32_t k, const std::vector<const Fr*>& d_values, const std::vector<const Fr*>& d_sigma, uint32_t first_col,
                              const Fr& beta, const Fr& gamma, const std::vector<Fr>& blinds, Fr last_z, Fr* d_z) {
  if (d_values.size() != d_sigma.size()) throw std::invalid_argument("permutation_product: one sigma per column");
  be.check(spb_permutation_product_dev(be.ctx(), k, d_values.data(), d_sigma.data(), (uint32_t)d_values.size(), first_col, &beta, &gamma,
                                       blinds.empty() ? nullptr : blinds.data(), (uint32_t)blinds.size(), &last_z, d_z), "spb_permutation_product_dev");
  return last_z;
}

inline void lookup_product(const Backend& be, size_t n, const Fr* d_compressed_input, const Fr* d_compressed_table, const Fr* d_permuted_input, const Fr* d_permuted_table,
                           const Fr& beta, const Fr& gamma, const std::vector<Fr>& blinds, Fr* d_z) {
  be.check(spb_lookup_product_dev(be.ctx(), n, d_compressed_input, d_compressed_table, d_permuted_input, d_permuted_table, &beta, &gamma,
                                  blinds.empty() ? nullptr : blinds.data(), (uint32_t)blinds.size(), d_z), "spb_lookup_product_dev");
}

}  // namespace plonk
}  // namespace halo2
