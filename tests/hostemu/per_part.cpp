// Host build of the device bodies a per-part proof adds (tests/test_plonk_per_part_keys.py): hostemu.cpp, included whole, plus
// the coset part transform (the NTT kernel's phases with the g^a power-table pre-scale), the coset form of the permutation row
// and the part scatter, each run serially on the CPU.
#include "hostemu.cpp"

extern "C" {
// One coset part: the n-point transform of in[a] * g^a, the pre-scale read from the two-level power table of g (split h of
// the plan, as the library builds it). Single-device plan; use_full: full twiddle table.
int he_ntt_part(const Fr* in, Fr* out, uint32_t k, const Fr* omega, const Fr* g, uint32_t max_digit, uint32_t tile_log, uint32_t threads, int use_full) {
  const uint64_t n = 1ull << k;
  NttPlan plan = ntt_make_plan(k, max_digit);
  const uint32_t h = k - plan.s[0];
  std::vector<Fr> tw_lo((size_t)1 << h), tw_hi((size_t)1 << (k - h)), tw_full, pre_lo(tw_lo.size()), pre_hi(tw_hi.size());
  for (size_t i = 0; i < tw_lo.size(); i++) { tw_lo[i] = fp_pow_u64(*omega, i); pre_lo[i] = fp_pow_u64(*g, i); }
  for (size_t i = 0; i < tw_hi.size(); i++) { tw_hi[i] = fp_pow_u64(*omega, (uint64_t)i << h); pre_hi[i] = fp_pow_u64(*g, (uint64_t)i << h); }
  if (use_full) { tw_full.resize(n); for (uint64_t i = 0; i < n; i++) tw_full[i] = fp_pow_u64(*omega, i); }
  NttOptsHost oh; oh.pre_lo = pre_lo.data(); oh.pre_hi = pre_hi.data();
  std::vector<Fr> buf(in, in + n), tmp(n);
  for (uint32_t pi = 0; pi < plan.npass; pi++) {
    NttPassParams p;
    p.src = pi == 0 ? buf.data() : tmp.data(); p.dst = pi == plan.npass - 1 ? out : tmp.data();
    p.tw_lo = tw_lo.data(); p.tw_hi = tw_hi.data(); p.tw_full = use_full ? tw_full.data() : nullptr;
    NttLaunch L = ntt_fill_pass(p, plan, pi, k, h, oh, NttShare(), tile_log, threads);
    run_pass(p, L);
  }
  return (int)plan.npass;
}
// the coset form: X = coset_generator * omega^idx (delta_start = beta * coset_generator, as the library's shared host function sets it)
void he_permutation_constraints_coset(Fr* values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len, const Fr* const* z,
                                      uint32_t n_cols, const Fr* const* col_values, const Fr* const* sigma, const Fr* l0, const Fr* l_last, const Fr* l_active,
                                      const Fr* beta, const Fr* gamma, const Fr* y, const Fr* coset_generator, const Fr* omega) {
  if (!n_sets) return;
  PermArgs a; memset(&a, 0, sizeof a);
  a.values = values; a.size = size; a.rot_scale = rot_scale; a.last_rotation = last_rotation; a.n_sets = n_sets; a.chunk_len = chunk_len; a.n_cols = n_cols;
  a.z = z; a.col_values = col_values; a.sigma = sigma; a.l0 = l0; a.l_last = l_last; a.l_active = l_active;
  a.beta = *beta; a.gamma = *gamma; a.y = *y; a.extended_omega = *omega;
  constexpr uint32_t delta[8] = SPB_FR_DELTA_MONT;
  a.delta = fr_macro(delta); a.delta_start = fp_mul(a.beta, *coset_generator);
  for (uint64_t idx = 0; idx < size; idx++) permutation_constraints_row(a, idx, fp_pow_u64(a.extended_omega, idx));
}
void he_extended_part_scatter(const Fr* part_values, Fr* extended, uint32_t part, uint32_t R, uint64_t n) {
  for (uint64_t m = 0; m < n; m++) extended_part_scatter_row(part_values, extended, part, R, m);
}
}
