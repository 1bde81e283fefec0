// Argument provers of halo2's create_proof on the device: the permutation grand product, the lookup grand product and
// the SHPLONK multi-open prover (SURVEY.md 8a rows a8, a9; 8f row 1 "device-resident proving pipeline").
//
//   [UPSTREAM] halo2_proofs/src/plonk/permutation/prover.rs   Argument::commit          -> spb_permutation_product_dev
//   [UPSTREAM] halo2_proofs/src/plonk/lookup/prover.rs        Permuted::commit_product  -> spb_lookup_product_dev
//   [UPSTREAM] halo2_proofs/src/poly/kzg/multiopen/shplonk/prover.rs ProverSHPLONK::create_proof
//                                                                                      -> spb_shplonk_begin_dev / _finish_dev
//
// Every polynomial stays in HBM; what crosses the ABI per call is challenges, blinding values and 96-byte commitments.
// All passes are HBM-streaming: algorithmic bytes per row = 32 B x (columns read + 1 written).
#include "common.cuh"
#include "quotient.cuh"
#include <string.h>

using namespace spb;

// omega^i = omega^(256 * block) * omega^thread: one long power per block (thread 0), an 8-bit power per thread; the row
// bodies are perm_terms_row / lookup_terms_row in quotient.cuh.
// rows [row_lo, row_hi) of the column (row_lo a multiple of 256); num / den receive them at local index row - row_lo
__global__ void __launch_bounds__(256) perm_terms_kernel(PermTermArgs a, uint64_t row_lo, uint64_t row_hi, Fr* num, Fr* den) {
  __shared__ Fr block_base;
  const uint64_t block_row = row_lo + blockIdx.x * (uint64_t)blockDim.x;
  if (threadIdx.x == 0) block_base = fp_pow_u64(a.omega, block_row);
  __syncthreads();
  uint64_t i = block_row + threadIdx.x;
  if (i < row_hi) perm_terms_row(a, i, fp_mul(block_base, fp_pow_u64(a.omega, threadIdx.x)), num - row_lo, den - row_lo);
}
__global__ void __launch_bounds__(256) lookup_terms_kernel(const Fr* ci, const Fr* ct, const Fr* pi, const Fr* pt, Fr beta, Fr gamma, uint64_t n, Fr* num, Fr* den) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) lookup_terms_row(ci, ct, pi, pt, beta, gamma, i, num, den);
}
__global__ void __launch_bounds__(256) frac_mul_kernel(Fr* num, const Fr* den_inv, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(num + i, fp_mul(ntt_ld_stream(num + i), ntt_ld_stream(den_inv + i)));
}
// out[i] = sum_p w[p] * polys[p][i]
__global__ void __launch_bounds__(256) weighted_sum_kernel(const Fr* const* polys, const Fr* w, uint32_t count, Fr* out, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr acc = fp_zero<FrParams>();
  for (uint32_t p = 0; p < count; p++) acc = fp_add(acc, fp_mul(w[p], ntt_ld_stream(polys[p] + i)));
  ntt_stg(out + i, acc);
}
// h[i] = alpha * h[i] + beta * (i < nx ? x[i] : 0)
__global__ void __launch_bounds__(256) scale_add_kernel(Fr* h, Fr alpha, const Fr* x, Fr beta, uint64_t nx, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr v = fp_mul(alpha, ntt_ld_stream(h + i));
  if (i < nx) v = fp_add(v, fp_mul(beta, ntt_ld_stream(x + i)));
  ntt_stg(h + i, v);
}
struct SmallPoly { Fr c[8]; uint32_t n; };
__global__ void sub_small_kernel(Fr* a, SmallPoly s) {
  uint32_t i = threadIdx.x;
  if (i < s.n) a[i] = fp_sub(a[i], s.c[i]);
}

namespace {

// z[0] = init, z[i+1] = z[i] * num[i] / den[i] over the n rows of one column, then the last n_blinds entries <- blinds and
// *tail_out <- z[n - n_blinds - 1] (synchronises). `terms(d, lo, cnt, num, den)` launches on d.stream the kernel that writes the
// cnt numerators / denominators of rows lo.. into the device-local buffers, and returns its status.
// One device: terms, chunked batch inversion, product pass, chunked scan. Several devices (row ranges): every device does the
// same on its range in its own HBM, reading the column inputs from the first device over NVLink; the 32-byte range totals are the
// ONE exchange (through the host: G - 1 field products give every range its seed); the seeded scans then write their slice of z
// straight into the caller's buffer on the first device. Bit-identical to the one-device scan (exact field arithmetic).
template <class Terms>
int fraction_product(spb_ctx* ctx, size_t n, const Terms& terms, const Fr& init, const spb_fr* blinds, uint32_t n_blinds, Fr* dz, Fr* tail_out) {
  DeviceState& d0 = ctx->dev[0];
  const std::vector<RowRange> ranges = row_ranges(ctx, n);
  const size_t G = ranges.size();
  std::vector<Fr*> nums(G, nullptr), dtot(G, nullptr);
  if (G > 1) { SPB_CUDA(ctx, cudaSetDevice(d0.device)); SPB_CUDA(ctx, cudaEventRecord(d0.dep_ev, d0.stream)); }   // the caller's inputs are ordered on d0.stream
  for (size_t r = 0; r < G; r++) {
    DeviceState& d = ctx->dev[ranges[r].dev_index];
    const size_t cnt = ranges[r].hi - ranges[r].lo;
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    if (ranges[r].dev_index != 0) SPB_CUDA(ctx, cudaStreamWaitEvent(d.stream, d0.dep_ev, 0));
    Fr* num = (Fr*)slot(ctx, d, "plonk_num", cnt * 32); Fr* den = (Fr*)slot(ctx, d, "plonk_den", cnt * 32);
    if (!num || !den) return SPB_ERR_OOM;
    nums[r] = num;
    SPB_TRY(terms(d, ranges[r].lo, cnt, num, den));
    SPB_TRY(dev_batch_invert(ctx, d, den, cnt));
    SPB_TRY(launch(ctx, d.stream, nblk(cnt, 256), 256, 0, frac_mul_kernel, num, den, cnt));
    if (G > 1) SPB_TRY(dev_product_enqueue(ctx, d, num, cnt, &dtot[r]));
  }
  // seeds: seed_0 = init, seed_r = seed_{r-1} * total_{r-1}
  std::vector<Fr> seed(G, init);
  if (G > 1) {
    std::vector<Fr> total(G);
    for (size_t r = 0; r < G; r++) {
      DeviceState& d = ctx->dev[ranges[r].dev_index];
      SPB_CUDA(ctx, cudaSetDevice(d.device));
      SPB_CUDA(ctx, cudaMemcpyAsync(&total[r], dtot[r], 32, cudaMemcpyDeviceToHost, d.stream));
      SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
    }
    for (size_t r = 1; r < G; r++) seed[r] = fp_mul(seed[r - 1], total[r - 1]);
  }
  for (size_t r = 0; r < G; r++) {
    DeviceState& d = ctx->dev[ranges[r].dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_TRY(dev_grand_product(ctx, d, nums[r], ranges[r].hi - ranges[r].lo, dz + ranges[r].lo, seed[r]));   // peer store into the first device's z
    if (ranges[r].dev_index != 0) { SPB_CUDA(ctx, cudaEventRecord(d.dep_ev, d.stream)); }
  }
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  for (size_t r = 0; r < G; r++) if (ranges[r].dev_index != 0) SPB_CUDA(ctx, cudaStreamWaitEvent(d0.stream, ctx->dev[ranges[r].dev_index].dep_ev, 0));
  if (n_blinds) SPB_CUDA(ctx, cudaMemcpyAsync(dz + (n - n_blinds), blinds, (size_t)n_blinds * 32, cudaMemcpyHostToDevice, d0.stream));
  if (tail_out) SPB_CUDA(ctx, cudaMemcpyAsync(tail_out, dz + (n - n_blinds - 1), 32, cudaMemcpyDeviceToHost, d0.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d0.stream));
  return 0;
}

}  // namespace

// ---- SHPLONK state kept between the two transcript round trips ------------------------------------------------------
struct spb_shplonk {
  spb_ctx* ctx = nullptr;
  bool from_slots = false;      // buffers are the context's grow-only workspace slots (one open handle at a time), else cudaMalloc'd
  int device = 0;
  size_t n = 0;
  const spb_srs* srs = nullptr;
  Fr* d_h = nullptr;            // h(X) = sum_i v^i Q_i(X), n coefficients
  Fr* d_tmp[2] = {nullptr, nullptr};
  const Fr** d_ptrs = nullptr;  // all opened polynomials, set by set
  Fr* d_w = nullptr;            // their weights
  uint32_t n_polys = 0;
  Fr y, v;
  struct Set {
    std::vector<Fr> points;
    uint32_t n_polys = 0;
    std::vector<Fr> evals;                 // n_polys x n_points
    std::vector<std::vector<Fr>> r;        // low-degree equivalents R_ij, n_points coefficients each
  };
  std::vector<Set> sets;
  std::vector<Fr> super_points;
};

namespace {

// coefficients of the unique polynomial of degree < m through (points[p], evals[p]); m <= 8
void lagrange_interpolate(const std::vector<Fr>& points, const Fr* evals, Fr* out) {
  const size_t m = points.size();
  for (size_t i = 0; i < m; i++) out[i] = fp_zero<FrParams>();
  for (size_t j = 0; j < m; j++) {
    Fr num[9]; size_t deg = 0; num[0] = fp_one<FrParams>();       // prod_{k != j} (X - x_k)
    Fr denom = fp_one<FrParams>();
    for (size_t k2 = 0; k2 < m; k2++) {
      if (k2 == j) continue;
      num[deg + 1] = fp_zero<FrParams>();
      for (size_t t = deg + 2; t-- > 0;) {   // num <- num * (X - x_k), from the top coefficient down
        Fr lower = t ? num[t - 1] : fp_zero<FrParams>();
        num[t] = fp_sub(lower, fp_mul(points[k2], num[t]));
      }
      deg++;
      denom = fp_mul(denom, fp_sub(points[j], points[k2]));
    }
    Fr scale = fp_mul(evals[j], fp_inv(denom));
    for (size_t t = 0; t <= deg; t++) out[t] = fp_add(out[t], fp_mul(scale, num[t]));
  }
}
Fr eval_small(const Fr* c, size_t m, const Fr& x) {
  Fr acc = fp_zero<FrParams>();
  for (size_t t = m; t-- > 0;) acc = fp_add(fp_mul(acc, x), c[t]);
  return acc;
}
Fr vanishing_eval(const std::vector<Fr>& roots, const Fr& x) {
  Fr acc = fp_one<FrParams>();
  for (const Fr& r : roots) acc = fp_mul(acc, fp_sub(x, r));
  return acc;
}
bool contains(const std::vector<Fr>& v, const Fr& x) {
  for (const Fr& e : v) if (fp_eq(e, x)) return true;
  return false;
}
// call with the context lock held
void shplonk_release(spb_shplonk* s) {
  if (!s) return;
  if (s->from_slots) {
    s->ctx->shplonk_slots_busy = false;
  } else {
    cudaSetDevice(s->device);
    cudaFree(s->d_h); cudaFree(s->d_tmp[0]); cudaFree(s->d_tmp[1]); cudaFree((void*)s->d_ptrs); cudaFree(s->d_w);
  }
  delete s;
}

}  // namespace

extern "C" {

int spb_permutation_product_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_values, const spb_fr* const* d_sigma, uint32_t n_cols, uint32_t first_col,
                                const spb_fr* beta, const spb_fr* gamma, const spb_fr* blinds, uint32_t n_blinds, spb_fr* last_z, spb_fr* d_z) {
  if (!ctx) return SPB_ERR_ARG;
  if (!d_values || !d_sigma || !beta || !gamma || !last_z || !d_z || (n_blinds && !blinds)) return set_error(ctx, SPB_ERR_ARG, "spb_permutation_product_dev: null argument");
  if (k > SPB_FR_S || n_cols == 0 || n_cols > kMaxSetCols) return set_error(ctx, SPB_ERR_ARG, "spb_permutation_product_dev: 1..%u columns per set, k <= %d", kMaxSetCols, SPB_FR_S);
  const size_t n = (size_t)1 << k;
  if ((size_t)n_blinds + 1 > n) return set_error(ctx, SPB_ERR_ARG, "spb_permutation_product_dev: more blinding rows than rows");
  SPB_ENTER(ctx);
  PermTermArgs a;
  for (uint32_t c = 0; c < n_cols; c++) { a.values[c] = (const Fr*)d_values[c]; a.sigma[c] = (const Fr*)d_sigma[c]; }
  a.n_cols = n_cols; a.beta = fr_load(beta); a.gamma = fr_load(gamma); a.delta = fr_delta(); a.omega = fr_root_of_unity(k);
  a.delta_start = fp_mul(a.beta, fp_pow_u64(a.delta, first_col));
  Fr tail;
  auto terms = [&](DeviceState& dv, size_t lo, size_t cnt, Fr* num, Fr* den) {
    return launch(ctx, dv.stream, nblk(cnt, 256), 256, 0, perm_terms_kernel, a, lo, lo + cnt, num, den);
  };
  SPB_TRY(fraction_product(ctx, n, terms, fr_load(last_z), blinds, n_blinds, (Fr*)d_z, &tail));
  memcpy(last_z, &tail, 32);
  return 0;
}

int spb_lookup_product_dev(spb_ctx* ctx, size_t n, const spb_fr* d_compressed_input, const spb_fr* d_compressed_table, const spb_fr* d_permuted_input,
                           const spb_fr* d_permuted_table, const spb_fr* beta, const spb_fr* gamma, const spb_fr* blinds, uint32_t n_blinds, spb_fr* d_z) {
  if (!ctx) return SPB_ERR_ARG;
  if (!d_compressed_input || !d_compressed_table || !d_permuted_input || !d_permuted_table || !beta || !gamma || !d_z || (n_blinds && !blinds))
    return set_error(ctx, SPB_ERR_ARG, "spb_lookup_product_dev: null argument");
  if (n == 0 || (size_t)n_blinds + 1 > n) return set_error(ctx, SPB_ERR_ARG, "spb_lookup_product_dev: more blinding rows than rows");
  SPB_ENTER(ctx);
  const Fr b = fr_load(beta), g = fr_load(gamma);
  auto terms = [&](DeviceState& dv, size_t lo, size_t cnt, Fr* num, Fr* den) {
    return launch(ctx, dv.stream, nblk(cnt, 256), 256, 0, lookup_terms_kernel, (const Fr*)d_compressed_input + lo, (const Fr*)d_compressed_table + lo,
                  (const Fr*)d_permuted_input + lo, (const Fr*)d_permuted_table + lo, b, g, cnt, num, den);
  };
  return fraction_product(ctx, n, terms, fp_one<FrParams>(), blinds, n_blinds, (Fr*)d_z, nullptr);
}

int spb_weighted_sum_dev(spb_ctx* ctx, const spb_fr* const* d_polys, const spb_fr* weights, size_t count, spb_fr* d_out, size_t n) {
  if (!ctx) return SPB_ERR_ARG;
  if (!d_polys || !weights || !count || !d_out) return set_error(ctx, SPB_ERR_ARG, "spb_weighted_sum_dev: null argument");
  if (!n) return 0;
  SPB_ENTER(ctx);
  char* buf = (char*)slot(ctx, d, "plonk_wsum", count * (sizeof(void*) + 32));
  if (!buf) return SPB_ERR_OOM;
  Fr* dw = (Fr*)buf; const Fr** dp = (const Fr**)(buf + count * 32);
  SPB_CUDA(ctx, cudaMemcpyAsync(dw, weights, count * 32, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(dp, d_polys, count * sizeof(void*), cudaMemcpyHostToDevice, d.stream));
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, weighted_sum_kernel, dp, dw, (uint32_t)count, (Fr*)d_out, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

// ---- SHPLONK -------------------------------------------------------------------------------------------------------
void spb_shplonk_abort(spb_ctx* ctx, spb_shplonk* s) {
  if (!ctx || !s) return;
  std::lock_guard<std::mutex> lk(ctx->mu);
  shplonk_release(s);
}

int spb_shplonk_begin_dev(spb_ctx* ctx, const spb_srs* srs, size_t n, const spb_rotation_set* sets, uint32_t n_sets, const spb_fr* y, const spb_fr* v,
                          spb_g1* h_commitment, spb_shplonk** out) {
  if (!ctx) return SPB_ERR_ARG;
  if (!srs || !sets || !n_sets || !y || !v || !h_commitment || !out || n < 2) return set_error(ctx, SPB_ERR_ARG, "spb_shplonk_begin_dev: null argument");
  *out = nullptr;
  uint32_t total = 0;
  for (uint32_t i = 0; i < n_sets; i++) {
    const spb_rotation_set& rs = sets[i];
    if (!rs.n_points || rs.n_points > 8 || rs.n_points >= n || !rs.n_polys || !rs.points || !rs.d_polys || !rs.evals)
      return set_error(ctx, SPB_ERR_ARG, "spb_shplonk_begin_dev: rotation set %u is malformed (1..8 points, >= 1 polynomial)", i);
    total += rs.n_polys;
  }
  spb_shplonk* s = new spb_shplonk();
  s->ctx = ctx; s->n = n; s->srs = srs; s->n_polys = total; s->y = fr_load(y); s->v = fr_load(v);
  // host side: the sets, the low-degree equivalents R_ij and the super point set
  std::vector<const Fr*> ptrs; ptrs.reserve(total);
  for (uint32_t i = 0; i < n_sets; i++) {
    const spb_rotation_set& rs = sets[i];
    spb_shplonk::Set st;
    st.n_polys = rs.n_polys;
    for (uint32_t p = 0; p < rs.n_points; p++) {
      Fr pt = fr_load(rs.points + p);
      if (contains(st.points, pt)) { delete s; return set_error(ctx, SPB_ERR_ARG, "spb_shplonk_begin_dev: repeated point in rotation set %u", i); }
      st.points.push_back(pt);
      if (!contains(s->super_points, pt)) s->super_points.push_back(pt);
    }
    st.evals.resize((size_t)rs.n_polys * rs.n_points);
    memcpy(st.evals.data(), rs.evals, st.evals.size() * 32);
    st.r.resize(rs.n_polys);
    for (uint32_t j = 0; j < rs.n_polys; j++) {
      st.r[j].resize(rs.n_points);
      lagrange_interpolate(st.points, st.evals.data() + (size_t)j * rs.n_points, st.r[j].data());
      ptrs.push_back((const Fr*)rs.d_polys[j]);
    }
    s->sets.push_back(std::move(st));
  }
  int rc = 0;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceState& d = ctx->dev[0];
    auto fail = [&](int code) { shplonk_release(s); return code; };
#define SHP_CUDA(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { shplonk_release(s); return set_error(ctx, SPB_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } } while (0)
    s->device = d.device;
    SHP_CUDA(cudaSetDevice(d.device));
    // workspace: the context's grow-only slots when no other handle holds them (no allocation in the steady state)
    if (!ctx->shplonk_slots_busy) {
      s->d_h = (Fr*)slot(ctx, d, "shplonk_h", n * 32);
      s->d_tmp[0] = (Fr*)slot(ctx, d, "shplonk_t0", n * 32);
      s->d_tmp[1] = (Fr*)slot(ctx, d, "shplonk_t1", n * 32);
      s->d_ptrs = (const Fr**)slot(ctx, d, "shplonk_ptrs", (size_t)total * sizeof(void*));
      s->d_w = (Fr*)slot(ctx, d, "shplonk_w", (size_t)total * 32);
      if (!s->d_h || !s->d_tmp[0] || !s->d_tmp[1] || !s->d_ptrs || !s->d_w) { delete s; return SPB_ERR_OOM; }
      s->from_slots = true; ctx->shplonk_slots_busy = true;
    } else {
      cudaError_t e = cudaMalloc(&s->d_h, n * 32);
      if (e == cudaSuccess) e = cudaMalloc(&s->d_tmp[0], n * 32);
      if (e == cudaSuccess) e = cudaMalloc(&s->d_tmp[1], n * 32);
      if (e == cudaSuccess) e = cudaMalloc((void**)&s->d_ptrs, (size_t)total * sizeof(void*));
      if (e == cudaSuccess) e = cudaMalloc(&s->d_w, (size_t)total * 32);
      if (e != cudaSuccess) { shplonk_release(s); return set_error(ctx, SPB_ERR_OOM, "spb_shplonk_begin_dev: %s", cudaGetErrorString(e)); }
    }
    SHP_CUDA(cudaMemcpyAsync((void*)s->d_ptrs, ptrs.data(), (size_t)total * sizeof(void*), cudaMemcpyHostToDevice, d.stream));
    SHP_CUDA(cudaMemsetAsync(s->d_h, 0, n * 32, d.stream));
    uint32_t base = 0;
    Fr vpow = fp_one<FrParams>();
    for (uint32_t i = 0; i < n_sets; i++) {
      spb_shplonk::Set& st = s->sets[i];
      const uint32_t m = st.n_polys, np = (uint32_t)st.points.size();
      // N_i(X) = sum_j y^j (P_ij(X) - R_ij(X))      (upstream: numerators.zip(powers(y)))
      std::vector<Fr> w(m);
      Fr pw = fp_one<FrParams>();
      for (uint32_t j = 0; j < m; j++) { w[j] = pw; pw = fp_mul(pw, s->y); }
      SmallPoly rsum; rsum.n = np;
      for (uint32_t t = 0; t < np; t++) rsum.c[t] = fp_zero<FrParams>();
      for (uint32_t j = 0; j < m; j++) for (uint32_t t = 0; t < np; t++) rsum.c[t] = fp_add(rsum.c[t], fp_mul(w[j], st.r[j][t]));
      SHP_CUDA(cudaMemcpyAsync(s->d_w + base, w.data(), (size_t)m * 32, cudaMemcpyHostToDevice, d.stream));
      if ((rc = launch(ctx, d.stream, nblk(n, 256), 256, 0, weighted_sum_kernel, s->d_ptrs + base, s->d_w + base, m, s->d_tmp[0], n)) != 0) return fail(rc);
      if ((rc = launch(ctx, d.stream, 1, 8, 0, sub_small_kernel, s->d_tmp[0], rsum)) != 0) return fail(rc);
      // Q_i(X) = N_i(X) / prod_p (X - point_p): one Kate division per point
      size_t len = n; int cur = 0;
      for (uint32_t p = 0; p < np; p++) {
        if ((rc = dev_kate_division(ctx, d, s->d_tmp[cur], len, st.points[p], s->d_tmp[cur ^ 1])) != 0) return fail(rc);
        cur ^= 1; len--;
      }
      // h <- h + v^i * Q_i (Q_i zero-extended to n)   (upstream: quotient_polynomials.zip(powers(v)))
      if ((rc = launch(ctx, d.stream, nblk(n, 256), 256, 0, scale_add_kernel, s->d_h, fp_one<FrParams>(), s->d_tmp[cur], vpow, len, n)) != 0) return fail(rc);
      vpow = fp_mul(vpow, s->v);
      SHP_CUDA(cudaStreamSynchronize(d.stream));   // w (host vector) must outlive the copy
      base += m;
    }
  }
  rc = spb_msm_dev(ctx, srs, SPB_BASIS_G, (const spb_fr*)s->d_h, n, h_commitment);
  if (rc != 0) { std::lock_guard<std::mutex> lk(ctx->mu); shplonk_release(s); return rc; }
  *out = s;
  return 0;
}

int spb_shplonk_finish_dev(spb_ctx* ctx, spb_shplonk* s, const spb_fr* u, spb_g1* commitment) {
  if (!ctx) return SPB_ERR_ARG;
  if (!s || !u || !commitment) return set_error(ctx, SPB_ERR_ARG, "spb_shplonk_finish_dev: null argument");
  const Fr uu = fr_load(u);
  const size_t n = s->n;
  const uint32_t n_sets = (uint32_t)s->sets.size();
  // weights w_ij = v^i * Z_{T \ S_i}(u) * y^j; constant = sum w_ij * R_ij(u); and -Z_T(u) on h
  std::vector<Fr> w; w.reserve(s->n_polys);
  Fr constant = fp_zero<FrParams>(), z0 = fp_one<FrParams>();
  Fr vpow = fp_one<FrParams>();
  std::vector<Fr> vp(n_sets);
  for (uint32_t i = 0; i < n_sets; i++) { vp[i] = vpow; vpow = fp_mul(vpow, s->v); }
  for (uint32_t i = 0; i < n_sets; i++) {
    const spb_shplonk::Set& st = s->sets[i];
    std::vector<Fr> diffs;
    for (const Fr& pt : s->super_points) if (!contains(st.points, pt)) diffs.push_back(pt);
    Fr zi = vanishing_eval(diffs, uu);
    if (i == 0) z0 = zi;
    Fr outer = fp_mul(vp[i], zi);
    std::vector<Fr> yp(st.n_polys);
    Fr pw = fp_one<FrParams>();
    for (uint32_t j = 0; j < st.n_polys; j++) { yp[j] = pw; pw = fp_mul(pw, s->y); }
    for (uint32_t j = 0; j < st.n_polys; j++) {
      Fr wij = fp_mul(outer, yp[j]);
      w.push_back(wij);
      constant = fp_add(constant, fp_mul(wij, eval_small(st.r[j].data(), st.points.size(), uu)));
    }
  }
  if (fp_is_zero(z0)) { spb_shplonk_abort(ctx, s); return set_error(ctx, SPB_ERR_ARG, "spb_shplonk_finish_dev: u is one of the opening points"); }
  const Fr zt = vanishing_eval(s->super_points, uu);
  const Fr z0_inv = fp_inv(z0);
  int rc = 0;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceState& d = ctx->dev[0];
    auto fail = [&](int code) { shplonk_release(s); return code; };
    SHP_CUDA(cudaSetDevice(d.device));
    SHP_CUDA(cudaMemcpyAsync(s->d_w, w.data(), (size_t)s->n_polys * 32, cudaMemcpyHostToDevice, d.stream));
    // L(X) = sum w_ij P_ij(X) - constant - Z_T(u) h(X)
    if ((rc = launch(ctx, d.stream, nblk(n, 256), 256, 0, weighted_sum_kernel, s->d_ptrs, s->d_w, s->n_polys, s->d_tmp[0], n)) != 0) return fail(rc);
    SmallPoly c0; c0.n = 1; c0.c[0] = constant;
    if ((rc = launch(ctx, d.stream, 1, 8, 0, sub_small_kernel, s->d_tmp[0], c0)) != 0) return fail(rc);
    // tmp0 <- 1 * tmp0 + (-zt) * h  ==  scale_add on a copy of h: h <- (-zt) * h + tmp0
    if ((rc = launch(ctx, d.stream, nblk(n, 256), 256, 0, scale_add_kernel, s->d_h, fp_neg(zt), s->d_tmp[0], fp_one<FrParams>(), n, n)) != 0) return fail(rc);
    // (L(X) / (X - u)) / Z_{T \ S_0}(u)
    if ((rc = dev_kate_division(ctx, d, s->d_h, n, uu, s->d_tmp[1])) != 0) return fail(rc);
    if ((rc = launch(ctx, d.stream, nblk(n - 1, 256), 256, 0, scale_add_kernel, s->d_tmp[1], z0_inv, nullptr, fp_zero<FrParams>(), 0, n - 1)) != 0) return fail(rc);
    SHP_CUDA(cudaStreamSynchronize(d.stream));
  }
  rc = spb_msm_dev(ctx, s->srs, SPB_BASIS_G, (const spb_fr*)s->d_tmp[1], n - 1, commitment);
  { std::lock_guard<std::mutex> lk(ctx->mu); shplonk_release(s); }
  return rc;
}

}  // extern "C"
