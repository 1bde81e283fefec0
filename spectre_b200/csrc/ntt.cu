// Host side of the NTT: power-table cache, digit plan, pass launches. Kernels are in ntt.cuh.
#define SPB_NTT_KERNELS 1
#include "common.cuh"
#include "ntt.cuh"
#include <string.h>

namespace spb {

// log2 elements per shared-memory tile. 2^11 elements (~68 KB of limb planes + twiddles) with 256 threads lets two
// CTAs share an SM (H100: 227 KB of shared memory per block, 228 KB per SM), so one tile's global load/store phases overlap
// the other's butterflies; 2^10 up to 2^20.
static uint32_t tile_elems_log(uint32_t k) { return k <= 20 ? 10 : 11; }
// largest sub-NTT held in one shared-memory tile (11: two passes up to 2^22; the tile is then 2048 x 2 columns)
static const uint32_t kMaxDigitBits = 11;
// threads per pass CTA
static const uint32_t kPassThreads = 256;
// full omega^i tables are kept while their total stays under this many bytes per device (else two-level tables)
static const size_t kFullTableBudget = (size_t)6 << 30;

static NttPlan make_plan(uint32_t k) { return ntt_make_plan(k, kMaxDigitBits); }

// Power tables of `omega` split at h, cached per (k, omega, h) in `cache`: the twiddle tables (d.ntt_tables, with a full table
// while the budget allows) or the pre-scale tables of coset generators (d.ntt_pre_tables, two-level only). The two caches are
// separate, so fetching one kind never evicts a table of the other kind that the same transform is about to use.
static int get_tables(spb_ctx* ctx, DeviceState& d, std::vector<NttTables>& cache, uint32_t k, const Fr& omega, uint32_t h, bool full_allowed, NttTables** out) {
  for (auto& t : cache)
    if (t.k == k && t.h == h && fp_eq(t.omega, omega)) { *out = &t; return 0; }
  NttTables t; t.omega = omega; t.k = k; t.h = h;
  size_t nlo = (size_t)1 << h, nhi = (size_t)1 << (k - h);
  SPB_CUDA(ctx, cudaMalloc(&t.tw_lo, nlo * sizeof(Fr)));
  SPB_CUDA(ctx, cudaMalloc(&t.tw_hi, nhi * sizeof(Fr)));
  SPB_TRY(launch(ctx, d.stream, nblk(nlo, 128), 128, 0, fr_pow_table_kernel, t.tw_lo, omega, nlo, 0));
  SPB_TRY(launch(ctx, d.stream, nblk(nhi, 128), 128, 0, fr_pow_table_kernel, t.tw_hi, omega, nhi, h));
  if (full_allowed) {
    size_t used = 0;
    for (auto& o : cache) if (o.tw_full) used += ((size_t)1 << o.k) * sizeof(Fr);
    size_t need = ((size_t)1 << k) * sizeof(Fr);
    if (k >= 12 && used + need <= kFullTableBudget && cudaMalloc(&t.tw_full, need) == cudaSuccess) {
      SPB_TRY(launch(ctx, d.stream, nblk((uint64_t)1 << k, 128), 128, 0, fr_pow_table_kernel, t.tw_full, omega, (uint64_t)1 << k, 0));
    } else {
      t.tw_full = nullptr;
      cudaGetLastError();  // the optional table's failed cudaMalloc must not be reported by the next launch check
    }
  }
  // a long-lived prover touches a handful of (k, omega) pairs; cap the cache anyway
  if (cache.size() >= 32) {
    cudaStreamSynchronize(d.stream);
    cudaFree(cache.front().tw_lo); cudaFree(cache.front().tw_hi); if (cache.front().tw_full) cudaFree(cache.front().tw_full);
    cache.erase(cache.begin());
  }
  cache.push_back(t);
  *out = &cache.back();
  return 0;
}

void ntt_free_tables(DeviceState& d) {
  for (auto* cache : {&d.ntt_tables, &d.ntt_pre_tables}) {
    for (auto& t : *cache) { cudaFree(t.tw_lo); cudaFree(t.tw_hi); if (t.tw_full) cudaFree(t.tw_full); }
    cache->clear();
  }
}

// Geometry of pass `pi` (ntt_fill_pass, shared with the host emulation) and its launch.
static int launch_pass(spb_ctx* ctx, DeviceState& d, const NttPlan& plan, uint32_t pi, uint32_t k, const NttTables* tb, uint32_t h,
                       const Fr* src, Fr* dst, const NttOpts& opts, const NttShare& sh, const NttTables* pre = nullptr) {
  NttPassParams p;
  p.src = src; p.dst = dst; p.tw_lo = tb->tw_lo; p.tw_hi = tb->tw_hi; p.tw_full = tb->tw_full;
  NttOptsHost oh; oh.n_in = opts.n_in; oh.n_out = opts.n_out; oh.pre3 = opts.pre3; oh.post3 = opts.post3;
  if (pre) { oh.pre_lo = pre->tw_lo; oh.pre_hi = pre->tw_hi; }
  NttLaunch L = ntt_fill_pass(p, plan, pi, k, h, oh, sh, tile_elems_log(k), kPassThreads);
  if (L.smem > 227 * 1024) return set_error(ctx, SPB_ERR_STATE, "ntt: tile needs %zu B of shared memory", L.smem);
  // persistent CTAs: as many as fit the SMs (shared memory bound), striding over the tiles
  uint64_t per_sm = (227 * 1024) / (L.smem + 1024); if (per_sm < 1) per_sm = 1; if (per_sm > 4) per_sm = 4;
  uint64_t grid = (uint64_t)d.sm_count * per_sm; if (grid > L.tiles) grid = L.tiles;
  // Persistence pays up to 2^20 (launch + twiddle staging amortised); beyond
  // that co-resident persistent CTAs run their load/compute phases in lockstep and lose the overlap that
  // hardware-scheduled one-tile CTAs get for free, so large transforms launch one CTA per tile.
  if (k > 20) grid = L.tiles;
  return launch(ctx, d.stream, (unsigned)grid, L.threads, L.smem, ntt_pass_kernel, p);
}

static int set_smem_attr(spb_ctx* ctx, DeviceState& d) {
  static std::map<int, bool> done;      // process-wide (several contexts may share a device)
  static std::mutex done_mu;
  std::lock_guard<std::mutex> lk(done_mu);
  if (!done[d.device]) {
    SPB_CUDA(ctx, cudaFuncSetAttribute(ntt_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    done[d.device] = true;
  }
  return 0;
}

int ntt_device(spb_ctx* ctx, DeviceState& d, const Fr* d_src, Fr* d_dst, uint32_t k, const Fr& omega, const NttOpts& opts) {
  if (k > 28) return set_error(ctx, SPB_ERR_ARG, "ntt: log_n = %u exceeds the two-adicity (28) of Fr", k);
  const uint64_t n = 1ull << k;
  NttPlan plan = make_plan(k);
  uint32_t h = k - plan.s[0];
  NttTables* tb = nullptr;
  NttTables* pre = nullptr;
  SPB_TRY(get_tables(ctx, d, d.ntt_tables, k, omega, h, true, &tb));
  if (opts.pre_generator) SPB_TRY(get_tables(ctx, d, d.ntt_pre_tables, k, *opts.pre_generator, h, false, &pre));
  Fr* tmp = nullptr;
  if (plan.npass > 1) {
    tmp = (Fr*)slot(ctx, d, "ntt_tmp", n * sizeof(Fr));
    if (!tmp) return SPB_ERR_OOM;
  }
  SPB_TRY(set_smem_attr(ctx, d));
  for (uint32_t pi = 0; pi < plan.npass; pi++) {
    const Fr* src = (pi == 0) ? d_src : tmp;
    Fr* dst = (pi == plan.npass - 1) ? d_dst : tmp;
    SPB_TRY(launch_pass(ctx, d, plan, pi, k, tb, h, src, dst, opts, NttShare(), pre));
  }
  return 0;
}

bool ntt_multi_applicable(spb_ctx* ctx, uint32_t k) {
  size_t G = ctx->dev.size();
  if (G < 2 || (G & (G - 1))) return false;
  if (k < 16) return false;
  NttPlan plan = make_plan(k);
  uint32_t g = 0; while ((1u << g) < G) g++;
  return plan.npass >= 2 && plan.s[0] > g && (k - plan.s[0]) > g + 1;
}

// Six-step NTT across the devices of the context, host buffers in and out (natural order both sides):
//   1. each device receives a block of COLUMNS of the n1 x (n/n1) input matrix (strided 2-D H2D copy),
//   2. first-digit pass + inter-digit twiddle locally,
//   3. ONE all-to-all over NVLink (peer 2-D copies) so that each device owns a block of first-digit values i_1 with all
//      remaining digits -- which is a contiguous slice of the positional intermediate array,
//   4. remaining passes locally; the last pass writes a (n/n1) x (n1/G) block,
//   5. strided 2-D D2H copy of that block into the natural-order result.
// ev_ms (optional): device milliseconds between the end of the H2D copies and the start of the D2H copies.
int ntt_multi_host(spb_ctx* ctx, const Fr* in, Fr* out, uint32_t k, const Fr& omega, const NttOpts& opts, float* ev_ms) {
  const size_t G = ctx->dev.size();
  uint32_t g = 0; while ((1u << g) < G) g++;
  const uint64_t n = 1ull << k;
  NttPlan plan = make_plan(k);
  const uint32_t s1 = plan.s[0], rest = k - s1, h = k - s1;
  const uint64_t n1 = 1ull << s1, lo_count = 1ull << rest, lo_loc = lo_count >> g, rows_loc = n1 >> g, per = n >> g;
  const uint64_t n_in = opts.n_in ? opts.n_in : n, n_out = opts.n_out ? opts.n_out : n;
  const uint64_t rows_in = (n_in + lo_count - 1) / lo_count;          // input rows that exist in the caller's buffer
  const uint64_t rows_out = (n_out + n1 - 1) / n1;                    // output rows (of n1 elements) to return
  std::vector<Fr*> A(G), B(G);
  std::vector<NttTables*> tbs(G);
  for (size_t q = 0; q < G; q++) {
    DeviceState& d = ctx->dev[q];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    A[q] = (Fr*)slot(ctx, d, "ntt_md_a", per * sizeof(Fr));
    B[q] = (Fr*)slot(ctx, d, "ntt_md_b", per * sizeof(Fr));
    if (!A[q] || !B[q]) return SPB_ERR_OOM;
    SPB_TRY(get_tables(ctx, d, d.ntt_tables, k, omega, h, true, &tbs[q]));
    SPB_TRY(set_smem_attr(ctx, d));
    // 1. column block q of the first rows_in rows
    if (rows_in) SPB_CUDA(ctx, cudaMemcpy2DAsync(A[q], lo_loc * sizeof(Fr), in + q * lo_loc, lo_count * sizeof(Fr), lo_loc * sizeof(Fr), rows_in, cudaMemcpyHostToDevice, d.stream));
    SPB_CUDA(ctx, cudaEventRecord(d.stage_ev[2], d.stream));   // "input block resident on q"
  }
  for (size_t q = 0; q < G; q++) {
    DeviceState& d = ctx->dev[q];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    // start the clock (and the compute) once every device has its block: the timed span is passes + all-to-all only
    for (size_t o = 0; o < G; o++) SPB_CUDA(ctx, cudaStreamWaitEvent(d.stream, ctx->dev[o].stage_ev[2], 0));
    SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
    // 2. first pass
    NttShare sh; sh.g_log = g; sh.q = (uint32_t)q; sh.mode = 1;
    SPB_TRY(launch_pass(ctx, d, plan, 0, k, tbs[q], h, A[q], A[q], opts, sh));
    SPB_CUDA(ctx, cudaEventRecord(d.stage_ev[0], d.stream));   // "pass 1 done on q"
  }
  // 3. all-to-all: destination qd pulls block (rows of qd, columns of qs) from every A[qs] into B[qd] at column offset qs.
  //    With peer access this is one kernel per destination reading peers' HBM over NVLink; without it, 2-D copies.
  for (size_t qd = 0; qd < G; qd++) {
    DeviceState& dd = ctx->dev[qd];
    SPB_CUDA(ctx, cudaSetDevice(dd.device));
    for (size_t qs = 0; qs < G; qs++) SPB_CUDA(ctx, cudaStreamWaitEvent(dd.stream, ctx->dev[qs].stage_ev[0], 0));
    if (ctx->peer_access && G <= 16) {
      NttGatherArgs ga; memset(&ga, 0, sizeof ga);
      for (size_t qs = 0; qs < G; qs++) ga.peers[qs] = A[qs];
      ga.dst = B[qd]; ga.rows_loc = rows_loc; ga.lo_loc = lo_loc; ga.row_base = qd * rows_loc; ga.g_log = g;
      SPB_TRY(launch(ctx, dd.stream, dd.sm_count * 8, 256, 0, ntt_gather_kernel, ga));
    } else {
      for (size_t qs = 0; qs < G; qs++)
        SPB_CUDA(ctx, cudaMemcpy2DAsync(B[qd] + qs * lo_loc, lo_count * sizeof(Fr), A[qs] + qd * rows_loc * lo_loc, lo_loc * sizeof(Fr),
                                        lo_loc * sizeof(Fr), rows_loc, cudaMemcpyDefault, dd.stream));
    }
    SPB_CUDA(ctx, cudaEventRecord(dd.stage_ev[1], dd.stream));  // "B[qd] complete": A[qs] blocks for qd have been read
  }
  // 4. remaining passes on the slice; the result block goes back into A[q] once every reader of A[q] is done
  for (size_t q = 0; q < G; q++) {
    DeviceState& d = ctx->dev[q];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    for (size_t o = 0; o < G; o++) SPB_CUDA(ctx, cudaStreamWaitEvent(d.stream, ctx->dev[o].stage_ev[1], 0));
    NttShare sh; sh.g_log = g; sh.q = (uint32_t)q; sh.mode = 2;
    Fr* vbase = B[q] - q * per;   // virtual base: the slice sits at its global position
    for (uint32_t pi = 1; pi < plan.npass; pi++) {
      bool last = pi == plan.npass - 1;
      SPB_TRY(launch_pass(ctx, d, plan, pi, k, tbs[q], h, vbase, last ? A[q] : vbase, opts, sh));
    }
    SPB_CUDA(ctx, cudaEventRecord(d.ev1, d.stream));
    // 5. (rows_out) x (n1/G) block -> natural-order host result
    if (rows_out) SPB_CUDA(ctx, cudaMemcpy2DAsync(out + q * rows_loc, n1 * sizeof(Fr), A[q], rows_loc * sizeof(Fr), rows_loc * sizeof(Fr), rows_out, cudaMemcpyDeviceToHost, d.stream));
  }
  float worst = 0.f;
  for (size_t q = 0; q < G; q++) {
    DeviceState& d = ctx->dev[q];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
    float ms = 0.f; cudaEventElapsedTime(&ms, d.ev0, d.ev1);
    if (ms > worst) worst = ms;
  }
  if (ev_ms) *ev_ms = worst;
  ctx->last_kernel_ms = worst;
  return 0;
}

}  // namespace spb
