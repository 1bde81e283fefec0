// Quotient numerator on the extended coset: the three row loops of halo2's Evaluator::evaluate_h
// ([UPSTREAM] halo2_proofs/src/plonk/evaluation.rs; SURVEY.md 8a row a6, stage 8 of create_proof):
//   * spb_graph_evaluate_dev      -- GraphEvaluator::evaluate for every extended row (custom gates, and the
//                                    compressed-expression product each lookup needs),
//   * spb_permutation_constraints_dev -- the permutation argument terms folded with powers of y,
//   * spb_lookup_constraints_dev  -- the five lookup-argument terms of one lookup.
// Each is one streaming pass over the extended polynomials it reads: algorithmic bytes = 32 B x (#input columns + 1
// read + 1 write of `values`) per extended row. The gate graph arrives in the flat encoding documented at
// include/spectre_b200.h (spb_graph) -- what the Rust shim produces from GraphEvaluator's `calculations`.
// Intermediates live in a device scratch laid out [intermediate][thread slot] (coalesced), rows are grid-strided.
// The per-row bodies are in quotient.cuh (host+device: tests/hostemu runs them on the CPU).
// Parity: bit-exact against the CPU restatement on synthetic constraint systems (tests/test_gpu_quotient.py);
// not pinned by any reference-owned vector (none exists for this row).
#include "common.cuh"
#include "quotient.cuh"
#include <string.h>
#include <algorithm>
#include <utility>
#include <vector>

using namespace spb;

__global__ void __launch_bounds__(256) graph_evaluate_kernel(GraphArgs a) {
  const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x, nslots = gridDim.x * blockDim.x;
  for (uint64_t row = a.row_lo + slot; row < a.row_hi; row += nslots) graph_evaluate_row(a, row, slot, nslots);
}

// one extended_omega power per block (thread 0: 2 log2(idx) products) times a 256-entry table entry per thread, instead of
// a full exponentiation per row
__global__ void __launch_bounds__(256, 3) permutation_constraints_kernel(PermArgs a) {
  __shared__ Fr base;
  const uint64_t block_row = a.row_lo + blockIdx.x * (uint64_t)blockDim.x;   // row_lo is a multiple of 256
  if (threadIdx.x == 0) base = fp_pow_u64(a.extended_omega, block_row);
  __syncthreads();
  const uint64_t idx = block_row + threadIdx.x;
  if (idx < a.row_hi) permutation_constraints_row(a, idx, fp_mul(base, ntt_ldg(a.omega_pow + threadIdx.x)));
}

__global__ void __launch_bounds__(256) lookup_constraints_kernel(LookupArgs a) {
  uint64_t idx = a.row_lo + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (idx < a.row_hi) lookup_constraints_row(a, idx);
}

__global__ void __launch_bounds__(256) extended_part_scatter_kernel(const Fr* part_values, Fr* extended, uint32_t part, uint32_t R, uint64_t row_lo, uint64_t row_hi) {
  uint64_t m = row_lo + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (m < row_hi) extended_part_scatter_row(part_values, extended, part, R, m);
}

namespace {

// Each pass runs in row-range shards over `size` extended rows (row_ranges; SURVEY.md 8e "evaluate_h / pointwise":
// embarrassingly parallel by extended-row range). The polynomials stay where the caller put them -- on the first device of the
// context; the other devices run the same kernel on their row range and read the inputs (rotations included: any row of any
// polynomial) and write their slice of `values` straight through NVLink peer access, so no halo is exchanged and no staging
// copy exists.
// shard_begin: the shard's device is made current, its stream ordered after everything queued on the first device's stream so far
int shard_begin(spb_ctx* ctx, const RowRange& sh) {
  DeviceState& d0 = ctx->dev[0];
  DeviceState& d = ctx->dev[sh.dev_index];
  SPB_CUDA(ctx, cudaSetDevice(d.device));
  // d0.dep_ev was recorded at entry (SPB_ENTER0), i.e. BEFORE the first device's own shard was enqueued: the other devices
  // wait for the caller's inputs only, not for the first device's share of this pass
  if (sh.dev_index != 0) SPB_CUDA(ctx, cudaStreamWaitEvent(d.stream, d0.dep_ev, 0));
  return 0;
}
// wait for every shard; last_kernel_ms = device time of the pass on the first device's clock
int shards_finish(spb_ctx* ctx, const std::vector<RowRange>& shards) {
  DeviceState& d0 = ctx->dev[0];
  for (auto& sh : shards) {
    if (sh.dev_index == 0) continue;
    DeviceState& d = ctx->dev[sh.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaEventRecord(d.dep_ev, d.stream));
    SPB_CUDA(ctx, cudaStreamWaitEvent(d0.stream, d.dep_ev, 0));
  }
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  SPB_CUDA(ctx, cudaEventRecord(d0.ev1, d0.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d0.stream));
  SPB_CUDA(ctx, cudaEventElapsedTime(&ctx->last_kernel_ms, d0.ev0, d0.ev1));
  for (auto& sh : shards) if (sh.dev_index != 0) { SPB_CUDA(ctx, cudaSetDevice(ctx->dev[sh.dev_index].device)); SPB_CUDA(ctx, cudaStreamSynchronize(ctx->dev[sh.dev_index].stream)); }
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  return 0;
}

// copy a host array of device pointers to the device (slot `name`)
const Fr* const* upload_ptrs(spb_ctx* ctx, DeviceState& d, const char* name, const spb_fr* const* p, uint32_t n) {
  void* dst = slot(ctx, d, name, (n ? n : 1) * sizeof(void*));
  if (!dst) return nullptr;
  if (n && cudaMemcpyAsync(dst, p, n * sizeof(void*), cudaMemcpyHostToDevice, d.stream) != cudaSuccess) return nullptr;
  return (const Fr* const*)dst;
}

// ---- program scheduling: fewer live intermediates per row ------------------------------------------------------------------
// GraphEvaluator's calculations come in "one intermediate per node" form, and its final Horner folds every gate at once, so all
// gate values are alive until the very end: 76 intermediates for the 15-gate halo2-lib shape, i.e. 2.4 KB of scratch per thread and
// 184 MB for the grid -- more than the L2, so the scratch traffic (not the column reads) set the kernel's time. The program is
// tiny and evaluated for millions of rows, so it is rescheduled here, once per call, on the host:
//  1. a Horner over k parts becomes k one-part Horner steps (same arithmetic: acc = acc * factor + part), each placed right after
//     the calculation that produces its part, so a gate's value dies as soon as it is folded in;
//  2. intermediates are renamed to scratch slots by liveness (a slot is reused once its value has been read for the last time).
// Values are unchanged bit for bit (the same field operations in the same operand order); only scratch addresses and the order of
// independent calculations move. Programs that write a target twice are left as they are.
struct Calc { uint32_t op, nparts, target; std::vector<std::pair<uint32_t, uint32_t>> src; double key; };
bool schedule_program(const uint32_t* words, size_t nwords, uint32_t ncalc, std::vector<uint32_t>& out, uint32_t& nslots_out, uint32_t& ncalc_out) {
  std::vector<Calc> calcs;
  size_t w = 0;
  uint32_t max_id = 0;
  for (uint32_t c = 0; c < ncalc; c++) {
    if (w + 2 > nwords) return false;
    Calc k; k.op = words[w] & 0xffu; k.nparts = words[w] >> 8; k.target = words[w + 1]; k.key = 0;
    const uint32_t ns = k.op <= 2 ? 2u : (k.op == 6 ? 2u + k.nparts : 1u);
    if (k.op > 7 || w + 2 + 2 * (size_t)ns > nwords) return false;
    for (uint32_t i = 0; i < ns; i++) k.src.push_back({words[w + 2 + 2 * i], words[w + 3 + 2 * i]});
    w += 2 + 2 * (size_t)ns;
    if (k.target > max_id) max_id = k.target;
    calcs.push_back(std::move(k));
  }
  if (calcs.empty()) return false;
  std::vector<int> producer(max_id + 1, -1);
  for (size_t i = 0; i < calcs.size(); i++) {
    if (producer[calcs[i].target] != -1) return false;           // a target written twice: keep the caller's schedule
    producer[calcs[i].target] = (int)i;
  }
  auto produced_at = [&](const std::pair<uint32_t, uint32_t>& s) -> int {   // index of the calculation a source waits for, -1 if none
    if (s.first != 1) return -1;
    const uint32_t id = s.second & 0xffffu;
    return id <= max_id ? producer[id] : -1;
  };
  // 1. split the Horners; key = position in the original order (+ a small offset that keeps the chain ordered)
  std::vector<Calc> sched;
  uint32_t next_id = max_id + 1;
  for (size_t i = 0; i < calcs.size(); i++) {
    Calc& k = calcs[i];
    for (auto& s : k.src) if (s.first == 1 && produced_at(s) < 0) return false;   // reads an intermediate nobody wrote
    if (k.op != 6 || k.nparts < 2) { k.key = (double)i; sched.push_back(k); continue; }
    const int ready0 = std::max(produced_at(k.src[0]), produced_at(k.src[1]));
    double prev_key = -1.0;
    std::pair<uint32_t, uint32_t> acc = k.src[0];
    for (uint32_t p = 0; p < k.nparts; p++) {
      Calc h; h.op = 6; h.nparts = 1;
      h.target = p + 1 == k.nparts ? k.target : next_id++;
      h.src = {acc, k.src[1], k.src[2 + p]};
      const int ready = std::max(ready0, produced_at(k.src[2 + p]));
      double key = (double)ready + 0.5;                            // right after the last producer it waits for ...
      if (key <= prev_key) key = prev_key + 1e-4;                  // ... but after the previous link of the chain
      if (key > (double)i) key = (double)i;                        // never later than the original Horner
      h.key = key; prev_key = key;
      acc = {1u, h.target};
      sched.push_back(std::move(h));
    }
  }
  if (next_id > 0xffffu) return false;
  // the row's result is whatever the LAST calculation produced: the caller's last calculation (or the last link of its Horner) stays last
  for (auto& k : sched) if (k.target == calcs.back().target) k.key = 1e18;
  std::stable_sort(sched.begin(), sched.end(), [](const Calc& a, const Calc& b) { return a.key < b.key; });
  // 2. liveness -> slots
  std::vector<int> last_use(next_id, -1);
  for (size_t i = 0; i < sched.size(); i++) for (auto& s : sched[i].src) if (s.first == 1) last_use[s.second & 0xffffu] = (int)i;
  std::vector<uint32_t> slot_of(next_id, 0xffffffffu), free_slots;
  uint32_t nslots = 0;
  out.clear();
  for (size_t i = 0; i < sched.size(); i++) {
    Calc& k = sched[i];
    std::vector<uint32_t> dying;
    for (auto& s : k.src) {
      if (s.first != 1) continue;
      const uint32_t id = s.second & 0xffffu;
      if (slot_of[id] == 0xffffffffu) return false;                // read before written: the sort broke a dependency (cannot happen)
      s.second = slot_of[id];
      if (last_use[id] == (int)i) dying.push_back(id);
    }
    std::sort(dying.begin(), dying.end()); dying.erase(std::unique(dying.begin(), dying.end()), dying.end());
    for (uint32_t id : dying) { free_slots.push_back(slot_of[id]); slot_of[id] = 0xfffffffeu; }   // the row body reads every source before it stores
    uint32_t sl;
    if (!free_slots.empty()) { sl = free_slots.back(); free_slots.pop_back(); } else sl = nslots++;
    slot_of[k.target] = sl;
    if (last_use[k.target] < 0 && i + 1 != sched.size()) free_slots.push_back(sl);   // never read (dead code): its slot is free at once
    out.push_back(k.op | (k.nparts << 8)); out.push_back(sl);
    for (auto& s : k.src) { out.push_back(s.first); out.push_back(s.second); }
  }
  nslots_out = nslots ? nslots : 1;
  ncalc_out = (uint32_t)sched.size();
  return true;
}

// The permutation pass with X = g * omega^idx at row idx: (zeta, extended_omega) over the whole extended coset, (zeta
// extended_omega^j, omega) over its coset part j.
int permutation_constraints(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len,
                            const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values, const spb_fr* const* d_sigma,
                            const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma,
                            const spb_fr* y, const Fr& g, const Fr& omega) {
  if (!size || (size & (size - 1))) return set_error(ctx, SPB_ERR_ARG, "permutation constraints: the domain size must be a power of two");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceState& d = ctx->dev[0];
  SPB_CUDA(ctx, cudaSetDevice(d.device));
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
  if (ctx->dev.size() > 1) SPB_CUDA(ctx, cudaEventRecord(d.dep_ev, d.stream));
  PermArgs a; memset(&a, 0, sizeof a);
  a.values = (Fr*)d_values; a.size = size; a.rot_scale = rot_scale; a.last_rotation = last_rotation;
  a.n_sets = n_sets; a.chunk_len = chunk_len; a.n_cols = n_cols;
  a.l0 = (const Fr*)d_l0; a.l_last = (const Fr*)d_l_last; a.l_active = (const Fr*)d_l_active;
  a.beta = fr_load(beta); a.gamma = fr_load(gamma); a.y = fr_load(y); a.extended_omega = omega;
  a.delta = fr_delta();
  a.delta_start = fp_mul(a.beta, g);
  std::vector<Fr> pw(256);
  pw[0] = fp_one<FrParams>();
  for (int j = 1; j < 256; j++) pw[j] = fp_mul(pw[j - 1], a.extended_omega);
  const std::vector<RowRange> shards = row_ranges(ctx, size);
  for (auto& sh : shards) {
    DeviceState& dv = ctx->dev[sh.dev_index];
    SPB_TRY(shard_begin(ctx, sh));
    a.z = upload_ptrs(ctx, dv, "q_z", d_z, n_sets);
    a.col_values = upload_ptrs(ctx, dv, "q_cols", d_col_values, n_cols);
    a.sigma = upload_ptrs(ctx, dv, "q_sigma", d_sigma, n_cols);
    Fr* dpw = (Fr*)slot(ctx, dv, "q_omega_pow", 256 * sizeof(Fr));
    if (!a.z || !a.col_values || !a.sigma || !dpw) return set_error(ctx, SPB_ERR_CUDA, "permutation: table upload failed");
    SPB_CUDA(ctx, cudaMemcpyAsync(dpw, pw.data(), 256 * sizeof(Fr), cudaMemcpyHostToDevice, dv.stream));
    a.omega_pow = dpw; a.row_lo = sh.lo; a.row_hi = sh.hi;
    SPB_TRY(launch(ctx, dv.stream, nblk(sh.hi - sh.lo, 256), 256, 0, permutation_constraints_kernel, a));
  }
  return shards_finish(ctx, shards);
}

}  // namespace

extern "C" {

// SPB_ENTER, then start the pass clock and mark the point the other devices' shards wait for (shard_begin)
#define SPB_ENTER0(ctx)                                  \
  SPB_ENTER(ctx);                                        \
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));       \
  if ((ctx)->dev.size() > 1) SPB_CUDA(ctx, cudaEventRecord(d.dep_ev, d.stream));

int spb_graph_evaluate_dev(spb_ctx* ctx, const spb_graph* g, const spb_fr* const* d_fixed, uint32_t n_fixed, const spb_fr* const* d_advice, uint32_t n_advice,
                           const spb_fr* const* d_instance, uint32_t n_instance, const spb_fr* challenges, uint32_t n_challenges, const spb_fr* beta,
                           const spb_fr* gamma, const spb_fr* theta, const spb_fr* y, spb_fr* d_values, uint64_t size, int32_t rot_scale) {
  if (!ctx || !g || !d_values || !beta || !gamma || !theta || !y || (g->program_words && !g->program)) return SPB_ERR_ARG;
  if (g->num_intermediates > 0xffff || g->num_constants > 0x10000 || g->num_rotations > 0xffff) return set_error(ctx, SPB_ERR_ARG, "graph: index fields are 16 bits");
  if (!size || (size & (size - 1))) return set_error(ctx, SPB_ERR_ARG, "graph: the extended domain size must be a power of two");
  // reschedule the program for few live intermediates (schedule_program above); fall back to the caller's words if it declines
  std::vector<uint32_t> prog_words;
  uint32_t n_inter = g->num_intermediates, n_calc = g->num_calculations;
  const uint32_t* prog = g->program;
  size_t prog_n = g->program_words;
  if (g->program_words && schedule_program(g->program, g->program_words, g->num_calculations, prog_words, n_inter, n_calc)) {
    prog = prog_words.data(); prog_n = prog_words.size();
  } else {
    n_inter = g->num_intermediates; n_calc = g->num_calculations;
  }
  SPB_ENTER0(ctx);
  std::vector<Fr> sc(4 + n_challenges);
  sc[0] = fr_load(beta); sc[1] = fr_load(gamma); sc[2] = fr_load(theta); sc[3] = fr_load(y);
  if (n_challenges) memcpy(&sc[4], challenges, (size_t)n_challenges * 32);
  const std::vector<RowRange> shards = row_ranges(ctx, size);
  for (auto& sh : shards) {
    DeviceState& dv = ctx->dev[sh.dev_index];
    SPB_TRY(shard_begin(ctx, sh));
    const uint32_t threads = 256, blocks = (uint32_t)dv.sm_count * 2;   // grid-stride: 2 x 256 threads per SM
    const uint64_t nslots = (uint64_t)threads * blocks;
    GraphArgs a; memset(&a, 0, sizeof a);
    uint32_t* dprog = (uint32_t*)slot(ctx, dv, "q_prog", (prog_n ? prog_n : 1) * 4);
    Fr* dconst = (Fr*)slot(ctx, dv, "q_const", (g->num_constants ? g->num_constants : 1) * sizeof(Fr));
    int32_t* drot = (int32_t*)slot(ctx, dv, "q_rot", (g->num_rotations ? g->num_rotations : 1) * 4);
    Fr* dscal = (Fr*)slot(ctx, dv, "q_scalars", (4 + (size_t)n_challenges) * sizeof(Fr));
    Fr* scratch = (Fr*)slot(ctx, dv, "q_scratch", (n_inter ? n_inter : 1) * nslots * sizeof(Fr));
    if (!dprog || !dconst || !drot || !dscal || !scratch) return SPB_ERR_OOM;
    SPB_CUDA(ctx, cudaMemcpyAsync(dprog, prog, prog_n * 4, cudaMemcpyHostToDevice, dv.stream));
    if (g->num_constants) SPB_CUDA(ctx, cudaMemcpyAsync(dconst, g->constants, (size_t)g->num_constants * 32, cudaMemcpyHostToDevice, dv.stream));
    if (g->num_rotations) SPB_CUDA(ctx, cudaMemcpyAsync(drot, g->rotations, (size_t)g->num_rotations * 4, cudaMemcpyHostToDevice, dv.stream));
    SPB_CUDA(ctx, cudaMemcpyAsync(dscal, sc.data(), sc.size() * 32, cudaMemcpyHostToDevice, dv.stream));
    a.fixed = upload_ptrs(ctx, dv, "q_fixed", d_fixed, n_fixed);
    a.advice = upload_ptrs(ctx, dv, "q_advice", d_advice, n_advice);
    a.instance = upload_ptrs(ctx, dv, "q_instance", d_instance, n_instance);
    if (!a.fixed || !a.advice || !a.instance) return set_error(ctx, SPB_ERR_CUDA, "graph: pointer table upload failed");
    a.prog = dprog; a.ncalc = n_calc; a.constants = dconst; a.rotations = drot; a.scalars = dscal;
    a.values = (Fr*)d_values; a.scratch = scratch; a.size = size; a.rot_scale = rot_scale; a.row_lo = sh.lo; a.row_hi = sh.hi;
    SPB_TRY(launch(ctx, dv.stream, blocks, threads, 0, graph_evaluate_kernel, a));
  }
  return shards_finish(ctx, shards);  // synchronises: `sc` and the caller's arrays outlive the copies
}

// the scheduling pass alone (no device involved): lets the CPU tests run the scheduled program through the oracle's interpreter
int spb_test_schedule_program(const uint32_t* program, size_t program_words, uint32_t num_calculations, uint32_t* out_words, size_t out_capacity,
                              size_t* out_count, uint32_t* num_slots, uint32_t* out_calculations) {
  if (!program || !out_words || !out_count || !num_slots || !out_calculations) return SPB_ERR_ARG;
  std::vector<uint32_t> w; uint32_t ns = 0, nc = 0;
  if (!schedule_program(program, program_words, num_calculations, w, ns, nc)) return SPB_ERR_STATE;
  if (w.size() > out_capacity) return SPB_ERR_ARG;
  memcpy(out_words, w.data(), w.size() * 4);
  *out_count = w.size(); *num_slots = ns; *out_calculations = nc;
  return 0;
}

int spb_permutation_constraints_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len,
                                    const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values, const spb_fr* const* d_sigma,
                                    const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma,
                                    const spb_fr* y, const spb_fr* extended_omega) {
  if (!ctx || !d_values || !beta || !gamma || !y || !extended_omega || !d_l0 || !d_l_last || !d_l_active) return SPB_ERR_ARG;
  if (!n_sets) return 0;
  if (!d_z || !chunk_len || (n_cols && (!d_col_values || !d_sigma))) return SPB_ERR_ARG;
  return permutation_constraints(ctx, d_values, size, rot_scale, last_rotation, n_sets, chunk_len, d_z, n_cols, d_col_values, d_sigma, d_l0, d_l_last,
                                 d_l_active, beta, gamma, y, fr_zeta(), fr_load(extended_omega));
}

int spb_permutation_constraints_coset_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets,
                                          uint32_t chunk_len, const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values,
                                          const spb_fr* const* d_sigma, const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active,
                                          const spb_fr* beta, const spb_fr* gamma, const spb_fr* y, const spb_fr* coset_generator, const spb_fr* omega) {
  if (!ctx || !d_values || !beta || !gamma || !y || !coset_generator || !omega || !d_l0 || !d_l_last || !d_l_active) return SPB_ERR_ARG;
  if (!n_sets) return 0;
  if (!d_z || !chunk_len || (n_cols && (!d_col_values || !d_sigma))) return SPB_ERR_ARG;
  return permutation_constraints(ctx, d_values, size, rot_scale, last_rotation, n_sets, chunk_len, d_z, n_cols, d_col_values, d_sigma, d_l0, d_l_last,
                                 d_l_active, beta, gamma, y, fr_load(coset_generator), fr_load(omega));
}

int spb_extended_part_scatter_dev(spb_ctx* ctx, const spb_domain* dm, uint32_t part, const spb_fr* d_part, spb_fr* d_extended) {
  if (!ctx || !dm || !d_part || !d_extended) return SPB_ERR_ARG;
  if (part >= dm->t_len) return set_error(ctx, SPB_ERR_ARG, "spb_extended_part_scatter_dev: part %u of %u", part, dm->t_len);
  SPB_ENTER0(ctx);
  const std::vector<RowRange> shards = row_ranges(ctx, 1ull << dm->k);
  for (auto& sh : shards) {
    SPB_TRY(shard_begin(ctx, sh));
    SPB_TRY(launch(ctx, ctx->dev[sh.dev_index].stream, nblk(sh.hi - sh.lo, 256), 256, 0, extended_part_scatter_kernel, (const Fr*)d_part, (Fr*)d_extended,
                   part, dm->t_len, sh.lo, sh.hi));
  }
  return shards_finish(ctx, shards);
}

int spb_lookup_constraints_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, const spb_fr* d_product, const spb_fr* d_permuted_input,
                               const spb_fr* d_permuted_table, const spb_fr* d_table_value, const spb_fr* d_l0, const spb_fr* d_l_last,
                               const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma, const spb_fr* y) {
  if (!ctx || !d_values || !d_product || !d_permuted_input || !d_permuted_table || !d_table_value || !d_l0 || !d_l_last || !d_l_active || !beta || !gamma || !y)
    return SPB_ERR_ARG;
  if (!size || (size & (size - 1))) return set_error(ctx, SPB_ERR_ARG, "lookup constraints: the extended domain size must be a power of two");
  SPB_ENTER0(ctx);
  LookupArgs a;
  a.values = (Fr*)d_values; a.size = size; a.rot_scale = rot_scale;
  a.product = (const Fr*)d_product; a.permuted_input = (const Fr*)d_permuted_input; a.permuted_table = (const Fr*)d_permuted_table;
  a.table_value = (const Fr*)d_table_value; a.l0 = (const Fr*)d_l0; a.l_last = (const Fr*)d_l_last; a.l_active = (const Fr*)d_l_active;
  a.beta = fr_load(beta); a.gamma = fr_load(gamma); a.y = fr_load(y);
  const std::vector<RowRange> shards = row_ranges(ctx, size);
  for (auto& sh : shards) {
    SPB_TRY(shard_begin(ctx, sh));
    a.row_lo = sh.lo; a.row_hi = sh.hi;
    SPB_TRY(launch(ctx, ctx->dev[sh.dev_index].stream, nblk(sh.hi - sh.lo, 256), 256, 0, lookup_constraints_kernel, a));
  }
  return shards_finish(ctx, shards);
}

}  // extern "C"
