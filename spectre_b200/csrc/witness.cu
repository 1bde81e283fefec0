// Witness check: halo2's MockProver::verify ([UPSTREAM] halo2_proofs/src/dev.rs) on the device, for the gates, lookups and
// copy constraints of a circuit whose columns are already resident. Three entry points, each ending in the same compaction:
//   * spb_nonzero_rows_dev        -- the rows of a range where a column (a gate evaluated by spb_graph_evaluate_dev) is nonzero,
//   * spb_lookup_missing_rows_dev -- the input rows whose compressed value is not among the table's usable rows: the table is
//                                    sorted with the lookup argument's own canonical sort, in its workspace, then every input
//                                    row binary-searches it in its original row order,
//   * spb_copy_mismatches_dev     -- the cells whose value differs from the value of the cell their sigma labels, sigma decoded
//                                    on the fly (witness.cuh): no sort, no scratch per cell.
// Compaction: a block of kWcRows rows counts its flagged rows (one kernel), cub's exclusive scan gives each block its first
// output slot and the total, and a second kernel writes the flagged rows of the blocks that have any and start below `cap`,
// re-evaluating the flag only there. Only the total and at most `cap` entries cross PCIe.
// The proving-key check (plonk.check_pk, the checked plonk.read_pk) adds two entry points:
//   * spb_fr_first_noncanonical_dev -- the first element not below r, by the params check's grid-stride kernel (common.cuh),
//   * spb_sigma_check_dev           -- sigma as a permutation of the cells: one pass per column decodes each entry once and
//                                      marks the cell it labels in a bitmap (slot "kc_maps"), then the same compaction reports
//                                      the bad entries and the cells no entry labels.
// Every entry point works on the first device of the context and synchronises before it returns.
#include "common.cuh"
#include "witness.cuh"
#include <cub/device/device_scan.cuh>

using namespace spb;

namespace {

struct NonzeroFlag {
  const Fr* values;
  __device__ bool operator()(uint64_t row) const { return !fp_is_zero(ntt_ldg(values + row)); }
  __device__ void store(uint32_t* out, uint64_t cap, uint64_t pos, uint64_t row) const { wc_store(out, cap, pos, row); }
};

struct MissingFlag {
  const Fr* input; const Fr* sorted_table; uint64_t rows;
  __device__ bool operator()(uint64_t row) const { return wc_lookup_missing(sorted_table, rows, ntt_ldg(input + row)); }
  __device__ void store(uint32_t* out, uint64_t cap, uint64_t pos, uint64_t row) const { wc_store(out, cap, pos, row); }
};

// flags a mismatch or a malformed sigma entry; the first malformed cell of the column (lowest row) goes to *bad
struct CopyFlag {
  CopyArgs a;
  unsigned long long* bad;
  __device__ bool operator()(uint64_t row) const {
    uint32_t col; uint64_t r;
    const int rc = copy_check_row(a, row, &col, &r);
    if (rc == 2) atomicMin(bad, ((unsigned long long)a.c << 32) | row);
    return rc != 0;
  }
  // (col, row, col', row') of a mismatch; a malformed entry (the call fails) writes its own cell as col', row'
  __device__ void store(uint32_t* out, uint64_t cap, uint64_t pos, uint64_t row) const {
    if (pos >= cap) return;
    uint32_t col = a.c; uint64_t r = row;
    copy_check_row(a, row, &col, &r);
    out[4 * pos] = a.c; out[4 * pos + 1] = (uint32_t)row; out[4 * pos + 2] = col; out[4 * pos + 3] = (uint32_t)r;
  }
};

// first_bad_kernel's predicate for a polynomial read from a key file
struct FrBad {
  const Fr* v;
  __device__ bool operator()(uint64_t i) const { return fr_noncanonical(ntt_ldg(v + i)); }
};

// the rows of column c whose bit in a cell map is `want`
struct MapFlag {
  const uint32_t* map; uint64_t words_per_col; uint32_t c; uint32_t want;
  __device__ bool operator()(uint64_t row) const { return ((map[sigma_map_word(words_per_col, c, row)] >> (row & 31u)) & 1u) == want; }
  __device__ void store(uint32_t* out, uint64_t cap, uint64_t pos, uint64_t row) const { wc_store(out, cap, pos, row); }
};

// One thread per row of sigma column c: the entry is decoded once (sigma_check_entry), the cell it labels is OR-ed into `hit`,
// and the column's words of `bad` are written whole, one ballot per warp (a word's 32 rows are one warp's, blocks start at
// multiples of 256 rows). Fixed points, nearly every cell of a real key, are marked with one atomic per warp.
__global__ void __launch_bounds__(kWcRows) sigma_mark_kernel(SigmaTables t, const Fr* sigma, uint32_t c, uint64_t n, uint64_t usable, uint64_t words_per_col,
                                                             uint32_t* hit, uint32_t* bad) {
  const uint64_t i = blockIdx.x * (uint64_t)kWcRows + threadIdx.x;
  bool is_bad = false, own = false;
  if (i < n) {
    uint32_t col; uint64_t row;
    if (sigma_check_entry(t, c, i, ntt_ldg(sigma + i), usable, &col, &row, &is_bad)) {
      own = col == c && row == i;
      if (!own) atomicOr(hit + sigma_map_word(words_per_col, col, row), sigma_map_bit(row));
    }
  }
  const unsigned own_m = __ballot_sync(0xffffffffu, own), bad_m = __ballot_sync(0xffffffffu, is_bad);
  const uint64_t first = i - (threadIdx.x & 31u);
  if ((threadIdx.x & 31u) == 0 && first < n) {
    const uint64_t w = sigma_map_word(words_per_col, c, first);
    bad[w] = bad_m;
    if (own_m) atomicOr(hit + w, own_m);
  }
}

template <class F>
__global__ void __launch_bounds__(kWcRows) wc_count_kernel(F f, uint64_t lo, uint64_t hi, uint32_t* counts) {
  const uint64_t row = lo + blockIdx.x * (uint64_t)kWcRows + threadIdx.x;
  const int c = __syncthreads_count(row < hi && f(row));
  if (threadIdx.x == 0) counts[blockIdx.x] = (uint32_t)c;
}

// offsets: exclusive scan of the block counts (nblocks + 1 entries); ranks inside a block by warp ballots, so rows keep their order
template <class F>
__global__ void __launch_bounds__(kWcRows) wc_scatter_kernel(F f, uint64_t lo, uint64_t hi, const uint32_t* offsets, uint64_t cap, uint32_t* out) {
  __shared__ uint32_t warp_base[kWcRows / 32];
  const uint32_t first = offsets[blockIdx.x];
  if (offsets[blockIdx.x + 1] == first || first >= cap) return;   // the same for the whole block
  const uint64_t row = lo + blockIdx.x * (uint64_t)kWcRows + threadIdx.x;
  const bool flag = row < hi && f(row);
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_base[warp] = (uint32_t)__popc(m);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int w = 0; w < kWcRows / 32; w++) { const uint32_t c = warp_base[w]; warp_base[w] = run; run += c; }
  }
  __syncthreads();
  if (flag) f.store(out, cap, (uint64_t)first + warp_base[warp] + (uint32_t)__popc(m & ((1u << lane) - 1u)), row);
}

// count + scan, enqueued: offsets[nblocks] is the total once the stream reaches it
template <class F>
int wc_count(spb_ctx* ctx, DeviceState& d, const F& f, uint64_t lo, uint64_t hi, uint32_t* counts, uint32_t* offsets, void* tmp, size_t tmp_bytes) {
  const unsigned blocks = nblk(hi - lo, kWcRows);
  SPB_TRY(launch(ctx, d.stream, blocks, kWcRows, 0, wc_count_kernel<F>, f, lo, hi, counts));
  SPB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, offsets, (int)blocks + 1, d.stream));
  return 0;
}
template <class F>
int wc_scatter(spb_ctx* ctx, DeviceState& d, const F& f, uint64_t lo, uint64_t hi, const uint32_t* offsets, uint64_t cap, uint32_t* out) {
  return launch(ctx, d.stream, nblk(hi - lo, kWcRows), kWcRows, 0, wc_scatter_kernel<F>, f, lo, hi, offsets, cap, out);
}

size_t scan_bytes(DeviceState& d, uint64_t items) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)items, d.stream);
  return b ? b : 16;
}

// one full compaction of f over [lo, hi) into the caller's host arrays, through the context slots "wc_*"
template <class F>
int compact_rows(spb_ctx* ctx, DeviceState& d, const F& f, uint64_t lo, uint64_t hi, uint32_t cap, uint32_t* rows_out, uint64_t* total_out) {
  const uint64_t blocks = nblk(hi - lo, kWcRows);
  uint32_t* counts = (uint32_t*)slot(ctx, d, "wc_counts", (2 * blocks + 2) * 4);
  uint32_t* out = (uint32_t*)slot(ctx, d, "wc_out", ((size_t)cap + 1) * 4);
  const size_t tmp_bytes = scan_bytes(d, blocks + 1);
  void* tmp = slot(ctx, d, "wc_tmp", tmp_bytes);
  if (!counts || !out || !tmp) return SPB_ERR_OOM;
  uint32_t* offsets = counts + blocks + 1;
  SPB_CUDA(ctx, cudaMemsetAsync(counts + blocks, 0, 4, d.stream));
  SPB_TRY(wc_count(ctx, d, f, lo, hi, counts, offsets, tmp, tmp_bytes));
  SPB_TRY(wc_scatter(ctx, d, f, lo, hi, offsets, cap, out));
  uint32_t total = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&total, offsets + blocks, 4, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  const uint64_t m = total < cap ? total : cap;
  if (m) {
    SPB_CUDA(ctx, cudaMemcpyAsync(rows_out, out, m * 4, cudaMemcpyDeviceToHost, d.stream));
    SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  }
  *total_out = total;
  return 0;
}

}  // namespace

extern "C" {

int spb_nonzero_rows_dev(spb_ctx* ctx, const spb_fr* d_values, uint64_t lo, uint64_t hi, uint32_t cap, uint32_t* rows_out, uint64_t* total_out) {
  if (!ctx || !total_out || (hi > lo && (!d_values || (cap && !rows_out)))) return SPB_ERR_ARG;
  *total_out = 0;
  if (hi <= lo) return 0;
  if (hi > 0xffffffffull) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  return compact_rows(ctx, d, NonzeroFlag{(const Fr*)d_values}, lo, hi, cap, rows_out, total_out);
}

int spb_lookup_missing_rows_dev(spb_ctx* ctx, const spb_fr* d_input, const spb_fr* d_table, size_t usable, uint32_t cap, uint32_t* rows_out, uint64_t* total_out) {
  if (!ctx || !total_out || (usable && (!d_input || !d_table || (cap && !rows_out)))) return SPB_ERR_ARG;
  *total_out = 0;
  if (!usable) return 0;
  if (usable >= 0x7fffffffull) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  LookupWork w;
  SPB_TRY(lookup_work(ctx, d, usable, &w));
  SPB_TRY(sort_canonical(ctx, d, w, (const Fr*)d_table, w.stb, usable));
  return compact_rows(ctx, d, MissingFlag{(const Fr*)d_input, w.stb, usable}, 0, usable, cap, rows_out, total_out);
}

int spb_copy_mismatches_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_values, const spb_fr* const* d_sigma, uint32_t n_cols, size_t usable, uint32_t cap,
                            uint32_t* cells_out, uint64_t* totals_out) {
  if (!ctx || (n_cols && (!d_values || !d_sigma || !totals_out)) || (n_cols && usable && cap && !cells_out)) return SPB_ERR_ARG;
  for (uint32_t c = 0; c < n_cols; c++) {
    if (!d_values[c] || !d_sigma[c]) return SPB_ERR_ARG;
    totals_out[c] = 0;
  }
  if (!n_cols || !usable) return 0;
  if (k < 1 || k > SPB_FR_S || usable > (1ull << k)) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  // tables (witness.cuh SigmaTables), then the value pointers: one upload
  std::vector<Fr> tab((size_t)3 * n_cols + 2 * k);
  sigma_tables_fill(tab.data(), k, n_cols, fr_delta(), fr_root_of_unity(k));
  const uint64_t blocks = nblk(usable, kWcRows);
  const size_t tab_bytes = tab.size() * 32, ptr_bytes = (size_t)n_cols * sizeof(void*);
  char* dtab = (char*)slot(ctx, d, "wc_tables", tab_bytes + ptr_bytes + 8);
  uint32_t* counts = (uint32_t*)slot(ctx, d, "wc_counts", (size_t)n_cols * (2 * blocks + 2) * 4);
  uint32_t* out = (uint32_t*)slot(ctx, d, "wc_out", ((size_t)n_cols * cap + 1) * 16);
  const size_t tmp_bytes = scan_bytes(d, blocks + 1);
  void* tmp = slot(ctx, d, "wc_tmp", tmp_bytes);
  if (!dtab || !counts || !out || !tmp) return SPB_ERR_OOM;
  unsigned long long* bad = (unsigned long long*)(dtab + tab_bytes + ptr_bytes);
  SPB_CUDA(ctx, cudaMemcpyAsync(dtab, tab.data(), tab_bytes, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(dtab + tab_bytes, d_values, ptr_bytes, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemsetAsync(bad, 0xff, 8, d.stream));
  CopyArgs a;
  a.t = sigma_tables_bind((const Fr*)dtab, k, n_cols);
  a.values = (const Fr* const*)(dtab + tab_bytes);
  a.usable = usable;
  for (uint32_t c = 0; c < n_cols; c++) {
    a.sigma = (const Fr*)d_sigma[c]; a.c = c;
    uint32_t* cc = counts + (size_t)c * (2 * blocks + 2), *offsets = cc + blocks + 1;
    SPB_CUDA(ctx, cudaMemsetAsync(cc + blocks, 0, 4, d.stream));
    SPB_TRY(wc_count(ctx, d, CopyFlag{a, bad}, 0, usable, cc, offsets, tmp, tmp_bytes));
    SPB_TRY(wc_scatter(ctx, d, CopyFlag{a, bad}, 0, usable, offsets, cap, out + (size_t)c * cap * 4));
  }
  std::vector<uint32_t> totals(n_cols);
  for (uint32_t c = 0; c < n_cols; c++)
    SPB_CUDA(ctx, cudaMemcpyAsync(&totals[c], counts + (size_t)c * (2 * blocks + 2) + 2 * blocks + 1, 4, cudaMemcpyDeviceToHost, d.stream));
  unsigned long long hbad = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  if (hbad != ~0ull)
    return set_error(ctx, SPB_ERR_DATA, "copy check: sigma of permutation column %u, row %u labels no usable cell (a malformed proving key)", (unsigned)(hbad >> 32),
                     (unsigned)(hbad & 0xffffffffu));
  for (uint32_t c = 0; c < n_cols; c++) {
    totals_out[c] = totals[c];
    const uint64_t m = totals[c] < cap ? totals[c] : cap;
    if (m) SPB_CUDA(ctx, cudaMemcpyAsync(cells_out + (size_t)c * cap * 4, out + (size_t)c * cap * 4, m * 16, cudaMemcpyDeviceToHost, d.stream));
  }
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

int spb_fr_first_noncanonical_dev(spb_ctx* ctx, const spb_fr* d_elems, size_t n, uint64_t* first_out) {
  if (!ctx || !first_out || (n && !d_elems)) return SPB_ERR_ARG;
  *first_out = n;
  if (!n) return 0;
  SPB_ENTER(ctx);
  unsigned long long* first = (unsigned long long*)slot(ctx, d, "kc_first", sizeof(unsigned long long));
  if (!first) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaMemsetAsync(first, 0xff, sizeof(unsigned long long), d.stream));
  SPB_TRY(first_bad_launch(ctx, d, FrBad{(const Fr*)d_elems}, n, first));
  unsigned long long h = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&h, first, sizeof h, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  *first_out = h < n ? (uint64_t)h : (uint64_t)n;
  return 0;
}

int spb_sigma_check_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_sigma, uint32_t n_cols, size_t usable, uint32_t cap, uint32_t* rows_out,
                        uint64_t* totals_out) {
  if (!ctx || (n_cols && (!d_sigma || !totals_out || (cap && !rows_out)))) return SPB_ERR_ARG;
  for (uint32_t c = 0; c < n_cols; c++) {
    if (!d_sigma[c]) return SPB_ERR_ARG;
    totals_out[3 * c] = totals_out[3 * c + 1] = totals_out[3 * c + 2] = 0;
  }
  if (!n_cols) return 0;
  if (k < 1 || k > SPB_FR_S || usable > (1ull << k)) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  const uint64_t n = 1ull << k, wpc = (n + 31) / 32, blocks = nblk(n, kWcRows), per = 2 * blocks + 2, kinds = 3ull * n_cols;
  std::vector<Fr> tab((size_t)3 * n_cols + 2 * k);
  sigma_tables_fill(tab.data(), k, n_cols, fr_delta(), fr_root_of_unity(k));
  const size_t tab_bytes = tab.size() * 32, map_bytes = (size_t)n_cols * wpc * 4;
  Fr* dtab = (Fr*)slot(ctx, d, "wc_tables", tab_bytes);
  uint32_t* maps = (uint32_t*)slot(ctx, d, "kc_maps", 2 * map_bytes);
  uint32_t* counts = (uint32_t*)slot(ctx, d, "wc_counts", kinds * per * 4);
  uint32_t* out = (uint32_t*)slot(ctx, d, "wc_out", (kinds * cap + 1) * 4);
  const size_t tmp_bytes = scan_bytes(d, blocks + 1);
  void* tmp = slot(ctx, d, "wc_tmp", tmp_bytes);
  if (!dtab || !maps || !counts || !out || !tmp) return SPB_ERR_OOM;
  uint32_t* hit = maps, *bad = maps + (size_t)n_cols * wpc;
  SPB_CUDA(ctx, cudaMemcpyAsync(dtab, tab.data(), tab_bytes, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemsetAsync(hit, 0, map_bytes, d.stream));
  const SigmaTables t = sigma_tables_bind(dtab, k, n_cols);
  for (uint32_t c = 0; c < n_cols; c++)
    SPB_TRY(launch(ctx, d.stream, (unsigned)blocks, kWcRows, 0, sigma_mark_kernel, t, (const Fr*)d_sigma[c], c, n, (uint64_t)usable, wpc, hit, bad));
  // kind q of column c: rows [lo, hi) of `bad` set (q = 0, 1) or of `hit` clear (q = 2)
  std::vector<uint64_t> lo(kinds), hi(kinds), nb(kinds);
  for (uint32_t c = 0; c < n_cols; c++) {
    for (uint32_t q = 0; q < 3; q++) {
      const uint64_t j = 3ull * c + q;
      lo[j] = q == 1 ? usable : 0; hi[j] = q == 0 ? usable : n; nb[j] = nblk(hi[j] - lo[j], kWcRows);
      if (hi[j] <= lo[j]) continue;
      const MapFlag f{q == 2 ? hit : bad, wpc, c, q == 2 ? 0u : 1u};
      uint32_t* cc = counts + j * per, *offsets = cc + nb[j] + 1;
      SPB_CUDA(ctx, cudaMemsetAsync(cc + nb[j], 0, 4, d.stream));
      SPB_TRY(wc_count(ctx, d, f, lo[j], hi[j], cc, offsets, tmp, tmp_bytes));
      SPB_TRY(wc_scatter(ctx, d, f, lo[j], hi[j], offsets, cap, out + j * cap));
    }
  }
  std::vector<uint32_t> totals(kinds, 0);
  for (uint64_t j = 0; j < kinds; j++)
    if (hi[j] > lo[j]) SPB_CUDA(ctx, cudaMemcpyAsync(&totals[j], counts + j * per + 2 * nb[j] + 1, 4, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  for (uint64_t j = 0; j < kinds; j++) {
    totals_out[j] = totals[j];
    const uint64_t m = totals[j] < cap ? totals[j] : cap;
    if (m) SPB_CUDA(ctx, cudaMemcpyAsync(rows_out + j * cap, out + j * cap, m * 4, cudaMemcpyDeviceToHost, d.stream));
  }
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

}  // extern "C"
