// Host build of the witness check's device bodies (tests/test_witness_check_cpu.py): hostemu.cpp, included whole, plus the
// sigma decode, the copy check row, the lookup membership search and the failing-row compaction of witness.cu, run serially.
#include "hostemu.cpp"
#include "../../spectre_b200/csrc/witness.cuh"
#include <algorithm>

namespace {
std::vector<Fr> sigma_tables(uint32_t k, uint32_t n_cols) {
  constexpr uint32_t delta[8] = SPB_FR_DELTA_MONT, root[8] = SPB_FR_ROOT_OF_UNITY_MONT;
  Fr omega = fr_macro(root);
  for (uint32_t i = k; i < SPB_FR_S; i++) omega = fp_sqr(omega);
  std::vector<Fr> tab((size_t)3 * n_cols + 2 * k + 1);
  sigma_tables_fill(tab.data(), k, n_cols, fr_macro(delta), omega);
  return tab;
}
}  // namespace

extern "C" {
// ok[i] = sigma_decode(sigma[i]) succeeded, (cols[i], rows[i]) = the cell it labels
void he_sigma_decode(const Fr* sigma, uint64_t count, uint32_t k, uint32_t n_cols, uint32_t* cols, uint64_t* rows, uint8_t* ok) {
  std::vector<Fr> tab = sigma_tables(k, n_cols);
  const SigmaTables t = sigma_tables_bind(tab.data(), k, n_cols);
  for (uint64_t i = 0; i < count; i++) { cols[i] = 0; rows[i] = 0; ok[i] = sigma_decode(t, sigma[i], cols + i, rows + i) ? 1 : 0; }
}
// copy_check_row for rows [0, usable) of permutation column c: rc[i] and the cell (cols[i], rows[i]) sigma_c[i] labels
void he_copy_check(uint32_t k, const Fr* const* values, const Fr* const* sigma, uint32_t n_cols, uint32_t c, uint64_t usable, int32_t* rc, uint32_t* cols,
                   uint64_t* rows) {
  std::vector<Fr> tab = sigma_tables(k, n_cols);
  CopyArgs a;
  a.t = sigma_tables_bind(tab.data(), k, n_cols); a.values = values; a.sigma = sigma[c]; a.c = c; a.usable = usable;
  for (uint64_t i = 0; i < usable; i++) { cols[i] = c; rows[i] = i; rc[i] = copy_check_row(a, i, cols + i, rows + i); }
}
// missing[i] = wc_lookup_missing(input[i]) against the first `rows` table values, sorted here by canonical value
void he_lookup_missing(const Fr* input, const Fr* table, uint64_t rows, uint8_t* missing) {
  std::vector<Fr> sorted(rows);
  for (uint64_t j = 0; j < rows; j++) sorted[j] = fp_from_mont(table[j]);
  std::sort(sorted.begin(), sorted.end(), [](const Fr& x, const Fr& y) { return wc_cmp(x, y) < 0; });
  for (uint64_t i = 0; i < rows; i++) missing[i] = wc_lookup_missing(sorted.data(), rows, input[i]) ? 1 : 0;
}
// the compaction of witness.cu over [lo, hi) with flags[r - lo]: per-block counts, their exclusive scan, then each block that
// has flagged rows and starts below cap stores its rows in order through wc_store. Returns the total.
uint64_t he_compact(const uint8_t* flags, uint64_t lo, uint64_t hi, uint64_t cap, uint32_t* rows_out) {
  const uint64_t blocks = (hi - lo + kWcRows - 1) / kWcRows;
  std::vector<uint32_t> offsets(blocks + 1, 0);
  for (uint64_t b = 0; b < blocks; b++) {
    uint32_t count = 0;
    for (uint64_t r = lo + b * kWcRows; r < hi && r < lo + (b + 1) * kWcRows; r++) count += flags[r - lo];
    offsets[b + 1] = offsets[b] + count;
  }
  for (uint64_t b = 0; b < blocks; b++) {
    if (offsets[b + 1] == offsets[b] || offsets[b] >= cap) continue;
    uint64_t pos = offsets[b];
    for (uint64_t r = lo + b * kWcRows; r < hi && r < lo + (b + 1) * kWcRows; r++) if (flags[r - lo]) wc_store(rows_out, cap, pos++, r);
  }
  return offsets[blocks];
}
}
