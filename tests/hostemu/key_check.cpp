// Host build of the proving-key check's device bodies (tests/test_key_check_cpu.py): witness.cpp, included whole (the sigma
// tables and the failing-row compaction), plus the canonical test of spb_fr_first_noncanonical_dev and the sigma pass of
// spb_sigma_check_dev, run serially.
#include "witness.cpp"

extern "C" {
// the first i < n with fr_noncanonical(a[i]), or n
uint64_t he_fr_first_noncanonical(const Fr* a, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) if (fr_noncanonical(a[i])) return i;
  return n;
}
// spb_sigma_check_dev on host arrays: each entry through sigma_check_entry, its cell marked in `hit` and its own in `bad` (the
// same word layout as the device maps), then the compaction of each kind; same outputs as the device call
void he_sigma_check(uint32_t k, const Fr* const* sigma, uint32_t n_cols, uint64_t usable, uint32_t cap, uint32_t* rows_out, uint64_t* totals_out) {
  const uint64_t n = 1ull << k, wpc = (n + 31) / 32;
  std::vector<Fr> tab = sigma_tables(k, n_cols);
  const SigmaTables t = sigma_tables_bind(tab.data(), k, n_cols);
  std::vector<uint32_t> hit(n_cols * wpc, 0), bad(n_cols * wpc, 0);
  for (uint32_t c = 0; c < n_cols; c++)
    for (uint64_t i = 0; i < n; i++) {
      uint32_t col; uint64_t row; bool b;
      if (sigma_check_entry(t, c, i, sigma[c][i], usable, &col, &row, &b)) hit[sigma_map_word(wpc, col, row)] |= sigma_map_bit(row);
      if (b) bad[sigma_map_word(wpc, c, i)] |= sigma_map_bit(i);
    }
  std::vector<uint8_t> flags(n);
  for (uint32_t c = 0; c < n_cols; c++)
    for (uint32_t q = 0; q < 3; q++) {
      const uint64_t lo = q == 1 ? usable : 0, hi = q == 0 ? usable : n, j = 3ull * c + q;
      const std::vector<uint32_t>& map = q == 2 ? hit : bad;
      for (uint64_t i = lo; i < hi; i++) flags[i - lo] = (((map[sigma_map_word(wpc, c, i)] >> (i & 31u)) & 1u) == (q == 2 ? 0u : 1u)) ? 1 : 0;
      totals_out[j] = hi > lo ? he_compact(flags.data(), lo, hi, cap, rows_out + j * cap) : 0;
    }
}
}
