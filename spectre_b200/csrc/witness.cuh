// Per-row bodies of the witness check (witness.cu), written host+device so that tests/hostemu/witness.cpp runs the very same
// code serially on the CPU. What each entry point computes: witness.cu and include/spectre_b200.h.
#pragma once
#include "ntt.cuh"

namespace spb {

// ---- failing-row compaction: a block of kWcRows rows counts its flagged rows, an exclusive scan of the block counts gives
// each block its first output slot, and the block writes the rows it flagged in ascending order from there. Only slots < cap
// are written, so the output holds the first `cap` flagged rows of the whole range.
static const int kWcRows = 256;

SPB_HD void wc_store(uint32_t* rows_out, uint64_t cap, uint64_t pos, uint64_t row) {
  if (pos < cap) rows_out[pos] = (uint32_t)row;
}

// ---- lookup membership: is the input value missing from the table's values sorted by canonical integer? ----
SPB_HD int wc_cmp(const Fr& a, const Fr& b) {
  for (int i = 7; i >= 0; i--) { if (a.l[i] != b.l[i]) return a.l[i] < b.l[i] ? -1 : 1; }
  return 0;
}
// input: Montgomery form; sorted_table: canonical values, ascending, `rows` of them
SPB_HD bool wc_lookup_missing(const Fr* sorted_table, uint64_t rows, const Fr& input) {
  const Fr v = fp_from_mont(input);
  uint64_t lo = 0, hi = rows;
  while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (wc_cmp(ntt_ldg(sorted_table + mid), v) < 0) lo = mid + 1; else hi = mid; }
  return lo >= rows || wc_cmp(ntt_ldg(sorted_table + lo), v) != 0;
}

// ---- sigma decode: sigma = delta^c * omega^i labels the cell (column c, row i) ----
// The tables (Montgomery form) a decode reads, n_cols = C columns, omega a primitive 2^k-th root of unity:
struct SigmaTables {
  const Fr* delta_n;         // C: delta^(c n). delta = 7^(2^28) has odd order, so sigma^n = delta^(c n) names the column
  const Fr* delta_inv;       // C: delta^-c
  const Fr* delta_pow;       // C: delta^c (the fixed-point test)
  const Fr* omega_pow2;      // k: omega^(2^j)
  const Fr* omega_inv_pow2;  // k: omega^-(2^j)
  Fr minus_one;
  uint32_t k, n_cols;
};

// Host: the table array behind SigmaTables, 3 C + 2 k elements (delta_n | delta_inv | delta_pow | omega_pow2 | omega_inv_pow2),
// from delta and omega (Montgomery form); sigma_tables_bind points SigmaTables into a copy of it at `tab`.
inline void sigma_tables_fill(Fr* tab, uint32_t k, uint32_t n_cols, const Fr& delta, const Fr& omega) {
  Fr* delta_n = tab, *delta_inv = tab + n_cols, *delta_pow = tab + 2 * n_cols, *om = tab + 3 * n_cols, *om_inv = om + k;
  const Fr delta_to_n = fp_pow_u64(delta, 1ull << k), delta_inverse = fp_inv(delta);
  Fr p = fp_one<FrParams>(), pn = p, pi = p;
  for (uint32_t c = 0; c < n_cols; c++) {
    delta_pow[c] = p; delta_n[c] = pn; delta_inv[c] = pi;
    p = fp_mul(p, delta); pn = fp_mul(pn, delta_to_n); pi = fp_mul(pi, delta_inverse);
  }
  Fr w = omega, wi = fp_inv(omega);
  for (uint32_t j = 0; j < k; j++) { om[j] = w; om_inv[j] = wi; w = fp_sqr(w); wi = fp_sqr(wi); }
}
inline SigmaTables sigma_tables_bind(const Fr* tab, uint32_t k, uint32_t n_cols) {
  SigmaTables t;
  t.delta_n = tab; t.delta_inv = tab + n_cols; t.delta_pow = tab + 2 * n_cols; t.omega_pow2 = tab + 3 * n_cols; t.omega_inv_pow2 = tab + 3 * n_cols + k;
  t.minus_one = fp_sub(fp_zero<FrParams>(), fp_one<FrParams>());
  t.k = k; t.n_cols = n_cols;
  return t;
}

// delta^c * omega^i, the label of cell (c, i): k products at most
SPB_HD Fr sigma_label(const SigmaTables& t, uint32_t c, uint64_t i) {
  Fr x = ntt_ldg(t.delta_pow + c);
  for (uint32_t j = 0; j < t.k; j++) if ((i >> j) & 1) x = fp_mul(x, ntt_ldg(t.omega_pow2 + j));
  return x;
}

// (col, row) of the cell `sigma` labels. Returns false when it labels no cell of the C columns. The column from sigma^n (k
// squarings, C comparisons); then x = sigma delta^-c has order dividing 2^k, x = omega^i, and i is recovered bit by bit
// (2-adic Pohlig-Hellman): with the bits below j removed, y = omega^(i - e) has (i - e) a multiple of 2^j, and
// y^(2^(k-1-j)) = (-1)^(bit j of i). k(k-1)/2 squarings in all.
SPB_HD bool sigma_decode(const SigmaTables& t, const Fr& sigma, uint32_t* col, uint64_t* row) {
  Fr s = sigma;
  for (uint32_t j = 0; j < t.k; j++) s = fp_sqr(s);
  uint32_t c = t.n_cols;
  for (uint32_t q = 0; q < t.n_cols; q++) if (fp_eq(s, ntt_ldg(t.delta_n + q))) { c = q; break; }
  if (c == t.n_cols) return false;
  Fr y = fp_mul(sigma, ntt_ldg(t.delta_inv + c));
  uint64_t i = 0;
  for (uint32_t j = 0; j < t.k; j++) {
    Fr z = y;
    for (uint32_t s2 = j + 1; s2 < t.k; s2++) z = fp_sqr(z);
    if (fp_eq(z, t.minus_one)) { i |= 1ull << j; y = fp_mul(y, ntt_ldg(t.omega_inv_pow2 + j)); }   // z is 1 or -1: x^(2^k) = 1
  }
  *col = c; *row = i;
  return true;
}

// The copy constraint of cell (c, i), i < usable: 0 when it holds, 1 when the value differs from the value of the cell
// sigma_c[i] labels (*col, *row), 2 when sigma_c[i] labels no usable cell (a malformed key). A cell whose sigma is its own
// label is a fixed point and needs no decode.
struct CopyArgs {
  SigmaTables t;
  const Fr* const* values;   // C columns
  const Fr* sigma;           // of the column checked
  uint32_t c;
  uint64_t usable;
};
SPB_HD int copy_check_row(const CopyArgs& a, uint64_t i, uint32_t* col, uint64_t* row) {
  const Fr s = ntt_ldg(a.sigma + i);
  if (fp_eq(s, sigma_label(a.t, a.c, i))) { *col = a.c; *row = i; return 0; }
  if (!sigma_decode(a.t, s, col, row) || *row >= a.usable) return 2;
  return fp_eq(ntt_ldg(a.values[a.c] + i), ntt_ldg(a.values[*col] + *row)) ? 0 : 1;
}

// ---- proving-key check (spb_fr_first_noncanonical_dev, spb_sigma_check_dev) ----
// an element whose stored limbs are not below r: halo2curves' RawBytes read refuses it
SPB_HD bool fr_noncanonical(const Fr& a) { return !fp_is_canonical(a); }

// The entry s = sigma_c[i] of a key. Returns whether it labels a cell (*col, *row) of the n_cols columns; a fixed point (its own
// label) needs no decode, and a non-canonical s labels nothing (the arithmetic of a decode assumes reduced inputs). *bad: the
// entry fails spb_sigma_check_dev's kind 0 (i < usable and it labels no usable cell) or kind 1 (i >= usable and it is not a
// fixed point).
SPB_HD bool sigma_check_entry(const SigmaTables& t, uint32_t c, uint64_t i, const Fr& s, uint64_t usable, uint32_t* col, uint64_t* row, bool* bad) {
  if (fp_eq(s, sigma_label(t, c, i))) { *col = c; *row = i; *bad = false; return true; }
  const bool ok = fp_is_canonical(s) && sigma_decode(t, s, col, row);
  *bad = i >= usable || !ok || *row >= usable;
  return ok;
}
// bit of cell (c, i) in a map of n_cols columns, words_per_col 32-bit words each
SPB_HD uint64_t sigma_map_word(uint64_t words_per_col, uint32_t c, uint64_t i) { return c * words_per_col + (i >> 5); }
SPB_HD uint32_t sigma_map_bit(uint64_t i) { return 1u << (i & 31u); }

}  // namespace spb
