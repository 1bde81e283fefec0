// Per-row bodies of the quotient-numerator kernels (quotient.cu) and of the argument-prover term kernels (plonk.cu),
// written host+device so that tests/hostemu runs the very same code serially on the CPU against the oracle
// (tests/test_hostemu_quotient.py). What each computes and which upstream routine it replaces: quotient.cu, plonk.cu.
#pragma once
#include "ntt.cuh"

namespace spb {

struct GraphArgs {
  const uint32_t* prog; uint32_t ncalc;
  const Fr* constants; const int32_t* rotations;
  const Fr* const* fixed; const Fr* const* advice; const Fr* const* instance;
  const Fr* scalars;   // [beta, gamma, theta, y, challenges...]
  Fr* values; Fr* scratch; uint64_t size; int32_t rot_scale;
  uint64_t row_lo, row_hi;   // this launch's extended rows [row_lo, row_hi): a row-range shard of a multi-device context
};

SPB_HD uint64_t rotation_idx(uint64_t idx, int32_t rot, int32_t rot_scale, uint64_t size) {
#if defined(__CUDA_ARCH__)
  // extended domains are powers of two (the entry points of quotient.cu reject anything else): wrap with a mask -- two's complement
  // makes it right for negative rotations too -- instead of a 64-bit remainder per column read
  return (idx + (uint64_t)((long long)rot * rot_scale)) & (size - 1);
#endif
  long long v = ((long long)idx + (long long)rot * rot_scale) % (long long)size;
  if (v < 0) v += (long long)size;
  return (uint64_t)v;
}

SPB_HD Fr graph_src(const GraphArgs& a, const uint32_t* w, uint64_t row, uint32_t slot, uint32_t nslots, const Fr& previous) {
  const uint32_t kind = w[0], idx = w[1] & 0xffffu, rot = w[1] >> 16;
  switch (kind) {
    case 0: return ntt_ldg(a.constants + idx);
    case 1: return a.scratch[(uint64_t)idx * nslots + slot];
    case 2: return ntt_ldg(a.fixed[idx] + rotation_idx(row, a.rotations[rot], a.rot_scale, a.size));
    case 3: return ntt_ldg(a.advice[idx] + rotation_idx(row, a.rotations[rot], a.rot_scale, a.size));
    case 4: return ntt_ldg(a.instance[idx] + rotation_idx(row, a.rotations[rot], a.rot_scale, a.size));
    case 5: return ntt_ldg(a.scalars + 4 + idx);
    case 6: return ntt_ldg(a.scalars + 0);
    case 7: return ntt_ldg(a.scalars + 1);
    case 8: return ntt_ldg(a.scalars + 2);
    case 9: return ntt_ldg(a.scalars + 3);
    default: return previous;
  }
}

// GraphEvaluator::evaluate for one row; intermediates live at scratch[intermediate * nslots + slot]
SPB_HD void graph_evaluate_row(const GraphArgs& a, uint64_t row, uint32_t slot, uint32_t nslots) {
  const Fr previous = a.values[row];
  const uint32_t* w = a.prog;
  Fr last = fp_zero<FrParams>();
  for (uint32_t c = 0; c < a.ncalc; c++) {
    const uint32_t op = w[0] & 0xffu, nparts = w[0] >> 8, target = w[1];
    Fr r;
    if (op <= 2) {
      Fr x = graph_src(a, w + 2, row, slot, nslots, previous), y = graph_src(a, w + 4, row, slot, nslots, previous);
      r = op == 0 ? fp_add(x, y) : op == 1 ? fp_sub(x, y) : fp_mul(x, y);
      w += 6;
    } else if (op == 6) {
      Fr acc = graph_src(a, w + 2, row, slot, nslots, previous), factor = graph_src(a, w + 4, row, slot, nslots, previous);
      for (uint32_t p = 0; p < nparts; p++) acc = fp_add(fp_mul(acc, factor), graph_src(a, w + 6 + 2 * p, row, slot, nslots, previous));
      r = acc; w += 6 + 2 * nparts;
    } else {
      Fr x = graph_src(a, w + 2, row, slot, nslots, previous);
      r = op == 3 ? fp_sqr(x) : op == 4 ? fp_dbl(x) : op == 5 ? fp_neg(x) : x;
      w += 4;
    }
    a.scratch[(uint64_t)target * nslots + slot] = r;
    last = r;
  }
  a.values[row] = last;
}

struct PermArgs {
  Fr* values; uint64_t size; int32_t rot_scale, last_rotation; uint32_t n_sets, chunk_len, n_cols;
  uint64_t row_lo, row_hi;   // row-range shard
  const Fr* omega_pow;       // extended_omega^j, j < 256 (device table): omega^idx = omega^(idx & ~255) * omega_pow[idx & 255]
  const Fr* const* z; const Fr* const* col_values; const Fr* const* sigma;
  const Fr* l0; const Fr* l_last; const Fr* l_active;
  // X at row idx is g * extended_omega^idx: delta_start = beta * g (g = zeta on the whole extended coset, zeta extended_omega^j
  // with extended_omega = omega on its coset part j)
  Fr beta, gamma, y, delta_start, delta, extended_omega;
};

// omega_idx = extended_omega^idx (the kernel derives it from one power per block and the 256-entry table)
SPB_HD void permutation_constraints_row(const PermArgs& a, uint64_t idx, const Fr& omega_idx) {
  const uint64_t r_next = rotation_idx(idx, 1, a.rot_scale, a.size), r_last = rotation_idx(idx, a.last_rotation, a.rot_scale, a.size);
  const Fr one = fp_one<FrParams>();
  Fr v = ntt_ld_stream(a.values + idx);
  const Fr l0 = ntt_ldg(a.l0 + idx), l_last = ntt_ldg(a.l_last + idx), l_active = ntt_ldg(a.l_active + idx);
  v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(one, ntt_ldg(a.z[0] + idx)), l0));
  { Fr zl = ntt_ldg(a.z[a.n_sets - 1] + idx); v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(fp_sqr(zl), zl), l_last)); }
  for (uint32_t s = 1; s < a.n_sets; s++)
    v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(ntt_ldg(a.z[s] + idx), ntt_ldg(a.z[s - 1] + r_last)), l0));
  Fr current_delta = fp_mul(a.delta_start, omega_idx);
  for (uint32_t s = 0; s < a.n_sets; s++) {
    const uint32_t lo = s * a.chunk_len, hi = lo + a.chunk_len < a.n_cols ? lo + a.chunk_len : a.n_cols;
    Fr left = ntt_ldg(a.z[s] + r_next), right = ntt_ldg(a.z[s] + idx);
    for (uint32_t c = lo; c < hi; c++) {
      Fr val = ntt_ldg(a.col_values[c] + idx);
      left = fp_mul(left, fp_add(fp_add(val, fp_mul(a.beta, ntt_ldg(a.sigma[c] + idx))), a.gamma));
      right = fp_mul(right, fp_add(fp_add(val, current_delta), a.gamma));
      current_delta = fp_mul(current_delta, a.delta);
    }
    v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(left, right), l_active));
  }
  ntt_stg(a.values + idx, v);
}

struct LookupArgs {
  Fr* values; uint64_t size; int32_t rot_scale;
  uint64_t row_lo, row_hi;   // row-range shard
  const Fr* product; const Fr* permuted_input; const Fr* permuted_table; const Fr* table_value;
  const Fr* l0; const Fr* l_last; const Fr* l_active;
  Fr beta, gamma, y;
};

SPB_HD void lookup_constraints_row(const LookupArgs& a, uint64_t idx) {
  const uint64_t r_next = rotation_idx(idx, 1, a.rot_scale, a.size), r_prev = rotation_idx(idx, -1, a.rot_scale, a.size);
  const Fr one = fp_one<FrParams>();
  const Fr l0 = ntt_ldg(a.l0 + idx), l_last = ntt_ldg(a.l_last + idx), l_active = ntt_ldg(a.l_active + idx);
  const Fr a_in = ntt_ldg(a.permuted_input + idx), s_tb = ntt_ldg(a.permuted_table + idx), zp = ntt_ldg(a.product + idx);
  const Fr a_minus_s = fp_sub(a_in, s_tb);
  Fr v = ntt_ld_stream(a.values + idx);
  v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(one, zp), l0));
  v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(fp_sqr(zp), zp), l_last));
  Fr lhs = fp_mul(fp_mul(ntt_ldg(a.product + r_next), fp_add(a_in, a.beta)), fp_add(s_tb, a.gamma));
  v = fp_add(fp_mul(v, a.y), fp_mul(fp_sub(lhs, fp_mul(zp, ntt_ldg(a.table_value + idx))), l_active));
  v = fp_add(fp_mul(v, a.y), fp_mul(a_minus_s, l0));
  v = fp_add(fp_mul(v, a.y), fp_mul(fp_mul(a_minus_s, fp_sub(a_in, ntt_ldg(a.permuted_input + r_prev))), l_active));
  ntt_stg(a.values + idx, v);
}

// one row of a coset part back into the extended buffer: row m of part `part` is extended row part + R m
SPB_HD void extended_part_scatter_row(const Fr* part_values, Fr* extended, uint32_t part, uint32_t R, uint64_t m) {
  ntt_stg(extended + part + (uint64_t)R * m, ntt_ld_stream(part_values + m));
}

// ---- argument-prover terms (plonk.cu) --------------------------------------------------------------------------------
const uint32_t kMaxSetCols = 16;   // columns of one permutation set (chunk_len = degree - 2; halo2-lib circuits: 2..7)
struct PermTermArgs {
  const Fr* values[kMaxSetCols];
  const Fr* sigma[kMaxSetCols];
  uint32_t n_cols;
  Fr beta, gamma, delta;
  Fr delta_start;   // beta * delta^first_col
  Fr omega;
};

// num[i] = prod_c (v_c[i] + beta * delta^(first_col + c) * omega^i + gamma),  den[i] = prod_c (v_c[i] + beta * sigma_c[i] + gamma)
SPB_HD void perm_terms_row(const PermTermArgs& a, uint64_t i, const Fr& omega_i, Fr* num, Fr* den) {
  Fr term = fp_mul(a.delta_start, omega_i);
  Fr nu = fp_one<FrParams>(), de = fp_one<FrParams>();
  for (uint32_t c = 0; c < a.n_cols; c++) {
    Fr v = ntt_ld_stream(a.values[c] + i);
    de = fp_mul(de, fp_add(fp_add(fp_mul(a.beta, ntt_ld_stream(a.sigma[c] + i)), a.gamma), v));
    nu = fp_mul(nu, fp_add(fp_add(term, a.gamma), v));
    term = fp_mul(term, a.delta);
  }
  ntt_stg(num + i, nu);
  ntt_stg(den + i, de);
}
// num[i] = (a[i] + beta)(s[i] + gamma),  den[i] = (a'[i] + beta)(s'[i] + gamma)
SPB_HD void lookup_terms_row(const Fr* ci, const Fr* ct, const Fr* pi, const Fr* pt, const Fr& beta, const Fr& gamma, uint64_t i, Fr* num, Fr* den) {
  ntt_stg(num + i, fp_mul(fp_add(ntt_ld_stream(ci + i), beta), fp_add(ntt_ld_stream(ct + i), gamma)));
  ntt_stg(den + i, fp_mul(fp_add(ntt_ld_stream(pi + i), beta), fp_add(ntt_ld_stream(pt + i), gamma)));
}

}  // namespace spb
