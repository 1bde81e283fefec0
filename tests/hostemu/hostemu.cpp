// Host build of the DEVICE arithmetic headers, for CPU-only unit tests (tests/test_hostemu.py).
// Compiled with -DSPB_EMULATE_PTX (the 32-bit-limb PTX carry-chain algorithms, instruction for instruction, with an
// emulated carry flag), without it (the 64-bit host-glue path), and with -DSPB_EMULATE_PTX -DSPB_EMULATE_PTX_TRACE
// (the emulated path recording its carries per call site: tests/arith_corpus.py).
#include "../../spectre_b200/csrc/curve.cuh"
#include <string.h>
using namespace spb;
extern "C" {
void he_fr_mul(Fr* o, const Fr* a, const Fr* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_mul(a[i], b[i]); }
void he_fr_sqr(Fr* o, const Fr* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_sqr(a[i]); }
void he_fq_sqr(Fq* o, const Fq* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_sqr(a[i]); }
void he_fq_mul_sub_mul(Fq* o, const Fq* a, const Fq* b, const Fq* c, const Fq* d, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_mul_sub_mul(a[i], b[i], c[i], d[i]); }
void he_fr_add(Fr* o, const Fr* a, const Fr* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_add(a[i], b[i]); }
void he_fr_sub(Fr* o, const Fr* a, const Fr* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_sub(a[i], b[i]); }
void he_fr_neg(Fr* o, const Fr* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_neg(a[i]); }
void he_fr_inv(Fr* o, const Fr* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_inv(a[i]); }
void he_fq_mul(Fq* o, const Fq* a, const Fq* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_mul(a[i], b[i]); }
void he_fq_add(Fq* o, const Fq* a, const Fq* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_add(a[i], b[i]); }
void he_fq_sub(Fq* o, const Fq* a, const Fq* b, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_sub(a[i], b[i]); }
void he_fq_inv(Fq* o, const Fq* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_inv(a[i]); }
void he_fr_from_mont(Fr* o, const Fr* a, size_t n) { for (size_t i = 0; i < n; i++) o[i] = fp_from_mont(a[i]); }
// acc (XYZZ, starts at identity) += each affine point in order; returns affine
void he_sum_mixed(G1Affine* out, const G1Affine* pts, size_t n) {
  G1Xyzz acc = xyzz_identity();
  for (size_t i = 0; i < n; i++) xyzz_add_mixed(acc, pts[i]);
  *out = xyzz_to_affine(acc);
}
// pairwise tree through the general XYZZ+XYZZ adder
void he_sum_general(G1Affine* out, const G1Affine* pts, size_t n) {
  G1Xyzz acc = xyzz_identity();
  for (size_t i = 0; i < n; i++) { G1Xyzz t = xyzz_from_affine(pts[i]); xyzz_add(acc, t); }
  *out = xyzz_to_affine(acc);
}
void he_mul_u32(G1Affine* out, const G1Affine* p, uint32_t k) { *out = xyzz_to_affine(xyzz_mul_u32(xyzz_from_affine(*p), k)); }
void he_dbl(G1Affine* out, const G1Affine* p) { *out = xyzz_to_affine(xyzz_dbl(xyzz_from_affine(*p))); }
int he_on_curve(const G1Affine* p) { return affine_on_curve(*p) ? 1 : 0; }
void he_jac_roundtrip(G1Affine* out, const G1Affine* p) { G1Jac j = jac_from_affine(*p); G1Xyzz x = xyzz_from_jac(j); *out = jac_to_affine(jac_from_affine(xyzz_to_affine(x))); }
}

// ---- the host twins of the spb_test_* field / curve hooks (capi.cu), same operation codes -------------------------------
namespace {
template <class P> Fp<P> field_op(int op, const Fp<P>& x, const Fp<P>& y) {
  switch (op) {
    case 0: return fp_mul(x, y);
    case 1: return fp_add(x, y);
    case 2: return fp_sub(x, y);
    case 3: return fp_sqr(x);
    case 4: return fp_neg(x);
    case 5: return fp_dbl(x);
    case 6: return fp_inv(x);
    case 7: return fp_to_mont(x);
    case 8: return fp_from_mont(x);
    case 9: { Fp<P> r = fp_zero<P>(); r.l[0] = fp_is_canonical(x) ? 1u : 0u; return r; }
    case 10: return fp_pow(x, y.l);
    default: return fp_pow_u64(x, ((uint64_t)y.l[1] << 32) | y.l[0]);
  }
}
#if defined(SPB_EMULATE_PTX_TRACE)
#define SPB_TRACE_MARK() ptx::trace_mark()
#else
#define SPB_TRACE_MARK() ((void)0)
#endif
template <class P> void field_ops(int op, const Fp256* a, const Fp256* b, Fp256* o, size_t n) {
  for (size_t i = 0; i < n; i++) {
    SPB_TRACE_MARK();
    const Fp<P> x = *(const Fp<P>*)&a[i], y = *(const Fp<P>*)&b[i];
    *(Fp<P>*)&o[i] = field_op<P>(op, x, y);
  }
}
template <class P> void mul_sub_muls(const Fp256* a, const Fp256* b, const Fp256* c, const Fp256* d, Fp256* o, size_t n) {
  for (size_t i = 0; i < n; i++) {
    SPB_TRACE_MARK();
    *(Fp<P>*)&o[i] = fp_mul_sub_mul(*(const Fp<P>*)&a[i], *(const Fp<P>*)&b[i], *(const Fp<P>*)&c[i], *(const Fp<P>*)&d[i]);
  }
}
G1Affine xy(const G1Xyzz& p) { G1Affine r; r.x = p.x; r.y = p.y; return r; }
G1Xyzz curve_test_op(int op, const G1Xyzz& p, const G1Xyzz& q, uint32_t k) {
  G1Xyzz r = p;
  switch (op) {
    case 0: xyzz_add_mixed(r, xy(q)); return r;
    case 1: xyzz_add(r, q); return r;
    case 2: return xyzz_dbl(p);
    case 3: return xyzz_dbl_affine(xy(p));
    case 4: { G1Affine a = xyzz_to_affine(p); r.x = a.x; r.y = a.y; r.zz = fp_zero<FqParams>(); r.zzz = fp_zero<FqParams>(); return r; }
    case 5: return xyzz_mul_u32(p, k);
    default: { r = G1Xyzz{}; r.x.l[0] = (uint32_t)affine_check(xy(p)); return r; }
  }
}
}  // namespace
extern "C" {
// field 0 = Fr, 1 = Fq; op as spb_test_field_op
void he_field_op(int field, int op, const Fp256* a, const Fp256* b, Fp256* o, size_t n) {
  if (field == 0) field_ops<FrParams>(op, a, b, o, n); else field_ops<FqParams>(op, a, b, o, n);
}
void he_field_mul_sub_mul(int field, const Fp256* a, const Fp256* b, const Fp256* c, const Fp256* d, Fp256* o, size_t n) {
  if (field == 0) mul_sub_muls<FrParams>(a, b, c, d, o, n); else mul_sub_muls<FqParams>(a, b, c, d, o, n);
}
// op as spb_test_curve_op: points are XYZZ {x, y, zz, zzz}; an affine operand is the (x, y) of its slot
void he_curve_op(int op, const G1Xyzz* p, const G1Xyzz* q, const uint32_t* k, G1Xyzz* o, size_t n) {
  for (size_t i = 0; i < n; i++) o[i] = curve_test_op(op, p[i], q[i], k ? k[i] : 0u);
}
#if defined(SPB_EMULATE_PTX_TRACE)
void he_trace_reset() { memset(ptx::g_trace, 0, sizeof ptx::g_trace); }
// the recorded sites, in table order: file, line, instance, instruction name, seen bits (ptx::kTrace*); returns the number written
size_t he_trace_read(const char** files, int32_t* lines, int32_t* seqs, const char** ops, uint32_t* seen, size_t cap) {
  size_t n = 0;
  for (int i = 0; i < ptx::kTraceCap && n < cap; i++) {
    const ptx::TraceSite& s = ptx::g_trace[i];
    if (s.file) { files[n] = s.file; lines[n] = s.line; seqs[n] = s.seq; ops[n] = s.op; seen[n] = s.seen; n++; }
  }
  return n;
}
#endif
}

// ---- MSM pipeline, emulated serially with the same per-thread bodies the CUDA kernels call -----------------
#include "../../spectre_b200/csrc/msm.cuh"
#include <vector>
extern "C" {
// c = 0: library's own geometry choice. precomp = 1: build the 2^(c*j) tables first and use one bucket set.
// Returns the number of sorted entries; *giants = number of chains that took the block path.
uint64_t he_msm(G1Affine* out, const Fr* scalars, const G1Affine* bases, size_t n, uint32_t c, uint32_t L, uint32_t cap, uint32_t* giants, int precomp) {
  if (!c) c = msm_choose_c(n ? n : 1, precomp != 0);
  MsmGeom g = msm_make_geometry(c, precomp != 0, (uint32_t)n);
  if (L) g.L = L;
  std::vector<G1Affine> table;
  const G1Affine* pts = bases;
  if (precomp) {
    table.resize((size_t)g.W * n);
    for (size_t i = 0; i < n; i++) table[i] = bases[i];
    for (uint64_t t = 0; t < n; t++) msm_precompute_thread(t, n, g.c, g.W, table.data());
    pts = table.data();
  }
  uint64_t nb = (uint64_t)g.BW * g.B;
  std::vector<uint32_t> counts(nb + 1, 0), offsets(nb + 1, 0);
  for (uint64_t t = 0; t < n; t++) msm_count_thread(t, n, scalars, g, counts.data());
  uint64_t run = 0;
  for (uint64_t i = 0; i <= nb; i++) { offsets[i] = (uint32_t)run; run += counts[i]; }
  uint64_t M = offsets[nb];
  std::vector<uint32_t> cursor(offsets);
  std::vector<MsmEntry> ent(M + 1);
  for (uint64_t t = 0; t < n; t++) msm_scatter_thread(t, n, scalars, g, cursor.data(), ent.data());
  std::vector<G1Xyzz> buckets(nb);
  memset(buckets.data(), 0xAB, nb * sizeof(G1Xyzz));   // never cleared on the device either: only written buckets may be read
  const uint32_t Leff = msm_effective_chunk(g.L, M);
  uint64_t T = (M + Leff - 1) / Leff;
  std::vector<uint32_t> hk(T + 1, 0x12345678u), tk(T + 1, 0x12345678u), glist(T + 2);
  std::vector<G1Xyzz> head(T + 1), tail(T + 1);
  for (uint64_t t = 0; t < T; t++) msm_accumulate_thread(t, M, g, ent.data(), pts, buckets.data(), hk.data(), head.data(), tk.data(), tail.data());
  uint32_t gcount = 0;
  for (uint64_t t = 0; t < T; t++) msm_stitch_thread(t, T, cap, hk.data(), head.data(), tk.data(), tail.data(), buckets.data(), &gcount, glist.data());
  for (uint32_t gi = 0; gi < gcount; gi++) {  // what msm_giant_kernel does, serially
    uint64_t t0 = glist[gi]; uint32_t key = tk[t0];
    G1Xyzz acc = xyzz_identity();
    for (uint64_t j = t0 + 1; j < T && hk[j] == key; j++) xyzz_add(acc, head[j]);
    xyzz_add(acc, tail[t0]);
    buckets[key] = acc;
  }
  if (giants) *giants = gcount;
  MsmTail tl = msm_tail_shape(g.c);
  uint32_t per = msm_tail_partials(tl);
  std::vector<G1Xyzz> partials((uint64_t)g.BW * per), win(g.BW);
  msm_tail_host(g, offsets.data(), buckets.data(), partials.data());
  for (uint32_t w = 0; w < g.BW; w++) win[w] = msm_tail_finish(g, partials.data() + (uint64_t)w * per);
  *out = xyzz_to_affine(msm_combine_windows(win.data(), g.BW, g.c));
  return M;
}
// ParamsKZG::downsize's g_to_lagrange: the per-thread bodies of the EC inverse-DFT kernels, run serially
void he_g_to_lagrange(G1Affine* out, const G1Affine* g, uint32_t k, const Fr* omega_inv, const Fr* n_inv) {
  const uint64_t n = 1ull << k;
  std::vector<G1Xyzz> p(n);
  for (uint64_t i = 0; i < n; i++) p[i] = xyzz_from_affine(g[i]);
  std::vector<Fr> tw(n / 2 ? n / 2 : 1);
  for (uint64_t i = 0; i < n / 2; i++) tw[i] = fp_pow_u64(*omega_inv, i);
  for (uint64_t half = n / 2; half >= 1; half >>= 1) for (uint64_t t = 0; t < n / 2; t++) ec_ntt_stage_thread(t, n, half, tw.data(), p.data());
  for (uint64_t t = 0; t < n; t++) ec_ntt_finish_thread(t, n, k, *n_inv, p.data(), out);
}
void he_geometry(uint64_t n, int precomp, uint32_t* c, uint32_t* W) { MsmGeom g = msm_make_geometry(msm_choose_c(n, precomp != 0), precomp != 0, 0); *c = g.c; *W = g.W; }
}

// ---- NTT: the kernel's phases run serially (every phase for all tid), single- and multi-device plans -----------------
#include "../../spectre_b200/csrc/ntt.cuh"
namespace {
void run_pass(const NttPassParams& p, const NttLaunch& L) {
  const uint32_t S = 1u << p.s, C = 1u << p.logc, T = L.threads;
  std::vector<uint32_t> smem(L.smem / 4 + 64, 0xdeadbeefu);
  NttSmem sm; sm.bind(smem.data(), S, C);
  for (uint32_t tid = 0; tid < T; tid++) ntt_phase_twiddles(p, sm, tid, T);
  for (uint64_t tile_it = 0; tile_it < p.ntiles; tile_it++) {
    NttTile t = ntt_tile_coords(p, tile_it + p.tile_base);
    for (uint32_t tid = 0; tid < T; tid++) ntt_phase_load(p, sm, t, tid, T);
    uint32_t m = S >> 1;
    if (p.s & 1) { for (uint32_t tid = 0; tid < T; tid++) ntt_phase_radix2(p, sm, m, tid, T); m >>= 1; }
    for (; m >= 2; m >>= 2) for (uint32_t tid = 0; tid < T; tid++) ntt_phase_radix4(p, sm, m, tid, T);
    for (uint32_t tid = 0; tid < T; tid++) ntt_phase_store(p, sm, t, tid, T);
  }
}
}  // namespace
extern "C" {
// in: n_in_copy elements (rest of the 2^k input is zero padding when n_in < n); out: n_out elements.
// g_log = 0: the single-device plan; > 0: the six-step plan across 2^g_log emulated devices. use_full: full twiddle table.
int he_ntt(const Fr* in, Fr* out, uint32_t k, const Fr* omega, uint32_t max_digit, uint32_t tile_log, uint32_t threads, uint32_t g_log,
           uint64_t n_in, uint64_t n_out, const Fr* pre3, const Fr* post3, int use_full) {
  const uint64_t n = 1ull << k;
  NttPlan plan = ntt_make_plan(k, max_digit);
  const uint32_t h = k - plan.s[0];
  std::vector<Fr> tw_lo((size_t)1 << h), tw_hi((size_t)1 << (k - h)), tw_full;
  for (size_t i = 0; i < tw_lo.size(); i++) tw_lo[i] = fp_pow_u64(*omega, i);
  for (size_t i = 0; i < tw_hi.size(); i++) tw_hi[i] = fp_pow_u64(*omega, (uint64_t)i << h);
  if (use_full) { tw_full.resize(n); for (uint64_t i = 0; i < n; i++) tw_full[i] = fp_pow_u64(*omega, i); }
  NttOptsHost oh; oh.n_in = n_in; oh.n_out = n_out; oh.pre3 = pre3; oh.post3 = post3;
  if (!n_in) n_in = n;
  if (!n_out) n_out = n;
  auto bind = [&](NttPassParams& p, const Fr* src, Fr* dst) { p.src = src; p.dst = dst; p.tw_lo = tw_lo.data(); p.tw_hi = tw_hi.data(); p.tw_full = use_full ? tw_full.data() : nullptr; };
  if (g_log == 0) {
    std::vector<Fr> buf(n), tmp(n);
    for (uint64_t i = 0; i < n_in; i++) buf[i] = in[i];   // elements >= n_in are never read
    for (uint32_t pi = 0; pi < plan.npass; pi++) {
      NttPassParams p; bind(p, pi == 0 ? buf.data() : tmp.data(), pi == plan.npass - 1 ? buf.data() : tmp.data());
      NttLaunch L = ntt_fill_pass(p, plan, pi, k, h, oh, NttShare(), tile_log, threads);
      run_pass(p, L);
    }
    for (uint64_t i = 0; i < n_out; i++) out[i] = buf[i];
    return (int)plan.npass;
  }
  if (plan.npass < 2 || plan.s[0] <= g_log || (k - plan.s[0]) <= g_log + 1) return -1;
  const uint32_t G = 1u << g_log, s1 = plan.s[0], rest = k - s1;
  const uint64_t n1 = 1ull << s1, lo_count = 1ull << rest, lo_loc = lo_count >> g_log, rows_loc = n1 >> g_log, per = n >> g_log;
  const uint64_t rows_in = (n_in + lo_count - 1) / lo_count, rows_out = (n_out + n1 - 1) / n1;
  std::vector<std::vector<Fr>> A(G, std::vector<Fr>(per));
  std::vector<Fr> Bfull(n);   // device q's slice B[q] sits at its global position q*per
  for (uint32_t q = 0; q < G; q++) {
    for (uint64_t r = 0; r < rows_in; r++) for (uint64_t c = 0; c < lo_loc; c++) { uint64_t gi = r * lo_count + q * lo_loc + c; if (gi < n_in) A[q][r * lo_loc + c] = in[gi]; }
    NttPassParams p; bind(p, A[q].data(), A[q].data());
    NttShare sh; sh.g_log = g_log; sh.q = q; sh.mode = 1;
    NttLaunch L = ntt_fill_pass(p, plan, 0, k, h, oh, sh, tile_log, threads);
    run_pass(p, L);
  }
  for (uint32_t qd = 0; qd < G; qd++)   // what ntt_gather_kernel does
    for (uint64_t row = 0; row < rows_loc; row++) for (uint32_t qs = 0; qs < G; qs++) for (uint64_t c = 0; c < lo_loc; c++)
      Bfull[qd * per + row * lo_count + qs * lo_loc + c] = A[qs][(qd * rows_loc + row) * lo_loc + c];
  for (uint32_t q = 0; q < G; q++) {
    NttShare sh; sh.g_log = g_log; sh.q = q; sh.mode = 2;
    for (uint32_t pi = 1; pi < plan.npass; pi++) {
      bool last = pi == plan.npass - 1;
      NttPassParams p; bind(p, Bfull.data(), last ? A[q].data() : Bfull.data());
      NttLaunch L = ntt_fill_pass(p, plan, pi, k, h, oh, sh, tile_log, threads);
      run_pass(p, L);
    }
    for (uint64_t r = 0; r < rows_out; r++) for (uint64_t c = 0; c < rows_loc; c++) { uint64_t o = r * n1 + q * rows_loc + c; if (o < n_out) out[o] = A[q][r * rows_loc + c]; }
  }
  return (int)plan.npass;
}
}

// ---- quotient numerator / argument-prover term kernels: the per-row bodies run serially ---------------------------------
#include "../../spectre_b200/csrc/quotient.cuh"
namespace {
Fr fr_macro(const uint32_t (&v)[8]) { Fr a; for (int i = 0; i < 8; i++) a.l[i] = v[i]; return a; }
}  // namespace
extern "C" {
// scalars: beta, gamma, theta, y, then challenges. nslots: how many "threads" share the scratch (any value >= 1).
void he_graph_evaluate(const uint32_t* prog, uint32_t ncalc, uint32_t n_inter, const Fr* constants, const int32_t* rotations, const Fr* const* fixed,
                       const Fr* const* advice, const Fr* const* instance, const Fr* scalars, Fr* values, uint64_t size, int32_t rot_scale, uint32_t nslots) {
  std::vector<Fr> scratch((size_t)(n_inter ? n_inter : 1) * nslots);
  GraphArgs a; memset(&a, 0, sizeof a);
  a.prog = prog; a.ncalc = ncalc; a.constants = constants; a.rotations = rotations; a.fixed = fixed; a.advice = advice; a.instance = instance;
  a.scalars = scalars; a.values = values; a.scratch = scratch.data(); a.size = size; a.rot_scale = rot_scale;
  for (uint32_t slot = 0; slot < nslots; slot++)
    for (uint64_t row = slot; row < size; row += nslots) graph_evaluate_row(a, row, slot, nslots);
}
void he_permutation_constraints(Fr* values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len, const Fr* const* z,
                                uint32_t n_cols, const Fr* const* col_values, const Fr* const* sigma, const Fr* l0, const Fr* l_last, const Fr* l_active,
                                const Fr* beta, const Fr* gamma, const Fr* y, const Fr* extended_omega) {
  if (!n_sets) return;
  PermArgs a; memset(&a, 0, sizeof a);
  a.values = values; a.size = size; a.rot_scale = rot_scale; a.last_rotation = last_rotation; a.n_sets = n_sets; a.chunk_len = chunk_len; a.n_cols = n_cols;
  a.z = z; a.col_values = col_values; a.sigma = sigma; a.l0 = l0; a.l_last = l_last; a.l_active = l_active;
  a.beta = *beta; a.gamma = *gamma; a.y = *y; a.extended_omega = *extended_omega;
  constexpr uint32_t zeta[8] = SPB_FR_ZETA_MONT; constexpr uint32_t delta[8] = SPB_FR_DELTA_MONT;
  a.delta = fr_macro(delta); a.delta_start = fp_mul(a.beta, fr_macro(zeta));
  for (uint64_t idx = 0; idx < size; idx++) permutation_constraints_row(a, idx, fp_pow_u64(a.extended_omega, idx));
}
void he_lookup_constraints(Fr* values, uint64_t size, int32_t rot_scale, const Fr* product, const Fr* permuted_input, const Fr* permuted_table, const Fr* table_value,
                           const Fr* l0, const Fr* l_last, const Fr* l_active, const Fr* beta, const Fr* gamma, const Fr* y) {
  LookupArgs a;
  a.values = values; a.size = size; a.rot_scale = rot_scale; a.product = product; a.permuted_input = permuted_input; a.permuted_table = permuted_table;
  a.table_value = table_value; a.l0 = l0; a.l_last = l_last; a.l_active = l_active; a.beta = *beta; a.gamma = *gamma; a.y = *y;
  for (uint64_t idx = 0; idx < size; idx++) lookup_constraints_row(a, idx);
}
// the two term kernels of the grand products, with the block/thread split of omega^i the kernel uses (block = 256 rows)
void he_perm_terms(uint32_t k, const Fr* const* values, const Fr* const* sigma, uint32_t n_cols, uint32_t first_col, const Fr* beta, const Fr* gamma,
                   const Fr* omega, Fr* num, Fr* den) {
  PermTermArgs a;
  for (uint32_t c = 0; c < n_cols; c++) { a.values[c] = values[c]; a.sigma[c] = sigma[c]; }
  constexpr uint32_t delta[8] = SPB_FR_DELTA_MONT;
  a.n_cols = n_cols; a.beta = *beta; a.gamma = *gamma; a.delta = fr_macro(delta); a.omega = *omega;
  a.delta_start = fp_mul(a.beta, fp_pow_u64(a.delta, first_col));
  const uint64_t n = 1ull << k;
  for (uint64_t block = 0; block * 256 < n; block++) {
    Fr base = fp_pow_u64(a.omega, block * 256);
    for (uint32_t t = 0; t < 256 && block * 256 + t < n; t++) perm_terms_row(a, block * 256 + t, fp_mul(base, fp_pow_u64(a.omega, t)), num, den);
  }
}
void he_lookup_terms(const Fr* ci, const Fr* ct, const Fr* pi, const Fr* pt, const Fr* beta, const Fr* gamma, uint64_t n, Fr* num, Fr* den) {
  for (uint64_t i = 0; i < n; i++) lookup_terms_row(ci, ct, pi, pt, *beta, *gamma, i, num, den);
}
}
