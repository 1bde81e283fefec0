// Fr number-theoretic transform for sm_90a: multi-pass (four-step / six-step family) decimation-in-frequency
// NTT with shared-memory tiles, radix-4 register butterflies and shared-memory twiddle staging.
//
// Replaces halo2_proofs::arithmetic::best_fft ([UPSTREAM] halo2_proofs/src/arithmetic.rs; reached from the
// reference through EvaluationDomain inside create_proof / keygen, lightclient-circuits/src/util/circuit.rs:
// 131,158,177,211,263). Contract kept exactly: out[i] = sum_j in[j] * omega^(i*j), natural order in and out,
// no 1/n scaling. The optional pre/post factors fuse what EvaluationDomain does around the transform
// (zeta-coset distribution, zero padding, 1/n, truncation) into the first load and the last store.
//
// Decomposition. n = 2^k is split into P <= 3 digits of s_1..s_P bits, most significant first on the
// input side: j = (j_1 | j_2 | j_3), and least significant first on the output side:
// i = i_1 + 2^{s_1} i_2 + 2^{s_1+s_2} i_3. Pass p transforms digit p (2^{s_p}-point sub-NTTs at stride
// 2^{b_p}, b_p = bits below the digit) for every value of the other digits, then multiplies by the
// inter-digit twiddle omega_{N}^{ j_{p+1} * (i_1 + 2^{s_1} i_2 + ...) }, N = 2^{s_1+..+s_{p+1}}. Passes
// 1..P-1 keep the positional layout (digit p now holds i_p); the last pass writes the digit-reversed
// address, which is the natural-order result. A tile is one sub-NTT length times C neighbouring
// columns, so every global access is a C*32-byte contiguous run.
//
// Inside a tile the sub-NTT is DIF (natural in, bit-reversed out): the bit reversal costs nothing
// because it is folded into the global row address of the store. Data sit in shared memory as eight
// 32-bit limb planes with one pad word per 32 (conflict-free for every power-of-two stride); each
// thread runs two butterfly levels in registers per shared-memory round trip.
//
// Roofline: algorithmic bytes = 64 B/element (SURVEY.md 8d); HBM traffic = P * 64 B/element. The kernel is
// bound by the INT32 multiply pipe ((k/2 + P-1 + [P>1]) Montgomery products of ~139 IMAD each per element),
// not by HBM -- DESIGN.md carries both numbers.
#pragma once
#include "field.cuh"

namespace spb {

struct NttPassParams {
  const Fr* src;
  Fr* dst;
  const Fr* tw_lo;   // omega^i,           i < 2^h
  const Fr* tw_hi;   // omega^(i * 2^h),   i < 2^(k-h)
  const Fr* tw_full; // omega^i, i < 2^k, or nullptr: every twiddle is then one load instead of a two-level product
  uint32_t k;        // log2 n
  uint32_t h;        // split of the two-level power table
  uint32_t s;        // log2 length of this pass's sub-NTT
  uint32_t a;        // bits above the digit (already transformed digits)
  uint32_t b;        // bits below the digit
  uint32_t logc;     // log2 columns per tile
  uint32_t s1;       // bits of the first digit (== s when a == 0)
  uint32_t b_next;   // bits below the NEXT digit (passes before the last)
  uint32_t first, last;
  // ---- multi-device (six-step across devices); all zero / equal to the global values on one device ----------
  uint64_t ntiles;      // tiles this launch covers; CTAs are persistent and stride over them
  uint64_t tile_base;   // added to the tile index: this device's first tile (passes sharded by the first digit)
  uint64_t lo_base;     // global index of this device's first column (first pass, sharded by columns)
  uint32_t b_addr;      // bits below the digit in THIS device's buffer (== b unless sharded by columns)
  uint32_t out_local;   // last pass: store at (o >> s1) * 2^out_cols_log + (i_1 - i1_base) instead of o
  uint32_t out_cols_log;
  uint32_t i1_base;
  uint32_t use_pre, use_post;   // use_pre: 1 = pre[i % 3], 2 = the power table g^i below
  uint64_t n_in;     // elements >= n_in of the input are zero (not read)
  uint64_t n_out;    // only outputs < n_out are stored
  const Fr* pre_lo;  // g^i,          i < 2^h    (use_pre == 2: input i multiplied by g^i in the first pass)
  const Fr* pre_hi;  // g^(i * 2^h),  i < 2^(k-h)
  Fr pre[3];         // input i multiplied by pre[i % 3]   (first pass)
  Fr post[3];        // output i multiplied by post[i % 3] (last pass)
};

// Shared-memory index maps. Data: XOR swizzle of the low five bits with bits 2..6 -- a warp that touches, at any
// butterfly level, 2^a consecutive elements from each of 32/2^a groups spaced 4*2^a apart (and any 32 aligned
// consecutive elements) then hits 32 distinct banks. Twiddles: one pad word per 32 makes every power-of-two stride
// the levels use conflict-free.
SPB_HD uint32_t ntt_swz(uint32_t i) { return i ^ ((i >> 2) & 31u); }
SPB_HD uint32_t ntt_pad(uint32_t i) { return i + (i >> 5); }
SPB_HD uint32_t ntt_col_stride(uint32_t S, uint32_t C) {
  uint32_t base = S < 32 ? 32 : S;  // the swizzle may touch indices up to the next multiple of 32
  return base + ((C >= 32) ? 1u : (32u / C) & 31u);
}
SPB_HD uint32_t ntt_tw_words(uint32_t S) { uint32_t h = S >> 1; return h ? h + (h >> 5) + 1 : 1; }
SPB_HD uint32_t ntt_brev(uint32_t v, uint32_t bits) {
#if defined(__CUDA_ARCH__)
  return bits ? (__brev(v) >> (32 - bits)) : 0;
#else
  uint32_t r = 0; for (uint32_t i = 0; i < bits; i++) { r = (r << 1) | (v & 1); v >>= 1; } return r;
#endif
}

struct NttSmem {
  uint32_t* data;   // 8 planes of plane_words
  uint32_t* tw;     // 8 planes of tw_words
  uint32_t plane_words, tw_words, col_stride;
  SPB_HD Fr load(uint32_t col, uint32_t i) const {
    Fr r; uint32_t o = col * col_stride + ntt_swz(i);
#pragma unroll
    for (int l = 0; l < 8; l++) r.l[l] = data[l * plane_words + o];
    return r;
  }
  SPB_HD void store(uint32_t col, uint32_t i, const Fr& v) const {
    uint32_t o = col * col_stride + ntt_swz(i);
#pragma unroll
    for (int l = 0; l < 8; l++) data[l * plane_words + o] = v.l[l];
  }
  SPB_HD Fr twiddle(uint32_t j) const {
    Fr r;
    uint32_t o = ntt_pad(j);
#pragma unroll
    for (int l = 0; l < 8; l++) r.l[l] = tw[l * tw_words + o];
    return r;
  }
  SPB_HD void set_twiddle(uint32_t j, const Fr& w) const {
    uint32_t o = ntt_pad(j);
#pragma unroll
    for (int l = 0; l < 8; l++) tw[l * tw_words + o] = w.l[l];
  }
  SPB_HD void bind(uint32_t* raw, uint32_t S, uint32_t C) {
    col_stride = ntt_col_stride(S, C);   // == 32/C (mod 32): a warp touching C columns x 32/C consecutive rows is conflict-free
    plane_words = col_stride * C;
    tw_words = ntt_tw_words(S);
    data = raw;
    tw = raw + 8 * plane_words;
  }
};
SPB_HD size_t ntt_smem_bytes(uint32_t S, uint32_t C) { return (size_t)8 * 4 * ((size_t)ntt_col_stride(S, C) * C + ntt_tw_words(S)); }

SPB_HD Fr ntt_ldg(const Fr* p) {
#if defined(__CUDA_ARCH__)
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 lo = __ldg(q), hi = __ldg(q + 1);
  Fr r; r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w; r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
  return r;
#else
  return *p;
#endif
}
SPB_HD Fr ntt_ld_stream(const Fr* p) {
#if defined(__CUDA_ARCH__)
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 lo = __ldcs(q), hi = __ldcs(q + 1);
  Fr r; r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w; r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
  return r;
#else
  return *p;
#endif
}
SPB_HD void ntt_stg(Fr* p, const Fr& v) {
#if defined(__CUDA_ARCH__)
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
  q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
#else
  *p = v;
#endif
}

// omega^E through the full table, or the two-level table (one product unless a level is trivial)
SPB_HD Fr ntt_omega_pow(const NttPassParams& p, uint64_t e) {
  if (p.tw_full) return ntt_ldg(p.tw_full + e);
  uint64_t hi = e >> p.h, lo = e & ((1ull << p.h) - 1);
  if (lo == 0) return ntt_ldg(p.tw_hi + hi);
  Fr wl = ntt_ldg(p.tw_lo + lo);
  if (hi == 0) return wl;
  return fp_mul(ntt_ldg(p.tw_hi + hi), wl);
}
// g^e through the two-level power table of the pre-scale (the same split h as the twiddles)
SPB_HD Fr ntt_pre_pow(const NttPassParams& p, uint64_t e) {
  uint64_t hi = e >> p.h, lo = e & ((1ull << p.h) - 1);
  if (lo == 0) return ntt_ldg(p.pre_hi + hi);
  Fr wl = ntt_ldg(p.pre_lo + lo);
  if (hi == 0) return wl;
  return fp_mul(ntt_ldg(p.pre_hi + hi), wl);
}

// ---- one tile, written as barrier-separated phases over (tid, T) so that tests/hostemu can run the identical code
// ---- serially (every phase for all tid, then the next phase) and the kernel runs it with __syncthreads between.
// tile coordinates:  not last: tile = (hi, lo chunk);            element (r, c) at ((hi << s) + r) << b  +  lo0 + c
//                    last    : tile = (hi-with-i_1-chunk, all);   column c is the row whose first digit is i1_0 + c
struct NttTile {
  uint64_t hi, lo0, i1_0, hi_rest;
  uint32_t rest_bits;   // bits of hi that are not the first digit (last pass, P = 3)
};
SPB_HD NttTile ntt_tile_coords(const NttPassParams& p, uint64_t tile) {
  NttTile t; t.hi = 0; t.lo0 = 0; t.i1_0 = 0; t.hi_rest = 0;
  t.rest_bits = p.a > p.s1 ? p.a - p.s1 : 0;
  if (!p.last) {
    const uint32_t chunks_log = p.b_addr - p.logc;
    t.hi = tile >> chunks_log;
    t.lo0 = (tile & ((1ull << chunks_log) - 1)) << p.logc;
  } else if (p.a > 0) {
    // chunk along the first digit; remaining hi bits (second digit when P = 3) are fixed per tile
    t.hi_rest = tile & ((1ull << t.rest_bits) - 1);
    t.i1_0 = (tile >> t.rest_bits) << p.logc;
  }
  return t;
}
// stage sub-NTT twiddles omega_{2^s}^j = omega^(j << (k-s)) into shared memory (once per CTA)
SPB_HD void ntt_phase_twiddles(const NttPassParams& p, const NttSmem& sm, uint32_t tid, uint32_t T) {
  const uint32_t S = 1u << p.s;
  for (uint32_t j = tid; j < (S >> 1); j += T) sm.set_twiddle(j, ntt_omega_pow(p, (uint64_t)j << (p.k - p.s)));
}
// load the tile (natural order), fusing zero padding and the pre-scale (zeta-coset factors, or powers of a coset generator)
SPB_HD void ntt_phase_load(const NttPassParams& p, const NttSmem& sm, const NttTile& t, uint32_t tid, uint32_t T) {
  const uint32_t S = 1u << p.s, C = 1u << p.logc;
  for (uint32_t e = tid; e < S * C; e += T) {
    // lanes run along the contiguous global direction: columns for strided passes, the row for the last one
    uint32_t c, r;
    uint64_t gi, gglob;   // address in this device's buffer, and the global element index
    if (!p.last) {
      c = e & (C - 1); r = e >> p.logc;
      gi = ((((t.hi << p.s) + r) << p.b_addr) + t.lo0 + c);
      gglob = ((((t.hi << p.s) + r) << p.b) + p.lo_base + t.lo0 + c);
    } else { r = e & (S - 1); c = e >> p.s; gi = ((((t.i1_0 + c) << t.rest_bits) + t.hi_rest) << p.s) + r; gglob = gi; }
    Fr v;
    if (p.first && gglob >= p.n_in) v = fp_zero<FrParams>();
    else {
      v = ntt_ld_stream(p.src + gi);
      if (p.first && p.use_pre == 1) { uint32_t m = (uint32_t)(gglob % 3); if (m) v = fp_mul(v, p.pre[m]); }
      else if (p.first && p.use_pre == 2 && gglob) v = fp_mul(v, ntt_pre_pow(p, gglob));
    }
    sm.store(c, r, v);
  }
}
// one radix-2 DIF level of half-size m (used first when the digit has an odd number of levels)
SPB_HD void ntt_phase_radix2(const NttPassParams& p, const NttSmem& sm, uint32_t m, uint32_t tid, uint32_t T) {
  const uint32_t S = 1u << p.s, C = 1u << p.logc;
  for (uint32_t e = tid; e < (S >> 1) * C; e += T) {
    uint32_t c = e / (S >> 1), t = e % (S >> 1);
    Fr x0 = sm.load(c, t), x1 = sm.load(c, t + m);
    Fr u = fp_add(x0, x1), d = fp_sub(x0, x1);
    if (m > 1 && t) d = fp_mul(d, sm.twiddle(t));
    sm.store(c, t, u); sm.store(c, t + m, d);
  }
}
// two DIF levels (half-sizes m and m/2) in registers per shared-memory round trip
SPB_HD void ntt_phase_radix4(const NttPassParams& p, const NttSmem& sm, uint32_t m, uint32_t tid, uint32_t T) {
  const uint32_t S = 1u << p.s, C = 1u << p.logc;
  const uint32_t q = m >> 1;                      // quarter stride
  const uint32_t tws = (S >> 1) / m;              // twiddle index step for level m
  for (uint32_t e = tid; e < (S >> 2) * C; e += T) {
    uint32_t c = e / (S >> 2), t = e % (S >> 2);
    uint32_t g = t / q, j = t % q, i = g * 2 * m + j;
    Fr x0 = sm.load(c, i), x1 = sm.load(c, i + q), x2 = sm.load(c, i + m), x3 = sm.load(c, i + m + q);
    // level m
    Fr u0 = fp_add(x0, x2), u2 = fp_sub(x0, x2);
    Fr u1 = fp_add(x1, x3), u3 = fp_sub(x1, x3);
    if (j) u2 = fp_mul(u2, sm.twiddle(j * tws));
    u3 = fp_mul(u3, sm.twiddle((j + q) * tws));
    // level m/2 (twiddle omega_m^j for both pairs)
    Fr v0 = fp_add(u0, u1), v1 = fp_sub(u0, u1);
    Fr v2 = fp_add(u2, u3), v3 = fp_sub(u2, u3);
    if (j) { Fr w = sm.twiddle(2 * j * tws); v1 = fp_mul(v1, w); v3 = fp_mul(v3, w); }
    sm.store(c, i, v0); sm.store(c, i + q, v1); sm.store(c, i + m, v2); sm.store(c, i + m + q, v3);
  }
}
// store: position qpos holds digit value rev(qpos); fuse the inter-digit twiddle / post-scale
SPB_HD void ntt_phase_store(const NttPassParams& p, const NttSmem& sm, const NttTile& t, uint32_t tid, uint32_t T) {
  const uint32_t S = 1u << p.s, C = 1u << p.logc;
  for (uint32_t e = tid; e < S * C; e += T) {
    uint32_t c = e & (C - 1), qpos = e >> p.logc;
    uint32_t kd = ntt_brev(qpos, p.s);
    Fr v = sm.load(c, qpos);
    if (!p.last) {
      // K' = i_1 + 2^{s_1} i_2 + ... restricted to the digits done so far. With P <= 3 the digits above the
      // current one are just i_1 (= hi), so K' = hi + 2^a * kd.
      uint64_t kprime = t.hi + ((uint64_t)kd << p.a);
      uint64_t lo = t.lo0 + c, lo_glob = p.lo_base + lo;
      // exponent of omega_n: j_next * K' * 2^(bits below the next digit)
      uint64_t jn = lo_glob >> p.b_next;
      uint64_t ex = (jn * kprime) << p.b_next;
      if (ex) v = fp_mul(v, ntt_omega_pow(p, ex));
      uint64_t go = ((((t.hi << p.s) + kd) << p.b_addr) + lo);
      ntt_stg(p.dst + go, v);
    } else {
      uint64_t o = (t.i1_0 + c) + (t.hi_rest << p.s1) + ((uint64_t)kd << p.a);
      if (o < p.n_out) {
        if (p.use_post) v = fp_mul(v, p.post[o % 3]);
        uint64_t addr = p.out_local ? (((o >> p.s1) << p.out_cols_log) + (t.i1_0 + c - p.i1_base)) : o;
        ntt_stg(p.dst + addr, v);
      }
    }
  }
}

// ---- host-side plan and per-pass geometry (no CUDA calls: shared by ntt.cu and tests/hostemu) -------------------
struct NttPlan { uint32_t npass; uint32_t s[3]; };
// digits of at most max_digit bits, larger digits first
inline NttPlan ntt_make_plan(uint32_t k, uint32_t max_digit) {
  NttPlan p; p.npass = 1; p.s[0] = k; p.s[1] = p.s[2] = 0;
  if (k <= max_digit) return p;
  p.npass = (k + max_digit - 1) / max_digit;
  uint32_t rem = k;
  for (uint32_t i = 0; i < p.npass; i++) { uint32_t left = p.npass - i; p.s[i] = (rem + left - 1) / left; rem -= p.s[i]; }
  return p;
}
// The device's share of a pass: g_log = log2(#devices) (0 on one device), q = this device's index,
// mode 0 = whole problem on this device, 1 = first pass sharded by columns, 2 = later pass sharded by the first digit.
struct NttShare { uint32_t g_log = 0, q = 0, mode = 0; };
struct NttOptsHost {   // what EvaluationDomain fuses around the transform
  uint64_t n_in = 0, n_out = 0;  // 0 = n
  const Fr* pre3 = nullptr;      // 3 factors, or nullptr
  const Fr* post3 = nullptr;
  const Fr* pre_lo = nullptr;    // two-level power table of g (split h of the plan), or nullptr: input i multiplied by g^i
  const Fr* pre_hi = nullptr;
};
struct NttLaunch { uint64_t tiles; uint32_t threads; size_t smem; };
// Fill everything of pass `pi` except the pointers (src, dst, twiddle tables).
inline NttLaunch ntt_fill_pass(NttPassParams& p, const NttPlan& plan, uint32_t pi, uint32_t k, uint32_t h, const NttOptsHost& opts, const NttShare& sh,
                               uint32_t tile_log, uint32_t max_threads) {
  const uint64_t n = 1ull << k;
  const Fr* src = p.src; Fr* dst = p.dst; const Fr* lo = p.tw_lo; const Fr* hi = p.tw_hi; const Fr* full = p.tw_full;
  p = NttPassParams();
  p.src = src; p.dst = dst; p.tw_lo = lo; p.tw_hi = hi; p.tw_full = full;
  uint32_t a = 0; for (uint32_t i = 0; i < pi; i++) a += plan.s[i];
  p.k = k; p.h = h;
  p.s = plan.s[pi]; p.a = a; p.b = k - a - p.s; p.s1 = plan.s[0];
  p.first = (pi == 0); p.last = (pi == plan.npass - 1);
  p.b_next = p.last ? 0 : p.b - plan.s[pi + 1];
  p.n_in = opts.n_in ? opts.n_in : n;
  p.n_out = opts.n_out ? opts.n_out : n;
  if (p.first && opts.pre3) { p.use_pre = 1; for (int i = 0; i < 3; i++) p.pre[i] = opts.pre3[i]; }
  if (p.first && opts.pre_lo) { p.use_pre = 2; p.pre_lo = opts.pre_lo; p.pre_hi = opts.pre_hi; }
  if (p.last && opts.post3) { p.use_post = 1; for (int i = 0; i < 3; i++) p.post[i] = opts.post3[i]; }
  p.b_addr = p.b;
  // columns per tile: as many as fit, bounded by what the direction offers on this device
  uint32_t avail = p.last ? (p.a ? p.s1 : 0) : p.b;
  if (sh.mode == 1) { avail = p.b - sh.g_log; p.b_addr = p.b - sh.g_log; p.lo_base = (uint64_t)sh.q << p.b_addr; }
  if (sh.mode == 2 && p.last) avail = p.s1 - sh.g_log;
  uint32_t logc = tile_log > p.s ? tile_log - p.s : 0;
  if (logc > avail) logc = avail;
  if (logc > 5) logc = 5;
  p.logc = logc;
  NttLaunch L;
  L.tiles = (n >> (p.s + logc)) >> sh.g_log;   // this device's tiles
  if (sh.mode == 2) {
    p.tile_base = L.tiles * sh.q;
    if (p.last) { p.out_local = 1; p.out_cols_log = p.s1 - sh.g_log; p.i1_base = sh.q << (p.s1 - sh.g_log); }
  }
  p.ntiles = L.tiles;
  uint32_t S = 1u << p.s, C = 1u << logc;
  uint32_t quads = (S * C) / 4; if (quads < 32) quads = 32;
  L.threads = quads < max_threads ? quads : max_threads;
  L.smem = ntt_smem_bytes(S, C);
  return L;
}

#if defined(__CUDACC__)
#if defined(SPB_NTT_KERNELS)
// One kernel for every pass. A CTA handles one tile (2^s rows of the digit x 2^logc columns) at a time and strides
// over `ntiles` tiles; the sub-NTT twiddles are staged once per CTA.
__global__ void __launch_bounds__(512) ntt_pass_kernel(const NttPassParams p) {
  extern __shared__ uint32_t smem_raw[];
  const uint32_t S = 1u << p.s, C = 1u << p.logc, T = blockDim.x, tid = threadIdx.x;
  NttSmem sm; sm.bind(smem_raw, S, C);
  ntt_phase_twiddles(p, sm, tid, T);
  for (uint64_t tile_it = blockIdx.x; tile_it < p.ntiles; tile_it += gridDim.x) {
    const NttTile t = ntt_tile_coords(p, tile_it + p.tile_base);
    ntt_phase_load(p, sm, t, tid, T);
    __syncthreads();
    uint32_t m = S >> 1;  // current half-size
    if (p.s & 1) { ntt_phase_radix2(p, sm, m, tid, T); m >>= 1; __syncthreads(); }
    for (; m >= 2; m >>= 2) { ntt_phase_radix4(p, sm, m, tid, T); __syncthreads(); }
    ntt_phase_store(p, sm, t, tid, T);
    __syncthreads();   // the next tile overwrites the shared-memory planes
  }
}

// All-to-all of the six-step NTT as ONE kernel per destination device: every thread pulls one 32-byte element
// straight out of a peer's buffer over NVLink (peer access enabled at spb_init) and drops it at its transposed place.
//   dst[row][qs * lo_loc + c] = peers[qs][(row_base + row) * lo_loc + c],   row < rows_loc, qs < G, c < lo_loc
struct NttGatherArgs { const Fr* peers[16]; Fr* dst; uint64_t rows_loc, lo_loc, row_base; uint32_t g_log; };
__global__ void __launch_bounds__(256) ntt_gather_kernel(NttGatherArgs a) {
  const uint64_t total = a.rows_loc * (a.lo_loc << a.g_log);
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t row = i / (a.lo_loc << a.g_log), col = i % (a.lo_loc << a.g_log);
    const uint64_t qs = col / a.lo_loc, c = col % a.lo_loc;
    const uint4* src = reinterpret_cast<const uint4*>(a.peers[qs] + (a.row_base + row) * a.lo_loc + c);
    uint4 lo = src[0], hi = src[1];
    uint4* d = reinterpret_cast<uint4*>(a.dst + i);
    d[0] = lo; d[1] = hi;
  }
}

// out[i] = base^(i << shift), i < count  (power tables; also reused for coset / vanishing constants)
__global__ void fr_pow_table_kernel(Fr* out, Fr base, uint64_t count, uint32_t shift) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  out[i] = fp_pow_u64(base, i << shift);
}

#endif  // SPB_NTT_KERNELS
#endif  // __CUDACC__
}  // namespace spb
