// BN254 G1 multi-scalar multiplication for sm_90a: signed-digit windowed Pippenger with a
// radix sort of the digits and a load-balanced segmented bucket accumulation.
//
// Replaces halo2_proofs::arithmetic::best_multiexp / multiexp_serial ([UPSTREAM] halo2_proofs/src/arithmetic.rs;
// reached from every ParamsKZG::commit / commit_lagrange inside create_proof and keygen, reference call sites
// lightclient-circuits/src/util/circuit.rs:131,158,177,211,263). The contract is the group element
// sum_i scalars[i] * bases[i]; integers are exact, so any correct schedule is bit-identical to the CPU
// result after affine normalisation.
//
// Pipeline (one MSM of n pairs, window width c, W = ceil(255/c) windows, B = 2^(c-1) buckets per bucket set; a basis
// with precomputed 2^(c*w) multiples folds all windows into ONE bucket set, otherwise there are W sets):
//   1. digits   : Montgomery -> canonical scalar (one product), signed c-bit digits d_w in (-B, B]; every non-zero digit
//                 becomes an entry (key = w*B + |d|-1, value = point index | sign << 31) in an unsorted list, compacted
//                 with one atomic per block. Zero digits are dropped here; the entry count M goes to the host.
//   2. sort     : LSD radix sort of the M entries by key (CUB onesweep over the key's bit length only); order inside a
//                 bucket is irrelevant.
//   3. offsets  : offsets[k] = first entry of bucket k (every bucket, empty ones included; offsets[BW*B] = M).
//   4. accumulate: the sorted entry list is cut into fixed chunks of L entries, ONE THREAD PER CHUNK, so every
//                 thread performs the same number of mixed XYZZ additions whatever the digit distribution
//                 (witness columns put hundreds of thousands of points into one bucket). A run of equal keys
//                 that lies inside a chunk is a complete bucket and is stored directly; the run that leaves
//                 a chunk ("tail") and the run that enters one ("head") are stored as chunk pieces.
//   5. stitch   : one thread per tail piece walks the following head pieces of the same key and stores the
//                 bucket; chains longer than a cap (giant buckets) go to block-wide / grid-wide tree reductions.
//                 (Summing the pieces inside the group reduction of step 6 instead costs more in the groups than it saves in
//                 the stitch -- three adder sites in one thread either cost 255 registers or an out-of-line adder.)
//   6. reduce   : per bucket set S = sum_b (b+1) * bucket[b]: groups of 8 buckets by a running sum per thread, then the group
//                 sums viewed as an R x C matrix: sum_t t*S1_t = C * sum_r r*Row_r + sum_c c*Col_c -- tree sums and local
//                 weights < 2^7 only.
//   7. host     : fold the few partial sums per bucket set, Horner over the sets (none with tables), one inversion.
//
// Roofline: algorithmic bytes = 96 B per pair (SURVEY.md 8d). The kernel that dominates (step 4) executes
// W mixed additions of 8M+2S (~1390 IMAD-class instructions each) per pair: it is bound by the INT32 multiply pipe by two
// orders of magnitude, not by HBM. DESIGN.md states both fractions.
//
// Every function below is written per thread (`tid`) so that tests/hostemu can run the identical code
// serially on the CPU (-DSPB_EMULATE_PTX) against the oracle.
#pragma once
#include <stdlib.h>
#include "curve.cuh"

namespace spb {

struct MsmGeom {
  uint32_t c;        // window bits
  uint32_t W;        // scalar windows
  uint32_t B;        // buckets per bucket-window = 2^(c-1)
  uint32_t L;        // entries per accumulation chunk
  uint32_t BW;       // bucket windows: W normally, 1 when the basis carries precomputed 2^(c*w) multiples
  uint32_t precomp;  // 1: window w of point i uses table point w*tab_stride + i and ALL windows share one bucket set
  uint32_t tab_stride;
};

struct alignas(8) MsmEntry { uint32_t key, val; };

// Chunk length actually used for a sorted list of M entries. The host picks L from the upper bound n * W; the long chunk it picks
// for lists beyond the L2 (kLongChunk) only pays when the list really is that long -- witness columns drop most of their
// digits -- so every kernel that cuts the list derives the same effective length from the entry count on the device.
static const uint32_t kLongChunk = 96, kShortChunk = 32;
#ifndef SPB_LONG_CHUNK_MIN_ENTRIES
// 2^23 entries = 64 MB of short-chunk pieces, beyond H100's 50 MB L2; tests/hostemu lowers it to run the long-chunk path on
// CPU-sized inputs
#define SPB_LONG_CHUNK_MIN_ENTRIES (1ull << 23)
#endif
static const uint64_t kLongChunkMinEntries = SPB_LONG_CHUNK_MIN_ENTRIES;
SPB_HD uint32_t msm_effective_chunk(uint32_t L, uint64_t M) { return (L == kLongChunk && M < kLongChunkMinEntries) ? kShortChunk : L; }

static const uint32_t kNoKey = 0xffffffffu;

#if defined(__CUDA_ARCH__)
SPB_D uint32_t spb_atomic_inc(uint32_t* p) { return atomicAdd(p, 1u); }
#else
inline uint32_t spb_atomic_inc(uint32_t* p) { uint32_t v = *p; *p = v + 1; return v; }
#endif

// canonical little-endian scalar -> signed digit of window w. carry chain recomputed from window 0: cheap
// (W <= 64 iterations of shifts) and keeps the digit kernels free of per-scalar storage.
struct DigitIter {
  uint32_t limbs[8];
  uint32_t c, carry, w;
  SPB_HD void init(const Fr& canonical, uint32_t c_) {
    for (int i = 0; i < 8; i++) limbs[i] = canonical.l[i];
    c = c_; carry = 0; w = 0;
  }
  // returns signed digit of the next window
  SPB_HD int32_t next() {
    uint32_t bit = w * c, word = bit >> 5, sh = bit & 31;
    uint64_t v = 0;
    if (word < 8) {
      v = limbs[word];
      if (word + 1 < 8) v |= (uint64_t)limbs[word + 1] << 32;
      v >>= sh;
    }
    uint32_t raw = (uint32_t)(v & ((1u << c) - 1)) + carry;
    w++;
    if (raw > (1u << (c - 1))) { carry = 1; return (int32_t)raw - (int32_t)(1u << c); }
    carry = 0;
    return (int32_t)raw;
  }
};

// ---- step 1: digits -> unsorted entries -----------------------------------------------------------------------
SPB_HD MsmEntry msm_make_entry(uint64_t tid, uint32_t w, int32_t d, const MsmGeom& g) {
  const uint32_t mag = d < 0 ? (uint32_t)(-d) : (uint32_t)d;
  MsmEntry e;
  e.key = (g.precomp ? 0u : w * g.B) + mag - 1;
  e.val = ((uint32_t)tid + (g.precomp ? w * g.tab_stride : 0u)) | (d < 0 ? 0x80000000u : 0u);
  return e;
}
// number of non-zero signed digits of a canonical scalar
SPB_HD uint32_t msm_digit_count(const Fr& s, const MsmGeom& g) {
  DigitIter it; it.init(s, g.c);
  uint32_t k = 0;
  for (uint32_t w = 0; w < g.W; w++) k += it.next() != 0;
  return k;
}
// Serial form of msm_digits_kernel: scalar `tid` reserves its entries with one counter increment and writes them in window
// order. The kernel reserves one range per block instead and writes each window of a warp contiguously; the list is sorted
// next, so only the multiset of entries matters.
SPB_HD void msm_digits_thread(uint64_t tid, uint64_t n, const Fr* scalars, MsmGeom g, uint32_t* total, MsmEntry* ent) {
  if (tid >= n) return;
  Fr s = fp_from_mont(scalars[tid]);
  if (fp_is_zero(s)) return;
  uint32_t pos = *total;
  *total = pos + msm_digit_count(s, g);
  DigitIter it; it.init(s, g.c);
  for (uint32_t w = 0; w < g.W; w++) {
    int32_t d = it.next();
    if (d != 0) ent[pos++] = msm_make_entry(tid, w, d, g);
  }
}

// ---- step 2: the radix sort looks at the bits of the largest bucket key BW*B - 1 only ------------------------------
inline int msm_key_bits(const MsmGeom& g) {
  int bits = 0;
  for (uint64_t k = (uint64_t)g.BW * g.B - 1; k; k >>= 1) bits++;
  return bits;
}

// ---- step 3: bucket offsets of the sorted list ------------------------------------------------------------------
// offsets[k] = number of entries with key < k, for every k in [0, nb] (so offsets[nb] = M): a lower-bound search per bucket,
// which costs the same for empty buckets, sparse lists and M = 0.
SPB_HD void msm_offsets_thread(uint64_t k, uint64_t nb, uint64_t M, const MsmEntry* sorted, uint32_t* offsets) {
  if (k > nb) return;
  uint64_t lo = 0, hi = M;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (sorted[mid].key < k) lo = mid + 1; else hi = mid;
  }
  offsets[k] = (uint32_t)lo;
}

// ---- serial reference of steps 1-3: a counting sort (histogram, exclusive scan, scatter at a cursor) ----------------
SPB_HD void msm_count_thread(uint64_t tid, uint64_t n, const Fr* scalars, MsmGeom g, uint32_t* counts) {
  if (tid >= n) return;
  Fr s = fp_from_mont(scalars[tid]);
  if (fp_is_zero(s)) return;
  DigitIter it; it.init(s, g.c);
  for (uint32_t w = 0; w < g.W; w++) {
    int32_t d = it.next();
    if (d == 0) continue;
    uint32_t mag = d < 0 ? (uint32_t)(-d) : (uint32_t)d;
    spb_atomic_inc(&counts[(g.precomp ? 0u : w * g.B) + mag - 1]);
  }
}

SPB_HD void msm_scatter_thread(uint64_t tid, uint64_t n, const Fr* scalars, MsmGeom g, uint32_t* cursor, MsmEntry* ent) {
  if (tid >= n) return;
  Fr s = fp_from_mont(scalars[tid]);
  if (fp_is_zero(s)) return;
  DigitIter it; it.init(s, g.c);
  for (uint32_t w = 0; w < g.W; w++) {
    int32_t d = it.next();
    if (d == 0) continue;
    uint32_t mag = d < 0 ? (uint32_t)(-d) : (uint32_t)d;
    uint32_t key = (g.precomp ? 0u : w * g.B) + mag - 1;
    uint32_t pos = spb_atomic_inc(&cursor[key]);
    MsmEntry e; e.key = key; e.val = ((uint32_t)tid + (g.precomp ? w * g.tab_stride : 0u)) | (d < 0 ? 0x80000000u : 0u);
    ent[pos] = e;
  }
}

// ---- step 4: chunked accumulation ----------------------------------------------------------------------
SPB_HD G1Affine msm_load_point(const G1Affine* bases, uint32_t val) {
#if defined(__CUDA_ARCH__)
  const uint4* q = reinterpret_cast<const uint4*>(bases + (val & 0x7fffffffu));
  uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
  G1Affine p;
  p.x.l[0] = a.x; p.x.l[1] = a.y; p.x.l[2] = a.z; p.x.l[3] = a.w; p.x.l[4] = b.x; p.x.l[5] = b.y; p.x.l[6] = b.z; p.x.l[7] = b.w;
  p.y.l[0] = c.x; p.y.l[1] = c.y; p.y.l[2] = c.z; p.y.l[3] = c.w; p.y.l[4] = d.x; p.y.l[5] = d.y; p.y.l[6] = d.z; p.y.l[7] = d.w;
#else
  G1Affine p = bases[val & 0x7fffffffu];
#endif
  if (val & 0x80000000u) p.y = fp_neg(p.y);
  return p;
}

// One chunk = entries [tid*L, min((tid+1)*L, M)). Outputs:
//   buckets[key]        for runs that are whole buckets
//   head_key/head[tid]  first run when it started in an earlier chunk (kNoKey if none)
//   tail_key/tail[tid]  last run when it continues into the next chunk, or a single-run chunk whose bucket
//                       starts here and continues (chain start)                      (kNoKey if none)
SPB_HD MsmEntry msm_load_entry(const MsmEntry* p) {
#if defined(__CUDA_ARCH__)
  uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
  MsmEntry e; e.key = v.x; e.val = v.y; return e;
#else
  return *p;
#endif
}

SPB_HD void msm_accumulate_thread(uint64_t tid, uint64_t M, MsmGeom g, const MsmEntry* ent,
                                  const G1Affine* bases, G1Xyzz* buckets, uint32_t* head_key, G1Xyzz* head,
                                  uint32_t* tail_key, G1Xyzz* tail) {
  const uint32_t L = msm_effective_chunk(g.L, M);
  uint64_t lo = tid * L;
  if (lo >= M) return;
  uint64_t hi = lo + L < M ? lo + L : M;
  uint32_t hk = kNoKey, tk = kNoKey;
  MsmEntry first = msm_load_entry(ent + lo);
  uint32_t cur = first.key;
  bool run_started_before = lo > 0 && msm_load_entry(ent + lo - 1).key == cur;  // the current run began in an earlier chunk
  G1Xyzz acc = xyzz_from_affine(msm_load_point(bases, first.val));
  for (uint64_t e = lo + 1; e < hi; e++) {
    MsmEntry en = msm_load_entry(ent + e);
    uint32_t k = en.key;
    G1Affine p = msm_load_point(bases, en.val);
    if (k == cur) {
      xyzz_add_mixed(acc, p);
    } else {
      // the run of `cur` ends inside this chunk
      if (run_started_before) { hk = cur; head[tid] = acc; }
      else buckets[cur] = acc;
      run_started_before = false;
      cur = k;
      acc = xyzz_from_affine(p);
    }
  }
  bool continues = hi < M && msm_load_entry(ent + hi).key == cur;
  if (continues) {
    if (run_started_before) { hk = cur; head[tid] = acc; }  // middle link of a chain
    else { tk = cur; tail[tid] = acc; }                     // chain start
  } else {
    if (run_started_before) { hk = cur; head[tid] = acc; }  // last link of a chain
    else buckets[cur] = acc;                                // whole bucket
  }
  head_key[tid] = hk;
  tail_key[tid] = tk;
}

// ---- step 5: stitch chains ------------------------------------------------------------------------------
// chain started by tail[tid]: links are head[tid+1], head[tid+2], ... while their key matches.
// Short chains are summed here; long ones are queued for msm_giant_block.
SPB_HD void msm_stitch_thread(uint64_t tid, uint64_t T, uint32_t cap, const uint32_t* head_key, const G1Xyzz* head,
                              const uint32_t* tail_key, const G1Xyzz* tail, G1Xyzz* buckets, uint32_t* giant_count,
                              uint32_t* giant_list) {
  if (tid >= T) return;
  uint32_t key = tail_key[tid];
  if (key == kNoKey) return;
  uint64_t j = tid + 1, len = 0;
  while (j < T && head_key[j] == key && len <= cap) { j++; len++; }
  if (len > cap) { uint32_t slot = spb_atomic_inc(giant_count); giant_list[slot] = (uint32_t)tid; return; }
  G1Xyzz acc = tail[tid];
  for (uint64_t q = tid + 1; q < tid + 1 + len; q++) xyzz_add(acc, head[q]);
  buckets[key] = acc;
}

// ---- step 6: weighted bucket sum  S_w = sum_b (b+1) * bucket[w][b] ---------------------------------------------
// Two levels, both free of scalar multiples and of long running sums:
//  (a) groups: thread t takes the m = 2^m_log consecutive buckets b = t*m + j and forms, with one running sum from the top,
//      S1_t = sum_j B_{t*m+j} and W1_t = sum_j j * B_{t*m+j} (2m - 1 additions, no synchronisation, every thread busy).
//      Empty buckets are recognised from the bucket offsets of the sort (step 3), so the bucket array is never cleared
//      and never read where nothing was written. Then S_w = sum_t W1_t + sum_t S1_t + m * sum_t t * S1_t.
//  (b) the T = B / m group sums S1 are viewed as an R x C matrix (t = r*C + c):
//      sum_t t*S1_t = C * sum_r r*Row_r + sum_c c*Col_c,   Row_r = sum_c S1[r][c],  Col_c = sum_r S1[r][c]
//      -- tree sums (log depth) and, per block of 128 rows / columns, one suffix scan: weights < 2^7 only. The W1 are
//      summed by rows next to it.
struct MsmTail {
  uint32_t m_log;         // buckets per group = 2^m_log
  uint32_t r_log, c_log;  // R = 2^r_log rows, C = 2^c_log columns, R*C = T = B >> m_log group sums
  uint32_t nbr, nbc;      // blocks (of 128 items) covering the rows / the columns in the weighted pass
};
inline MsmTail msm_tail_shape(uint32_t c) {
  MsmTail t; uint32_t bits = c - 1;
  t.m_log = bits < 3 ? bits : 3;
  bits -= t.m_log;
  t.c_log = bits / 2; t.r_log = bits - t.c_log;
  t.nbr = ((1u << t.r_log) + 127) / 128; t.nbc = ((1u << t.c_log) + 127) / 128;
  return t;
}
// Partial layout per bucket set: [A(nbr) | S(nbr) | D(nbc) | T(nbc) | V(nbr)], each over a block of 128 rows / columns with
// LOCAL weights: A[j] = sum_i i * Row_{128j+i}, S[j] = sum_i Row_{128j+i}, D[j] = sum_i i * Col_{128j+i}, T[j] = sum_i
// Col_{128j+i}, V[j] = sum_i WRow_{128j+i} (WRow_r = sum_c W1[r][c]). The host adds the 128*j offsets (msm_tail_finish).
SPB_HD uint32_t msm_tail_partials(const MsmTail& t) { return 3 * t.nbr + 2 * t.nbc; }

// (a): one group of buckets. offsets[b+1] - offsets[b] entries are in bucket b (step 3).
SPB_HD void msm_group_thread(uint64_t tid, uint64_t ngroups, uint32_t m_log, const uint32_t* offsets, const G1Xyzz* buckets, G1Xyzz* s1, G1Xyzz* w1) {
  if (tid >= ngroups) return;
  const uint64_t b0 = tid << m_log;
  G1Xyzz run = xyzz_identity(), acc = xyzz_identity();
  uint32_t hi = offsets[b0 + (1u << m_log)];
  for (int j = (int)(1u << m_log) - 1; j >= 0; j--) {
    const uint32_t lo = offsets[b0 + (uint64_t)j];
    if (hi != lo) xyzz_add(run, buckets[b0 + (uint64_t)j]);
    hi = lo;
    if (j >= 1) xyzz_add(acc, run);   // after the loop: acc = sum_{j>=1} (sum_{i>=j} B_i) = sum_i i * B_i
  }
  s1[tid] = run;
  w1[tid] = acc;
}
// host-side reference of the kernels below (tests/hostemu): buckets -> partials
inline void msm_tail_host(const MsmGeom& g, const uint32_t* offsets, const G1Xyzz* buckets, G1Xyzz* partials) {
  MsmTail t = msm_tail_shape(g.c);
  uint32_t R = 1u << t.r_log, C = 1u << t.c_log, per = msm_tail_partials(t);
  const uint64_t T = (uint64_t)g.B >> t.m_log;
  G1Xyzz* s1 = (G1Xyzz*)malloc(sizeof(G1Xyzz) * T * g.BW);
  G1Xyzz* w1 = (G1Xyzz*)malloc(sizeof(G1Xyzz) * T * g.BW);
  for (uint64_t tid = 0; tid < T * g.BW; tid++) msm_group_thread(tid, T * g.BW, t.m_log, offsets, buckets, s1, w1);
  for (uint32_t w = 0; w < g.BW; w++) {
    const G1Xyzz* X = s1 + (uint64_t)w * T;
    const G1Xyzz* V = w1 + (uint64_t)w * T;
    G1Xyzz* out = partials + (uint64_t)w * per;
    for (uint32_t i = 0; i < per; i++) out[i] = xyzz_identity();
    for (uint32_t r = 0; r < R; r++) {
      G1Xyzz row = xyzz_identity(), wrow = xyzz_identity();
      for (uint32_t c = 0; c < C; c++) { xyzz_add(row, X[(uint64_t)r * C + c]); xyzz_add(wrow, V[(uint64_t)r * C + c]); }
      G1Xyzz wr = xyzz_mul_u32(row, r % 128);
      xyzz_add(out[r / 128], wr);
      xyzz_add(out[t.nbr + r / 128], row);
      xyzz_add(out[2 * t.nbr + 2 * t.nbc + r / 128], wrow);
    }
    for (uint32_t c = 0; c < C; c++) {
      G1Xyzz col = xyzz_identity();
      for (uint32_t r = 0; r < R; r++) xyzz_add(col, X[(uint64_t)r * C + c]);
      G1Xyzz wc = xyzz_mul_u32(col, c % 128);
      xyzz_add(out[2 * t.nbr + c / 128], wc);
      xyzz_add(out[2 * t.nbr + t.nbc + c / 128], col);
    }
  }
  free(s1); free(w1);
}
// host: window sum from its partials
inline G1Xyzz msm_tail_finish(const MsmGeom& g, const G1Xyzz* part) {
  MsmTail t = msm_tail_shape(g.c);
  // sum_j (X[j] + 128 j Y[j]) = sum_j X[j] + 128 * sum_j j Y[j]; the second sum by running sums from the top block down
  auto fold = [](const G1Xyzz* X, const G1Xyzz* Y, uint32_t nb, G1Xyzz* plain) {
    G1Xyzz sx = xyzz_identity(), run = xyzz_identity(), wsum = xyzz_identity();
    for (int j = (int)nb - 1; j >= 0; j--) {
      xyzz_add(sx, X[j]);
      if (j >= 1) { xyzz_add(run, Y[j]); xyzz_add(wsum, run); }   // after the loop: wsum = sum_j j * Y[j]
    }
    if (plain) { *plain = run; xyzz_add(*plain, Y[0]); }
    for (int i = 0; i < 7; i++) wsum = xyzz_dbl(wsum);
    xyzz_add(sx, wsum);
    return sx;
  };
  G1Xyzz S;
  G1Xyzz A = fold(part, part + t.nbr, t.nbr, &S);                                   // sum_r r * Row_r ; S = sum_t S1_t
  G1Xyzz D = fold(part + 2 * t.nbr, part + 2 * t.nbr + t.nbc, t.nbc, nullptr);      // sum_c c * Col_c
  for (uint32_t i = 0; i < t.c_log; i++) A = xyzz_dbl(A);
  xyzz_add(A, D);                                                                   // sum_t t * S1_t
  for (uint32_t i = 0; i < t.m_log; i++) A = xyzz_dbl(A);
  xyzz_add(A, S);
  for (uint32_t j = 0; j < t.nbr; j++) xyzz_add(A, part[2 * t.nbr + 2 * t.nbc + j]);  // sum_t W1_t
  return A;
}

#if defined(__CUDACC__) && defined(SPB_MSM_KERNELS)
// ---- kernels --------------------------------------------------------------------------------------------
// The accumulation and every later kernel read the number of sorted entries M from device memory (the entry total the
// digit kernel counts); the host reads it once per MSM, to give the radix sort its length.
//
// Step 1: one scalar per thread, 256 threads per block. The block's entries form one range reserved by ONE atomic on the
// entry total (one atomic per warp would put eight times as many on that single address); inside it every warp writes its
// entries window by window, so each store instruction of a warp covers consecutive entries. Digits are derived twice from the
// canonical scalar (count, then write): shifts only, the Montgomery conversion is done once.
static const unsigned kDigitsThreads = 256;
__global__ void __launch_bounds__(kDigitsThreads) msm_digits_kernel(uint64_t n, const Fr* scalars, MsmGeom g, uint32_t* total, MsmEntry* ent) {
  __shared__ uint32_t s_warp[kDigitsThreads / 32];
  __shared__ uint32_t s_base;
  const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  bool live = tid < n;
  Fr s = live ? fp_from_mont(scalars[tid]) : fp_zero<FrParams>();
  live = live && !fp_is_zero(s);
  uint32_t wsum = live ? msm_digit_count(s, g) : 0u;
  for (int o = 16; o; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
  if (lane == 0) s_warp[warp] = wsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (unsigned i = 0; i < kDigitsThreads / 32; i++) { const uint32_t v = s_warp[i]; s_warp[i] = run; run += v; }
    s_base = run ? atomicAdd(total, run) : 0u;
  }
  __syncthreads();
  uint32_t pos = s_base + s_warp[warp];
  DigitIter it; it.init(s, g.c);
  for (uint32_t w = 0; w < g.W; w++) {
    const int32_t d = it.next();
    const bool act = live && d != 0;
    const unsigned m = __ballot_sync(0xffffffffu, act);
    if (act) ent[pos + (uint32_t)__popc(m & ((1u << lane) - 1u))] = msm_make_entry(tid, w, d, g);
    pos += (uint32_t)__popc(m);
  }
}
// Step 3: one thread per bucket k in [0, nb].
__global__ void __launch_bounds__(256) msm_offsets_kernel(const uint32_t* total, uint64_t nb, const MsmEntry* sorted, uint32_t* offsets) {
  msm_offsets_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, nb, *total, sorted, offsets);
}
#ifndef SPB_ACC_MINBLOCKS
#define SPB_ACC_MINBLOCKS 1
#endif
__global__ void __launch_bounds__(128, SPB_ACC_MINBLOCKS) msm_accumulate_kernel(const uint32_t* total, MsmGeom g, const MsmEntry* ent,
                                                             const G1Affine* bases, G1Xyzz* buckets, uint32_t* head_key, G1Xyzz* head,
                                                             uint32_t* tail_key, G1Xyzz* tail) {
  msm_accumulate_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, *total, g, ent, bases, buckets, head_key, head, tail_key, tail);
}
__global__ void __launch_bounds__(128) msm_stitch_kernel(const uint32_t* total, uint32_t L, uint32_t cap, const uint32_t* head_key, const G1Xyzz* head,
                                                         const uint32_t* tail_key, const G1Xyzz* tail, G1Xyzz* buckets, uint32_t* giant_count, uint32_t* giant_list) {
  L = msm_effective_chunk(L, *total);
  uint64_t T = ((uint64_t)*total + L - 1) / L;
  msm_stitch_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, T, cap, head_key, head, tail_key, tail, buckets, giant_count, giant_list);
}

// block-wide sum of NT points held one per thread; result in thread 0's `v`
template <int NT>
__device__ void block_sum_xyzz(G1Xyzz& v, G1Xyzz* sh) {
  const int tid = threadIdx.x;
  for (int stride = NT / 2; stride >= 1; stride >>= 1) {
    if (tid >= stride && tid < 2 * stride) sh[tid - stride] = v;
    __syncthreads();
    if (tid < stride) xyzz_add(v, sh[tid]);
    __syncthreads();
  }
}

// same for two points per thread at once (one pass of barriers instead of two)
template <int NT>
__device__ void block_sum2_xyzz(G1Xyzz& a, G1Xyzz& b, G1Xyzz* sh /* NT entries */) {
  const int tid = threadIdx.x;
  for (int stride = NT / 2; stride >= 1; stride >>= 1) {
    if (tid >= stride && tid < 2 * stride) { sh[2 * (tid - stride)] = a; sh[2 * (tid - stride) + 1] = b; }
    __syncthreads();
    if (tid < stride) { xyzz_add(a, sh[2 * tid]); xyzz_add(b, sh[2 * tid + 1]); }
    __syncthreads();
  }
}

// giant chains (queued by the stitch kernel): one block per chain, grid-stride over the queue. Chains with more than
// kHugeChain links (a column of equal scalars puts n/32 pieces into one bucket) are handed on to the huge-chain
// kernels, which spread ONE chain over the whole grid.
static const uint32_t kHugeChain = 4096;
static const uint32_t kHugeBlocks = 1056;   // 8 CTAs of 128 threads per SM on 132 SMs (H100 SXM)
__global__ void __launch_bounds__(128) msm_giant_kernel(const uint32_t* total, uint32_t L, const uint32_t* giant_count, const uint32_t* giant_list,
                                                        const uint32_t* head_key, const G1Xyzz* head, const uint32_t* tail_key, const G1Xyzz* tail,
                                                        G1Xyzz* buckets, uint32_t* huge_count, uint32_t* huge_list /* pairs: t0, end */) {
  __shared__ G1Xyzz sh[64];
  __shared__ uint64_t s_end;
  L = msm_effective_chunk(L, *total);
  const uint64_t T = ((uint64_t)*total + L - 1) / L;
  const uint32_t count = *giant_count;
  for (uint32_t gi = blockIdx.x; gi < count; gi += gridDim.x) {
    uint64_t t0 = giant_list[gi];
    uint32_t key = tail_key[t0];
    if (threadIdx.x == 0) {
      // links are head[t0+1 .. end): keys are sorted, so "head_key[j] == key" is true on that range and never again
      uint64_t lo = t0 + 1, hi = T;
      while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (head_key[mid] == key) lo = mid + 1; else hi = mid; }
      s_end = lo;
    }
    __syncthreads();
    const uint64_t end = s_end;
    if (end - (t0 + 1) > kHugeChain) {
      if (threadIdx.x == 0) { uint32_t slot = atomicAdd(huge_count, 1u); huge_list[2 * slot] = (uint32_t)t0; huge_list[2 * slot + 1] = (uint32_t)end; }
      __syncthreads();
      continue;
    }
    G1Xyzz acc = xyzz_identity();
    for (uint64_t j = t0 + 1 + threadIdx.x; j < end; j += 128) xyzz_add(acc, head[j]);
    block_sum_xyzz<128>(acc, sh);
    if (threadIdx.x == 0) { xyzz_add(acc, tail[t0]); buckets[key] = acc; }
    __syncthreads();
  }
}
// The huge chains share the grid: with `count` chains every chain gets nparts = gridDim / count blocks (all of them when there is
// one chain, one block each when there are more chains than blocks); block `work` sums a strided share of its chain's pieces
// -> partial[chain * gridDim + part]. All chains proceed at once (a column of equal scalars makes one huge chain per window).
__global__ void __launch_bounds__(128) msm_huge_kernel(const uint32_t* huge_count, const uint32_t* huge_list, const G1Xyzz* head, G1Xyzz* partial) {
  __shared__ G1Xyzz sh[64];
  const uint32_t count = *huge_count;
  if (!count) return;
  const uint32_t nparts = gridDim.x / count ? gridDim.x / count : 1;
  for (uint64_t work = blockIdx.x; work < (uint64_t)count * nparts; work += gridDim.x) {
    const uint32_t hi = (uint32_t)(work / nparts), part = (uint32_t)(work % nparts);
    const uint64_t t0 = huge_list[2 * hi], end = huge_list[2 * hi + 1];
    G1Xyzz acc = xyzz_identity();
    for (uint64_t j = t0 + 1 + (uint64_t)part * 128 + threadIdx.x; j < end; j += (uint64_t)nparts * 128) xyzz_add(acc, head[j]);
    block_sum_xyzz<128>(acc, sh);
    if (threadIdx.x == 0) partial[(uint64_t)hi * gridDim.x + part] = acc;
    __syncthreads();
  }
}
// one block per huge chain: fold its per-part partials and the chain's tail piece into the bucket (grid_parts = the grid of msm_huge_kernel)
__global__ void __launch_bounds__(128) msm_huge_finish_kernel(const uint32_t* huge_count, const uint32_t* huge_list, uint32_t grid_parts, const G1Xyzz* partial,
                                                              const uint32_t* tail_key, const G1Xyzz* tail, G1Xyzz* buckets) {
  __shared__ G1Xyzz sh[64];
  const uint32_t count = *huge_count;
  if (!count) return;
  const uint32_t nparts = grid_parts / count ? grid_parts / count : 1;
  for (uint32_t hi = blockIdx.x; hi < count; hi += gridDim.x) {
    G1Xyzz acc = xyzz_identity();
    for (uint32_t j = threadIdx.x; j < nparts; j += 128) xyzz_add(acc, partial[(uint64_t)hi * grid_parts + j]);
    block_sum_xyzz<128>(acc, sh);
    const uint64_t t0 = huge_list[2 * hi];
    if (threadIdx.x == 0) { xyzz_add(acc, tail[t0]); buckets[tail_key[t0]] = acc; }
    __syncthreads();
  }
}

// (a) one thread per group of 2^m_log buckets
__global__ void __launch_bounds__(128) msm_group_kernel(uint64_t ngroups, uint32_t m_log, const uint32_t* offsets, const G1Xyzz* buckets, G1Xyzz* s1, G1Xyzz* w1) {
  msm_group_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, ngroups, m_log, offsets, buckets, s1, w1);
}
// (b) block (w, idx): idx < R -> row sum of S1, idx < R + C -> column sum of S1, else row sum of W1
// 64 threads per vector: more serial additions per thread and a shorter tree keep more lanes busy than 128 would
__global__ void __launch_bounds__(64) msm_rowcol_kernel(uint32_t T, MsmTail t, const G1Xyzz* s1, const G1Xyzz* w1, G1Xyzz* row_out, G1Xyzz* col_out, G1Xyzz* wrow_out) {
  __shared__ G1Xyzz sh[32];
  const uint32_t R = 1u << t.r_log, C = 1u << t.c_log;
  const uint32_t w = blockIdx.x / (2 * R + C), idx = blockIdx.x % (2 * R + C);
  const G1Xyzz* X = (idx < R + C ? s1 : w1) + (uint64_t)w * T;
  G1Xyzz acc = xyzz_identity();
  if (idx < R) { for (uint32_t c = threadIdx.x; c < C; c += 64) xyzz_add(acc, X[(uint64_t)idx * C + c]); }
  else if (idx < R + C) { const uint32_t col = idx - R; for (uint32_t r = threadIdx.x; r < R; r += 64) xyzz_add(acc, X[(uint64_t)r * C + col]); }
  else { const uint32_t row = idx - R - C; for (uint32_t c = threadIdx.x; c < C; c += 64) xyzz_add(acc, X[(uint64_t)row * C + c]); }
  block_sum_xyzz<64>(acc, sh);
  if (threadIdx.x == 0) {
    if (idx < R) row_out[(uint64_t)w * R + idx] = acc;
    else if (idx < R + C) col_out[(uint64_t)w * C + (idx - R)] = acc;
    else wrow_out[(uint64_t)w * R + (idx - R - C)] = acc;
  }
}
// block (w, j): j < nbr -> rows [128 j, 128 j + 128), j < nbr + nbc -> columns, else the W1 row sums (plain sum only).
// Local weighted sum without any scalar multiple: sum_i i * X_i = sum_{i >= 1} (suffix sum S_i), so one suffix scan
// (7 steps) and one tree sum (7 steps).
__global__ void __launch_bounds__(128) msm_weighted_kernel(MsmTail t, const G1Xyzz* row_out, const G1Xyzz* col_out, const G1Xyzz* wrow_out, G1Xyzz* partials) {
  __shared__ G1Xyzz sh[128];
  __shared__ G1Xyzz sh2[64];
  const uint32_t R = 1u << t.r_log, C = 1u << t.c_log, per = msm_tail_partials(t);
  const uint32_t nblk = 2 * t.nbr + t.nbc;
  const uint32_t w = blockIdx.x / nblk, j = blockIdx.x % nblk;
  const int kind = j < t.nbr ? 0 : (j < t.nbr + t.nbc ? 1 : 2);
  const uint32_t jb = kind == 0 ? j : (kind == 1 ? j - t.nbr : j - t.nbr - t.nbc), idx = jb * 128 + threadIdx.x, tid = threadIdx.x;
  G1Xyzz* out = partials + (uint64_t)w * per;
  G1Xyzz x = xyzz_identity();
  if (kind == 0) { if (idx < R) x = row_out[(uint64_t)w * R + idx]; }
  else if (kind == 1) { if (idx < C) x = col_out[(uint64_t)w * C + idx]; }
  else { if (idx < R) x = wrow_out[(uint64_t)w * R + idx]; }
  if (kind == 2) {   // plain sum
    block_sum_xyzz<128>(x, sh2);
    if (tid == 0) out[2 * t.nbr + 2 * t.nbc + jb] = x;
    return;
  }
  // inclusive suffix scan: x <- sum_{t >= tid} X_t
  for (uint32_t off = 1; off < 128; off <<= 1) {
    sh[tid] = x;
    __syncthreads();
    if (tid + off < 128) xyzz_add(x, sh[tid + off]);
    __syncthreads();
  }
  G1Xyzz total = x;                       // thread 0 holds the plain block sum
  if (tid == 0) x = xyzz_identity();      // weights start at 0: drop S_0 from the weighted sum
  block_sum_xyzz<128>(x, sh2);
  if (tid == 0) {
    if (kind == 0) { out[jb] = x; out[t.nbr + jb] = total; }
    else { out[2 * t.nbr + jb] = x; out[2 * t.nbr + t.nbc + jb] = total; }
  }
}

// out[i] = scalars[i] * G1 (affine): plain double-and-add per thread + one inversion. Setup / test utility.
__global__ void __launch_bounds__(128) g1_fixed_base_mul_kernel(const Fr* scalars, uint64_t n, G1Affine* out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr s = fp_from_mont(scalars[i]);
  G1Affine gen; gen.x = fp_one<FqParams>(); gen.y = fp_dbl(gen.x);  // (1, 2)
  G1Xyzz acc = xyzz_identity();
  for (int b = 253; b >= 0; b--) {
    acc = xyzz_dbl(acc);
    if ((s.l[b >> 5] >> (b & 31)) & 1) xyzz_add_mixed(acc, gen);
  }
  out[i] = xyzz_to_affine(acc);
}

// scalars of ParamsKZG::setup: mode 0: out[i] = s^i ; mode 1: out[i] = coef * w^i / (s - w^i)  (L_i(s))
__global__ void srs_scalars_kernel(int mode, Fr s, Fr w, Fr coef, uint64_t start, uint64_t n, Fr* out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mode == 0) { out[i] = fp_pow_u64(s, start + i); return; }
  Fr wi = fp_pow_u64(w, start + i);
  out[i] = fp_mul(fp_mul(coef, wi), fp_inv(fp_sub(s, wi)));
}
#endif

// ---- ParamsKZG::downsize: g_to_lagrange = inverse DFT over the group ------------------------------------------------------
// k * P for a canonical (non-Montgomery) 254-bit scalar: MSB-first double-and-add
SPB_HD G1Xyzz xyzz_mul_scalar(const G1Xyzz& p, const Fr& k) {
  int top = 255;
  while (top >= 0 && !((k.l[top >> 5] >> (top & 31)) & 1)) top--;
  G1Xyzz r = xyzz_identity();
  for (int i = top; i >= 0; i--) {
    r = xyzz_dbl(r);
    if ((k.l[i >> 5] >> (i & 31)) & 1) xyzz_add(r, p);
  }
  return r;
}
// one decimation-in-frequency stage of the group DFT, butterfly `tid` of n/2: (a, b) <- (a + b, (a - b) * w^(j * stride)) with
// j = tid mod half. tw[i] = w^i (Montgomery), i < n/2. After log2 n stages the result sits in bit-reversed order.
SPB_HD void ec_ntt_stage_thread(uint64_t tid, uint64_t n, uint64_t half, const Fr* tw, G1Xyzz* p) {
  if (tid >= n / 2) return;
  const uint64_t j = tid & (half - 1), base = ((tid - j) << 1) + j, stride = (n / 2) / half;
  G1Xyzz a = p[base], b = p[base + half];
  G1Xyzz sum = a; xyzz_add(sum, b);
  G1Xyzz diff = a; xyzz_add(diff, xyzz_neg(b));
  p[base] = sum;
  p[base + half] = j == 0 ? diff : xyzz_mul_scalar(diff, fp_from_mont(tw[j * stride]));
}
// out[i] = scale * p[bitrev_k(i)] as an affine point (scale = 1/n, Montgomery)
SPB_HD void ec_ntt_finish_thread(uint64_t tid, uint64_t n, uint32_t k, const Fr& scale, const G1Xyzz* p, G1Affine* out) {
  if (tid >= n) return;
  uint64_t r = 0;
  for (uint32_t b = 0; b < k; b++) r |= ((tid >> b) & 1ull) << (k - 1 - b);
  out[tid] = xyzz_to_affine(xyzz_mul_scalar(p[r], fp_from_mont(scale)));
}

// ---- spb_srs_contribute: a powers-of-tau update g'[j] = t^j g[j] -----------------------------------------------------------
// point `tid` of a shard whose first point has global index `start`: out = t^(start + tid) in, affine. xyzz_mul_scalar's
// MSB-first double-and-add with mixed additions (the base is affine); the power is computed per thread (at most 2 log2 n
// products, against about 3800 for the multiple). The identity stays the identity.
SPB_HD void srs_scale_thread(uint64_t tid, uint64_t start, uint64_t n, const Fr& t, const G1Affine* in, G1Affine* out) {
  if (tid >= n) return;
  const Fr k = fp_from_mont(fp_pow_u64(t, start + tid));
  const G1Affine p = in[tid];
  int top = 255;
  while (top >= 0 && !((k.l[top >> 5] >> (top & 31)) & 1)) top--;
  G1Xyzz r = xyzz_identity();
  for (int i = top; i >= 0; i--) {
    r = xyzz_dbl(r);
    if ((k.l[i >> 5] >> (i & 31)) & 1) xyzz_add_mixed(r, p);
  }
  out[tid] = xyzz_to_affine(r);
}
#if defined(__CUDACC__) && defined(SPB_MSM_KERNELS)
__global__ void __launch_bounds__(128) srs_scale_kernel(uint64_t start, uint64_t n, Fr t, const G1Affine* in, G1Affine* out) {
  srs_scale_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, start, n, t, in, out);
}
__global__ void __launch_bounds__(128) ec_lift_kernel(uint64_t n, const G1Affine* in, G1Xyzz* out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = xyzz_from_affine(in[i]);
}
__global__ void __launch_bounds__(128) ec_ntt_stage_kernel(uint64_t n, uint64_t half, const Fr* tw, G1Xyzz* p) {
  ec_ntt_stage_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, n, half, tw, p);
}
__global__ void __launch_bounds__(128) ec_ntt_finish_kernel(uint64_t n, uint32_t k, Fr scale, const G1Xyzz* p, G1Affine* out) {
  ec_ntt_finish_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, n, k, scale, p, out);
}
__global__ void fr_powers_kernel(Fr* out, Fr base, uint64_t count) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < count) out[i] = fp_pow_u64(base, i);
}
#endif

// ---- step 7 (host): Horner over the bucket windows ------------------------------------------------------
inline G1Xyzz msm_combine_windows(const G1Xyzz* S, uint32_t BW, uint32_t c) {
  G1Xyzz acc = xyzz_identity();
  for (int w = (int)BW - 1; w >= 0; w--) {
    if (w != (int)BW - 1) for (uint32_t i = 0; i < c; i++) acc = xyzz_dbl(acc);
    xyzz_add(acc, S[w]);
  }
  return acc;
}

inline MsmGeom msm_make_geometry(uint32_t c, bool precomp, uint32_t tab_stride) {
  MsmGeom g;
  g.c = c; g.W = (255 + c - 1) / c; g.B = 1u << (c - 1); g.L = 32;
  g.precomp = precomp ? 1 : 0; g.BW = precomp ? 1 : g.W; g.tab_stride = tab_stride;
  return g;
}

// Window width minimising the modelled work in Montgomery products:
//   10 * n * W  (mixed additions)  +  2 * 14 * BW * 2^(c-1)  (running sums over the buckets, full additions)
// BW = W without precomputed tables, 1 with them (all windows share one bucket set).
inline uint32_t msm_choose_c(uint64_t n, bool precomp) {
  uint32_t best = 0; double best_cost = 0;
  for (uint32_t c = 3; c <= 22; c++) {
    uint32_t W = (255 + c - 1) / c;
    double cost = 10.0 * (double)n * W + 28.0 * (precomp ? 1.0 : (double)W) * (double)(1u << (c - 1));
    if (!best || cost < best_cost) { best = c; best_cost = cost; }
  }
  return best;
}
inline MsmGeom msm_choose_geometry(uint64_t n) { return msm_make_geometry(msm_choose_c(n, false), false, 0); }

// W-1 further table rows for point p: row j = 2^(c*j) * p, affine. Thread i handles base i.
SPB_HD void msm_precompute_thread(uint64_t tid, uint64_t count, uint32_t c, uint32_t W, G1Affine* table /* W rows of `count` */) {
  if (tid >= count) return;
  G1Xyzz p = xyzz_from_affine(table[tid]);
  for (uint32_t j = 1; j < W; j++) {
    for (uint32_t i = 0; i < c; i++) p = xyzz_dbl(p);
    table[(uint64_t)j * count + tid] = xyzz_to_affine(p);
  }
}
#if defined(__CUDACC__) && defined(SPB_MSM_KERNELS)
__global__ void __launch_bounds__(128) msm_precompute_kernel(uint64_t count, uint32_t c, uint32_t W, G1Affine* table) {
  msm_precompute_thread(blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, count, c, W, table);
}
#endif

}  // namespace spb
