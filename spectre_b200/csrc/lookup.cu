// Lookup argument, stage 4 of create_proof: permute_expression_pair on the device.
// Replaces [UPSTREAM] halo2_proofs/src/plonk/lookup/prover.rs::permute_expression_pair (SURVEY.md 8a row a8 / 8f rank 3:
// after MSM and NTT move to the GPU this sort + BTreeMap walk is the serial CPU tail of a proof).
// Same result as the CPU algorithm, element for element:
//   permuted_input  = the input values sorted by canonical integer (halo2curves' Ord for Fr),
//   permuted_table  = at the first row of each distinct input value that value; the remaining table elements
//                     (ascending) handed to the repeated rows from the LAST repeated row backwards.
// Built from data-parallel primitives: Montgomery -> canonical, a stable LSD radix sort over the four 64-bit limbs carrying row
// indices (this file's own counting-sort passes; only the exclusive scans are cub::DeviceScan), adjacent-difference flags, a
// binary search of every distinct input value in the sorted table, two exclusive scans and a scatter.
// Algorithmic bytes: 4 x 32 B per row (two columns in, two out).
#include "common.cuh"
#include "ntt.cuh"
#include <cub/device/device_scan.cuh>
#include <string.h>

using namespace spb;

// ---- stable LSD radix sort of (64-bit key, 32-bit row index) pairs: the sort that IS permute_expression_pair -------------
// Eight 8-bit digits per limb. One histogram kernel counts all eight digit positions at once; a digit on which every key
// agrees (range-check columns are < 2^20: five of their eight bytes, and three whole limbs, are zero) is skipped without a
// pass. A pass is a counting sort: per-tile digit histograms, one exclusive scan over (digit, tile), and a scatter that
// ranks keys inside a tile in their original order (warp match + per-warp digit counters), which is what makes it stable.
namespace {
const int kRsThreads = 256, kRsItems = 8, kRsTile = kRsThreads * kRsItems;   // keys per tile

__global__ void __launch_bounds__(kRsThreads) rs_hist_all_kernel(const unsigned long long* keys, uint64_t n, uint32_t* hist /* 8 x 256 */) {
  __shared__ uint32_t sh[8 * 256];
  for (int i = threadIdx.x; i < 8 * 256; i += kRsThreads) sh[i] = 0;
  __syncthreads();
  for (uint64_t i = blockIdx.x * (uint64_t)kRsThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kRsThreads) {
    const unsigned long long k = keys[i];
#pragma unroll
    for (int d = 0; d < 8; d++) atomicAdd(&sh[d * 256 + (uint32_t)((k >> (8 * d)) & 0xff)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * 256; i += kRsThreads) if (sh[i]) atomicAdd(&hist[i], sh[i]);
}
// tile_hist[digit * ntiles + tile] = keys of that tile with that digit
__global__ void __launch_bounds__(kRsThreads) rs_tile_hist_kernel(const unsigned long long* keys, uint64_t n, uint32_t shift, uint32_t ntiles, uint32_t* tile_hist) {
  __shared__ uint32_t sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t base = (uint64_t)blockIdx.x * kRsTile;
#pragma unroll
  for (int r = 0; r < kRsItems; r++) {
    const uint64_t i = base + (uint64_t)r * kRsThreads + threadIdx.x;
    if (i < n) atomicAdd(&sh[(uint32_t)((keys[i] >> shift) & 0xff)], 1u);
  }
  __syncthreads();
  tile_hist[(uint64_t)threadIdx.x * ntiles + blockIdx.x] = sh[threadIdx.x];
}
// offsets = exclusive scan of tile_hist; keys of one tile are taken in rounds of 256 (round-major = original order)
__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const unsigned long long* keys_in, const uint32_t* idx_in, unsigned long long* keys_out, uint32_t* idx_out,
                                                                uint64_t n, uint32_t shift, uint32_t ntiles, const uint32_t* offsets) {
  __shared__ uint32_t digit_base[256];          // next free output slot of each digit for this tile
  __shared__ uint32_t warp_count[8][256];       // this round: keys of each digit per warp -> exclusive prefix over the warps
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  digit_base[threadIdx.x] = offsets[(uint64_t)threadIdx.x * ntiles + blockIdx.x];
  const uint64_t base = (uint64_t)blockIdx.x * kRsTile;
  for (int r = 0; r < kRsItems; r++) {
    for (int w = 0; w < 8; w++) warp_count[w][threadIdx.x] = 0;
    __syncthreads();
    const uint64_t i = base + (uint64_t)r * kRsThreads + threadIdx.x;
    const bool live = i < n;
    unsigned long long k = 0; uint32_t v = 0, dgt = 0, rank = 0;
    if (live) { k = keys_in[i]; v = idx_in[i]; dgt = (uint32_t)((k >> shift) & 0xff); }
    const unsigned livemask = __ballot_sync(0xffffffffu, live);
    if (live) {
      const unsigned peers = __match_any_sync(livemask, dgt);
      rank = (uint32_t)__popc(peers & ((1u << lane) - 1u));
      if (rank == 0) warp_count[warp][dgt] = (uint32_t)__popc(peers);
    }
    __syncthreads();
    {   // thread d: exclusive prefix of digit d's counts over the 8 warps, then advance the digit's base by the round total
      uint32_t run = 0;
      for (int w = 0; w < 8; w++) { const uint32_t c = warp_count[w][threadIdx.x]; warp_count[w][threadIdx.x] = run; run += c; }
      const uint32_t b = digit_base[threadIdx.x];
      __syncthreads();
      if (live) { const uint32_t pos = digit_base[dgt] + warp_count[warp][dgt] + rank; keys_out[pos] = k; idx_out[pos] = v; }
      __syncthreads();
      digit_base[threadIdx.x] = b + run;
    }
    __syncthreads();
  }
}

// sorts (keys_a, idx_a) by key, ascending, stable; the result ends up back in keys_a / idx_a. `hist` (8 x 256 u32) and `tile_hist`
// (256 x ntiles + 1 u32, plus the scan's temp) are device scratch. One 8 KB D2H of the digit histograms per call.
int radix_sort_pairs_u64(spb_ctx* ctx, DeviceState& d, unsigned long long* keys_a, unsigned long long* keys_b, uint32_t* idx_a, uint32_t* idx_b, uint64_t n,
                         uint32_t* hist, uint32_t* tile_hist, void* scan_tmp, size_t scan_bytes) {
  const uint32_t ntiles = (uint32_t)((n + kRsTile - 1) / kRsTile);
  SPB_CUDA(ctx, cudaMemsetAsync(hist, 0, 8 * 256 * 4, d.stream));
  unsigned hb = ntiles < (unsigned)d.sm_count * 4 ? ntiles : (unsigned)d.sm_count * 4;
  SPB_TRY(launch(ctx, d.stream, hb ? hb : 1, kRsThreads, 0, rs_hist_all_kernel, keys_a, n, hist));
  uint32_t h[8 * 256];
  SPB_CUDA(ctx, cudaMemcpyAsync(h, hist, sizeof h, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  int passes = 0;
  for (int dg = 0; dg < 8; dg++) {
    bool trivial = false;
    for (int b = 0; b < 256; b++) if (h[dg * 256 + b] == n) trivial = true;
    if (trivial) continue;
    SPB_TRY(launch(ctx, d.stream, ntiles, kRsThreads, 0, rs_tile_hist_kernel, keys_a, n, 8 * dg, ntiles, tile_hist));
    SPB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, tile_hist, tile_hist, (int)(256 * ntiles), d.stream));
    SPB_TRY(launch(ctx, d.stream, ntiles, kRsThreads, 0, rs_scatter_kernel, keys_a, idx_a, keys_b, idx_b, n, 8 * dg, ntiles, tile_hist));
    unsigned long long* tk = keys_a; keys_a = keys_b; keys_b = tk;
    uint32_t* ti = idx_a; idx_a = idx_b; idx_b = ti;
    passes++;
  }
  if (passes & 1) {   // an odd number of passes left the result in the caller's b buffers
    SPB_CUDA(ctx, cudaMemcpyAsync(keys_b, keys_a, n * 8, cudaMemcpyDeviceToDevice, d.stream));
    SPB_CUDA(ctx, cudaMemcpyAsync(idx_b, idx_a, n * 4, cudaMemcpyDeviceToDevice, d.stream));
  }
  return 0;
}
}  // namespace

__global__ void lk_canon_kernel(const Fr* in, Fr* out, uint32_t* idx, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  ntt_stg(out + i, fp_from_mont(ntt_ldg(in + i)));
  idx[i] = (uint32_t)i;
}
__global__ void lk_gather_limb_kernel(const Fr* canon, const uint32_t* idx, uint32_t limb, unsigned long long* keys, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr& v = canon[idx[i]];
  keys[i] = ((unsigned long long)v.l[2 * limb + 1] << 32) | v.l[2 * limb];
}
__global__ void lk_gather_kernel(const Fr* canon, const uint32_t* idx, Fr* sorted, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(sorted + i, ntt_ldg(canon + idx[i]));
}
__device__ __forceinline__ int lk_cmp(const Fr& a, const Fr& b) {
  for (int i = 7; i >= 0; i--) { if (a.l[i] != b.l[i]) return a.l[i] < b.l[i] ? -1 : 1; }
  return 0;
}
// first[i] = 1 on the first row of each distinct sorted input value; those rows look their value up in the sorted table
__global__ void lk_match_kernel(const Fr* sin, const Fr* stb, uint64_t n, uint32_t* repeated_flag, uint32_t* used, int* error) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr v = ntt_ldg(sin + i);
  bool first = i == 0 || lk_cmp(v, ntt_ldg(sin + i - 1)) != 0;
  repeated_flag[i] = first ? 0u : 1u;
  if (!first) return;
  uint64_t lo = 0, hi = n;
  while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (lk_cmp(ntt_ldg(stb + mid), v) < 0) lo = mid + 1; else hi = mid; }
  if (lo >= n || lk_cmp(ntt_ldg(stb + lo), v) != 0) { atomicExch(error, 1); return; }
  used[lo] = 1u;   // distinct values hit distinct first occurrences
}
__global__ void lk_leftover_flag_kernel(const uint32_t* used, uint32_t* left_flag, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) left_flag[i] = used[i] ? 0u : 1u;
}
// rep_rows[rank] = row for repeated rows; first rows get permuted_table = value
__global__ void lk_emit_input_kernel(const Fr* sin, const uint32_t* repeated_flag, const uint32_t* rep_rank, uint32_t* rep_rows, Fr* pin, Fr* ptab, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr m = fp_to_mont(ntt_ldg(sin + i));
  ntt_stg(pin + i, m);
  if (repeated_flag[i]) rep_rows[rep_rank[i]] = (uint32_t)i;
  else ntt_stg(ptab + i, m);
}
// leftover element of ascending rank r goes to the repeated row of rank m-1-r
__global__ void lk_emit_leftover_kernel(const Fr* stb, const uint32_t* left_flag, const uint32_t* left_rank, const uint32_t* rep_rows, uint32_t m, Fr* ptab, uint64_t n) {
  uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j >= n || !left_flag[j]) return;
  uint32_t r = left_rank[j];
  if (r >= m) return;
  ntt_stg(ptab + rep_rows[m - 1 - r], fp_to_mont(ntt_ldg(stb + j)));
}

namespace spb {
int lookup_work(spb_ctx* ctx, DeviceState& d, uint64_t n, LookupWork* w) {
  w->canon = (Fr*)slot(ctx, d, "lk_canon", n * 32);
  w->sin = (Fr*)slot(ctx, d, "lk_sin", n * 32);
  w->stb = (Fr*)slot(ctx, d, "lk_stb", n * 32);
  w->idx_a = (uint32_t*)slot(ctx, d, "lk_idx_a", n * 4);
  w->idx_b = (uint32_t*)slot(ctx, d, "lk_idx_b", n * 4);
  w->keys_a = (unsigned long long*)slot(ctx, d, "lk_keys_a", n * 8);
  w->keys_b = (unsigned long long*)slot(ctx, d, "lk_keys_b", n * 8);
  w->flags = (uint32_t*)slot(ctx, d, "lk_flags", (4 * n + 8) * 4);   // permute_expression_pair: repeated_flag | rep_rank | used->left_flag | left_rank
  w->err = (int*)slot(ctx, d, "lk_err", 16);
  const uint32_t ntiles = (uint32_t)((n + kRsTile - 1) / kRsTile);
  w->rs_hist = (uint32_t*)slot(ctx, d, "lk_rs_hist", 8 * 256 * 4);
  w->rs_tile = (uint32_t*)slot(ctx, d, "lk_rs_tile", ((size_t)256 * ntiles + 1) * 4);
  size_t scan_a = 0, scan_b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_a, w->flags, w->flags, (int)n + 1, d.stream);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, w->rs_tile, w->rs_tile, (int)(256 * ntiles), d.stream);
  w->tmp_bytes = scan_a > scan_b ? scan_a : scan_b;
  w->tmp = slot(ctx, d, "lk_tmp", w->tmp_bytes ? w->tmp_bytes : 16);
  if (!w->canon || !w->sin || !w->stb || !w->idx_a || !w->idx_b || !w->keys_a || !w->keys_b || !w->flags || !w->err || !w->tmp || !w->rs_hist || !w->rs_tile)
    return SPB_ERR_OOM;
  return 0;
}

int sort_canonical(spb_ctx* ctx, DeviceState& d, const LookupWork& w, const Fr* src, Fr* sorted, uint64_t n) {
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_canon_kernel, src, w.canon, w.idx_a, n));
  for (uint32_t limb = 0; limb < 4; limb++) {
    SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_gather_limb_kernel, w.canon, w.idx_a, limb, w.keys_a, n));
    SPB_TRY(radix_sort_pairs_u64(ctx, d, w.keys_a, w.keys_b, w.idx_a, w.idx_b, n, w.rs_hist, w.rs_tile, w.tmp, w.tmp_bytes));   // result back in keys_a / idx_a
  }
  return launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_gather_kernel, w.canon, w.idx_a, sorted, n);
}
}  // namespace spb

extern "C" {

int spb_permute_expression_pair_dev(spb_ctx* ctx, const spb_fr* d_input, const spb_fr* d_table, size_t usable, spb_fr* d_permuted_input, spb_fr* d_permuted_table) {
  if (!ctx || (usable && (!d_input || !d_table || !d_permuted_input || !d_permuted_table))) return SPB_ERR_ARG;
  if (!usable) return 0;
  if (usable >= 0x7fffffffull) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  const uint64_t n = usable;
  LookupWork w;
  SPB_TRY(lookup_work(ctx, d, n, &w));
  Fr* sin = w.sin, *stb = w.stb;
  uint32_t* flags = w.flags, *used = flags + 2 * (n + 1);
  void* tmp = w.tmp;
  size_t tmp_bytes = w.tmp_bytes;
  int* err = w.err;
  uint32_t* repeated_flag = flags, *rep_rank = flags + (n + 1), *left_rank = flags + 3 * (n + 1);

  SPB_TRY(sort_canonical(ctx, d, w, (const Fr*)d_input, sin, n));
  SPB_TRY(sort_canonical(ctx, d, w, (const Fr*)d_table, stb, n));
  SPB_CUDA(ctx, cudaMemsetAsync(flags, 0, (4 * n + 8) * 4, d.stream));
  SPB_CUDA(ctx, cudaMemsetAsync(err, 0, 4, d.stream));
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_match_kernel, sin, stb, n, repeated_flag, used, err));
  SPB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, repeated_flag, rep_rank, (int)n + 1, d.stream));   // rep_rank[n] = #repeated
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_leftover_flag_kernel, used, used, n));                   // in place: used -> left_flag
  SPB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, used, left_rank, (int)n + 1, d.stream));            // left_rank[n] = #leftover
  uint32_t counts[2] = {0, 0}; int herr = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&counts[0], rep_rank + n, 4, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(&counts[1], left_rank + n, 4, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(&herr, err, 4, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  if (herr || counts[0] != counts[1]) return set_error(ctx, SPB_ERR_CONSTRAINT, "permute_expression_pair: an input value does not occur in the table (ConstraintSystemFailure)");
  uint32_t* rep_rows = w.idx_b;   // free again
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_emit_input_kernel, sin, repeated_flag, rep_rank, rep_rows, (Fr*)d_permuted_input, (Fr*)d_permuted_table, n));
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lk_emit_leftover_kernel, stb, used, left_rank, rep_rows, counts[0], (Fr*)d_permuted_table, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

}  // extern "C"
