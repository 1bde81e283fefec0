// Batch polynomial arithmetic over Fr on the device: replaces halo2_proofs::arithmetic::{eval_polynomial,
// kate_division, parallelize-d axpy/scale loops} and ff::BatchInvert as used by plonk::{permutation, lookup,
// vanishing} and the SHPLONK opener ([UPSTREAM] halo2_proofs/src/arithmetic.rs, src/plonk/permutation/prover.rs,
// src/poly/kzg/multiopen/shplonk/prover.rs; SURVEY.md 8a rows a8-a10). All are HBM-streaming passes:
// algorithmic bytes = 64 B/element (read + write), 32 B/element for the reductions.
//
// The three scans (grand product, Kate division, batch inversion) are chunked three-phase scans, all on the device:
// per-chunk partials, a carry pass over the chunk partials (one block: prefix product / suffix scan of affine maps;
// batch inversion needs none -- every chunk inverts its own product), and a fix-up pass. Element order and results
// are exactly the serial CPU recurrences'.
#include "common.cuh"
#include "ntt.cuh"
#include <string.h>

using namespace spb;

static const uint32_t kChunk = 64;        // batch inversion: one Fermat inversion per chunk (2^20 rows: 16384 chains of 64; ncu: 256-long chains left the SMs 93 % idle)
static const uint32_t kScanChunk = 64;    // grand product / Kate division: short serial chains, carries scanned on the device

__global__ void vec_mul_kernel(Fr* a, const Fr* b, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(a + i, fp_mul(ntt_ld_stream(a + i), ntt_ld_stream(b + i)));
}
__global__ void vec_axpy_kernel(Fr* y, Fr alpha, const Fr* x, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(y + i, fp_add(ntt_ld_stream(y + i), fp_mul(alpha, ntt_ld_stream(x + i))));
}
__global__ void vec_scale_kernel(Fr* a, Fr alpha, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(a + i, fp_mul(alpha, ntt_ld_stream(a + i)));
}

// ---- grand product -------------------------------------------------------------------------------------------
__global__ void chunk_product_kernel(const Fr* a, uint64_t n, Fr* partial) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t lo = c * kScanChunk;
  if (lo >= n) return;
  uint64_t hi = lo + kScanChunk < n ? lo + kScanChunk : n;
  Fr p = fp_one<FrParams>();
  for (uint64_t i = lo; i < hi; i++) p = fp_mul(p, ntt_ldg(a + i));
  partial[c] = p;
}
// z[i] = init * carry[c] * prod_{lo <= j < i} a[j]
__global__ void chunk_product_fix_kernel(const Fr* a, uint64_t n, const Fr* carry, Fr init, Fr* z) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t lo = c * kScanChunk;
  if (lo >= n) return;
  uint64_t hi = lo + kScanChunk < n ? lo + kScanChunk : n;
  Fr p = fp_mul(carry[c], init);
  for (uint64_t i = lo; i < hi; i++) { Fr v = ntt_ldg(a + i); ntt_stg(z + i, p); p = fp_mul(p, v); }
}

// ---- Kate division: q[i] = a[i+1] + b*q[i+1], q has n-1 entries ----------------------------------------------
// with_store = 0: only the chunk head q[lo] (carry-in 0) is produced; 1: full chunk with the true carry-in.
__global__ void kate_chunk_kernel(const Fr* a, uint64_t nq, Fr b, const Fr* carry_in, Fr* heads, Fr* q, int with_store) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t lo = c * kScanChunk;
  if (lo >= nq) return;
  uint64_t hi = lo + kScanChunk < nq ? lo + kScanChunk : nq;
  Fr t = with_store ? carry_in[c] : fp_zero<FrParams>();
  for (uint64_t i = hi; i-- > lo;) {
    t = fp_add(ntt_ldg(a + i + 1), fp_mul(b, t));
    if (with_store) ntt_stg(q + i, t);
  }
  if (!with_store) heads[c] = t;
}

// ---- carry passes of the two scans, one block of 1024 threads (the partial arrays are n / 64 long) ---------------
// part[c] <- prod_{c' < c} part[c']   (exclusive prefix product, in place)
__global__ void __launch_bounds__(1024) carry_product_kernel(Fr* part, uint64_t m) {
  __shared__ Fr sh[1024];
  const uint32_t tid = threadIdx.x;
  const uint64_t per = (m + 1023) / 1024, lo = tid * per, hi = lo + per < m ? lo + per : m;
  Fr local = fp_one<FrParams>();
  for (uint64_t i = lo; i < hi; i++) local = fp_mul(local, part[i]);
  sh[tid] = local;
  __syncthreads();
  for (uint32_t off = 1; off < 1024; off <<= 1) {           // inclusive Hillis-Steele scan
    Fr v = sh[tid];
    if (tid >= off) v = fp_mul(sh[tid - off], v);
    __syncthreads();
    sh[tid] = v;
    __syncthreads();
  }
  Fr run = tid ? sh[tid - 1] : fp_one<FrParams>();
  for (uint64_t i = lo; i < hi; i++) { Fr t = part[i]; part[i] = run; run = fp_mul(run, t); }
}
// out[0] = prod of part[0..m): one block (row-sharded grand products exchange this one value per rank, SURVEY.md 8e)
__global__ void __launch_bounds__(1024) total_product_kernel(const Fr* part, uint64_t m, Fr* out) {
  __shared__ Fr sh[1024];
  const uint32_t tid = threadIdx.x;
  Fr local = fp_one<FrParams>();
  for (uint64_t i = tid; i < m; i += 1024) local = fp_mul(local, part[i]);
  sh[tid] = local;
  __syncthreads();
  for (uint32_t stride = 512; stride >= 1; stride >>= 1) {
    if (tid < stride) sh[tid] = fp_mul(sh[tid], sh[tid + stride]);
    __syncthreads();
  }
  if (tid == 0) out[0] = sh[0];
}
// Kate: chunk recurrence t_c = head_c + B_c * t_{c+1}, t_m = 0, B_c = b^64 except the last chunk (b_last).
// carry[c] <- t_{c+1}. Affine maps (H, B): t_lo = H + B * t_hi compose associatively, scanned from the right.
__global__ void __launch_bounds__(512) carry_kate_kernel(const Fr* heads, Fr* carry, uint64_t m, Fr b_chunk, Fr b_last) {
  __shared__ Fr shH[512];
  __shared__ Fr shB[512];
  const uint32_t tid = threadIdx.x;
  const uint64_t per = (m + 511) / 512, lo = tid * per, hi = lo + per < m ? lo + per : m;
  Fr H = fp_zero<FrParams>(), B = fp_one<FrParams>();      // identity map
  for (uint64_t c = hi; c-- > lo;) {                         // prepend chunk c: t_c = head_c + B_c * (H + B * t_hi)
    Fr Bc = (c == m - 1) ? b_last : b_chunk;
    H = fp_add(heads[c], fp_mul(Bc, H));
    B = fp_mul(Bc, B);
  }
  shH[tid] = H; shB[tid] = B;
  __syncthreads();
  for (uint32_t off = 1; off < 512; off <<= 1) {            // inclusive suffix scan of map composition
    Fr h = shH[tid], bb = shB[tid];
    if (tid + off < 512) { h = fp_add(h, fp_mul(bb, shH[tid + off])); bb = fp_mul(bb, shB[tid + off]); }
    __syncthreads();
    shH[tid] = h; shB[tid] = bb;
    __syncthreads();
  }
  // value entering this thread's range from the right: t_{hi} = H-component of the suffix starting at tid+1 (t_m = 0)
  Fr t = (tid + 1 < 512) ? shH[tid + 1] : fp_zero<FrParams>();
  for (uint64_t c = hi; c-- > lo;) {
    carry[c] = t;
    Fr Bc = (c == m - 1) ? b_last : b_chunk;
    t = fp_add(heads[c], fp_mul(Bc, t));
  }
}

// ---- batch inversion (zeros stay zero) ----------------------------------------------------------------------------
// phase 1: prefix products inside a chunk skipping zeros -> scratch, chunk product -> partial
__global__ void inv_chunk_prefix_kernel(const Fr* a, uint64_t n, Fr* scratch, Fr* partial) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t lo = c * kChunk;
  if (lo >= n) return;
  uint64_t hi = lo + kChunk < n ? lo + kChunk : n;
  Fr p = fp_one<FrParams>();
  for (uint64_t i = lo; i < hi; i++) { ntt_stg(scratch + i, p); Fr v = ntt_ldg(a + i); if (!fp_is_zero(v)) p = fp_mul(p, v); }
  partial[c] = p;
}
// phase 3: inv_total[c] = inverse of the chunk product
__global__ void inv_chunk_fix_kernel(Fr* a, uint64_t n, const Fr* scratch, const Fr* inv_total) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t lo = c * kChunk;
  if (lo >= n) return;
  uint64_t hi = lo + kChunk < n ? lo + kChunk : n;
  Fr run = inv_total[c];
  for (uint64_t i = hi; i-- > lo;) {
    Fr v = ntt_ldg(a + i);
    if (fp_is_zero(v)) continue;
    ntt_stg(a + i, fp_mul(run, ntt_ldg(scratch + i)));
    run = fp_mul(run, v);
  }
}
// one thread per chunk: plain Fermat inversion of the chunk product (n/256 inversions, fully parallel)
__global__ void inv_partials_kernel(Fr* partial, uint64_t m) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < m) partial[i] = fp_inv(partial[i]);
}

// ---- polynomial evaluation: p(x) = sum_t x^t * q_t(x^T), q_t = coefficients t, t+T, ... (coalesced Horner) ------
// T threads in blocks of 256; thread t runs the Horner of q_t, the block folds its 256 terms with a shared-memory tree. The
// block's partial sum is valid in thread 0.
__device__ __forceinline__ Fr eval_block_partial(const Fr* poly, uint64_t n, Fr x, Fr xT, uint32_t T) {
  __shared__ Fr sh[128];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  Fr acc = fp_zero<FrParams>();
  if (t < T && t < n) {
    uint64_t last = t + ((n - 1 - t) / T) * T;
    for (uint64_t i = last;; i -= T) { acc = fp_add(fp_mul(acc, xT), ntt_ldg(poly + i)); if (i < T) break; }
    acc = fp_mul(acc, fp_pow_u64(x, t));
  }
  for (int stride = 128; stride >= 1; stride >>= 1) {
    if ((int)threadIdx.x >= stride && (int)threadIdx.x < 2 * stride) sh[threadIdx.x - stride] = acc;
    __syncthreads();
    if ((int)threadIdx.x < stride) acc = fp_add(acc, sh[threadIdx.x]);
    __syncthreads();
  }
  return acc;
}
__global__ void __launch_bounds__(256) eval_strided_kernel(const Fr* poly, uint64_t n, Fr x, Fr xT, uint32_t T, Fr* partial) {
  Fr acc = eval_block_partial(poly, n, x, xT, T);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}
// the same for a whole list of (polynomial, point) queries in ONE launch: blockIdx.y = query (create_proof evaluates every
// opened polynomial at every queried rotation after squeezing x: 153 queries in the sync-step shape)
__global__ void __launch_bounds__(256) eval_many_kernel(const Fr* const* polys, const Fr* xs /* (x, x^T) per query */, uint64_t n, uint32_t T, Fr* partial) {
  const uint32_t q = blockIdx.y;
  Fr acc = eval_block_partial(polys[q], n, xs[2 * q], xs[2 * q + 1], T);
  if (threadIdx.x == 0) partial[(uint64_t)q * gridDim.x + blockIdx.x] = acc;
}

// out[i] = sum_p y^p * polys[p][i]  evaluated as Horner over p from the last polynomial down (the "fold with powers
// of y" that evaluate_h, vanishing::evaluate and the SHPLONK opener all do): reads each polynomial once.
__global__ void lincomb_kernel(const Fr* const* polys, uint32_t count, Fr y, Fr* out, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr acc = ntt_ld_stream(polys[count - 1] + i);
  for (int p = (int)count - 2; p >= 0; p--) acc = fp_add(fp_mul(acc, y), ntt_ld_stream(polys[p] + i));
  ntt_stg(out + i, acc);
}

namespace spb {

// ---- device-resident cores (all pointers on device d, work enqueued on d.stream; no final synchronisation unless noted)
static int dev_vec_mul(spb_ctx* ctx, DeviceState& d, Fr* da, const Fr* db, size_t n) {
  return launch(ctx, d.stream, nblk(n, 256), 256, 0, vec_mul_kernel, da, db, n);
}
static int dev_vec_axpy(spb_ctx* ctx, DeviceState& d, Fr* dy, const Fr& alpha, const Fr* dx, size_t n) {
  return launch(ctx, d.stream, nblk(n, 256), 256, 0, vec_axpy_kernel, dy, alpha, dx, n);
}
static int dev_vec_scale(spb_ctx* ctx, DeviceState& d, Fr* da, const Fr& alpha, size_t n) {
  return launch(ctx, d.stream, nblk(n, 256), 256, 0, vec_scale_kernel, da, alpha, n);
}

int dev_grand_product(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, Fr* dz, const Fr& init) {
  size_t m = (n + kScanChunk - 1) / kScanChunk;
  Fr* dp = (Fr*)slot(ctx, d, "poly_partial", 2 * m * 32);
  if (!dp) return SPB_ERR_OOM;
  SPB_TRY(launch(ctx, d.stream, nblk(m, 128), 128, 0, chunk_product_kernel, da, n, dp));
  SPB_TRY(launch(ctx, d.stream, 1, 1024, 0, carry_product_kernel, dp, m));
  return launch(ctx, d.stream, nblk(m, 128), 128, 0, chunk_product_fix_kernel, da, n, dp, init, dz);
}

// product of da[0..n) -> *d_total (one Fr in device memory of d, in the slot "poly_total"); enqueue only
int dev_product_enqueue(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, Fr** d_total) {
  size_t m = (n + kScanChunk - 1) / kScanChunk;
  Fr* dp = (Fr*)slot(ctx, d, "poly_partial", 2 * m * 32);
  Fr* dt = (Fr*)slot(ctx, d, "poly_total", 32);
  if (!dp || !dt) return SPB_ERR_OOM;
  SPB_TRY(launch(ctx, d.stream, nblk(m, 128), 128, 0, chunk_product_kernel, da, n, dp));
  SPB_TRY(launch(ctx, d.stream, 1, 1024, 0, total_product_kernel, dp, m, dt));
  *d_total = dt;
  return 0;
}

int dev_kate_division(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, const Fr& bb, Fr* dq) {
  size_t nq = n - 1, m = (nq + kScanChunk - 1) / kScanChunk;
  Fr* dh = (Fr*)slot(ctx, d, "poly_partial", 2 * m * 32);
  if (!dh) return SPB_ERR_OOM;
  SPB_TRY(launch(ctx, d.stream, nblk(m, 128), 128, 0, kate_chunk_kernel, da, nq, bb, nullptr, dh, nullptr, 0));
  size_t last_len = nq - (m - 1) * kScanChunk;
  SPB_TRY(launch(ctx, d.stream, 1, 512, 0, carry_kate_kernel, dh, dh + m, m, fp_pow_u64(bb, kScanChunk), fp_pow_u64(bb, last_len)));
  return launch(ctx, d.stream, nblk(m, 128), 128, 0, kate_chunk_kernel, da, nq, bb, dh + m, nullptr, dq, 1);
}

int dev_batch_invert(spb_ctx* ctx, DeviceState& d, Fr* da, size_t n) {
  size_t m = (n + kChunk - 1) / kChunk;
  Fr* ds = (Fr*)slot(ctx, d, "poly_scratch", n * 32);
  Fr* dp = (Fr*)slot(ctx, d, "poly_partial", 2 * m * 32);
  if (!ds || !dp) return SPB_ERR_OOM;
  SPB_TRY(launch(ctx, d.stream, nblk(m, 64), 64, 0, inv_chunk_prefix_kernel, da, n, ds, dp));
  SPB_TRY(launch(ctx, d.stream, nblk(m, 64), 64, 0, inv_partials_kernel, dp, m));
  return launch(ctx, d.stream, nblk(m, 64), 64, 0, inv_chunk_fix_kernel, da, n, ds, dp);
}

int dev_eval_polynomial(spb_ctx* ctx, DeviceState& d, const Fr* dp, size_t n, const Fr& x, Fr* out_host) {
  // enough threads that each runs a short Horner chain (16 steps at n = 2^20), a multiple of the block size
  uint32_t T = 256;
  while (T < 65536 && (uint64_t)T * 16 < n) T <<= 1;
  const uint32_t blocks = T / 256;
  Fr* dpart = (Fr*)slot(ctx, d, "poly_partial", (size_t)blocks * 32 > 64 ? (size_t)blocks * 32 : 64);
  if (!dpart) return SPB_ERR_OOM;
  SPB_TRY(launch(ctx, d.stream, blocks, 256, 0, eval_strided_kernel, dp, n, x, fp_pow_u64(x, T), T, dpart));
  std::vector<Fr> part(blocks);
  SPB_CUDA(ctx, cudaMemcpyAsync(part.data(), dpart, (size_t)blocks * 32, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  Fr acc = fp_zero<FrParams>();
  for (uint32_t t = 0; t < blocks; t++) acc = fp_add(acc, part[t]);
  *out_host = acc;
  return 0;
}

}  // namespace spb

// ---- Fr::random from a ChaCha20 keystream, on the device -------------------------------------------------------------------
// out[i] = the (first + i)-th `Fr::random(&mut ChaCha20Rng::from_seed(seed))` draw ([UPSTREAM] rand_chacha ChaCha20Rng: djb
// variant, 64-bit block counter in words 12-13, stream id 0; halo2curves Fr::random = from_u512 of eight next_u64() draws =
// exactly keystream block first + i). from_u512(lo + 2^256 hi) = lo * R2 + hi * R3 in Montgomery arithmetic; both 256-bit
// halves are brought below r first (at most five conditional subtractions) because fp_mul takes reduced operands.
// create_proof draws its blinding rows and the vanishing argument's random polynomial from the caller's RNG (upstream passes
// OsRng at lightclient-circuits/src/util/circuit.rs:158,211): drawing the 2^k-coefficient polynomial here means it never
// crosses PCIe, and seeding the host-side CPU restatement identically reproduces the same proof bytes.
__device__ __forceinline__ uint32_t chacha_rotl(uint32_t v, int n) { return (v << n) | (v >> (32 - n)); }
#define SPB_CHACHA_QR(a, b, c, d) a += b; d ^= a; d = chacha_rotl(d, 16); c += d; b ^= c; b = chacha_rotl(b, 12); a += b; d ^= a; d = chacha_rotl(d, 8); c += d; b ^= c; b = chacha_rotl(b, 7);
struct ChaChaKey { uint32_t w[8]; };
__global__ void fr_random_chacha_kernel(ChaChaKey key, uint64_t first, uint64_t n, Fr* out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t counter = first + i;
  uint32_t s[16], x[16];
  s[0] = 0x61707865u; s[1] = 0x3320646eu; s[2] = 0x79622d32u; s[3] = 0x6b206574u;
#pragma unroll
  for (int j = 0; j < 8; j++) s[4 + j] = key.w[j];
  s[12] = (uint32_t)counter; s[13] = (uint32_t)(counter >> 32); s[14] = 0; s[15] = 0;
#pragma unroll
  for (int j = 0; j < 16; j++) x[j] = s[j];
#pragma unroll
  for (int r = 0; r < 10; r++) {
    SPB_CHACHA_QR(x[0], x[4], x[8], x[12]) SPB_CHACHA_QR(x[1], x[5], x[9], x[13]) SPB_CHACHA_QR(x[2], x[6], x[10], x[14]) SPB_CHACHA_QR(x[3], x[7], x[11], x[15])
    SPB_CHACHA_QR(x[0], x[5], x[10], x[15]) SPB_CHACHA_QR(x[1], x[6], x[11], x[12]) SPB_CHACHA_QR(x[2], x[7], x[8], x[13]) SPB_CHACHA_QR(x[3], x[4], x[9], x[14])
  }
  Fr lo, hi, r2, r3, m;
#pragma unroll
  for (int j = 0; j < 8; j++) { lo.l[j] = x[j] + s[j]; hi.l[j] = x[8 + j] + s[8 + j]; r2.l[j] = FrParams::r2(j); }
  { constexpr uint32_t v[8] = SPB_FR_R3;
#pragma unroll
    for (int j = 0; j < 8; j++) r3.l[j] = v[j]; }
#pragma unroll
  for (int j = 0; j < 8; j++) m.l[j] = FrParams::mod(j);
  // fp_sub(a, r) = a - r if a >= r, else a (the borrow adds r back): 2^256 < 5.3 r, so five rounds bring any 256-bit value below r
#pragma unroll
  for (int t = 0; t < 5; t++) { lo = fp_sub(lo, m); hi = fp_sub(hi, m); }
  out[i] = fp_add(fp_mul(lo, r2), fp_mul(hi, r3));
}

extern "C" {

// ---- element-wise -------------------------------------------------------------------------------------------------
int spb_vec_mul_dev(spb_ctx* ctx, spb_fr* d_a, const spb_fr* d_b, size_t n) {
  if (!ctx || !d_a || !d_b) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_vec_mul(ctx, d, (Fr*)d_a, (const Fr*)d_b, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_vec_axpy_dev(spb_ctx* ctx, spb_fr* d_y, const spb_fr* alpha, const spb_fr* d_x, size_t n) {
  if (!ctx || !d_y || !alpha || !d_x) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_vec_axpy(ctx, d, (Fr*)d_y, fr_load(alpha), (const Fr*)d_x, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_vec_scale_dev(spb_ctx* ctx, spb_fr* d_a, const spb_fr* alpha, size_t n) {
  if (!ctx || !d_a || !alpha) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_vec_scale(ctx, d, (Fr*)d_a, fr_load(alpha), n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_lincomb_dev(spb_ctx* ctx, const spb_fr* const* d_polys, size_t count, const spb_fr* y, spb_fr* d_out, size_t n) {
  if (!ctx || !d_polys || !count || !y || !d_out) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  const Fr** dptrs = (const Fr**)slot(ctx, d, "poly_ptrs", count * sizeof(void*));
  if (!dptrs) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaMemcpyAsync(dptrs, d_polys, count * sizeof(void*), cudaMemcpyHostToDevice, d.stream));
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, lincomb_kernel, dptrs, (uint32_t)count, fr_load(y), (Fr*)d_out, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

int spb_vec_mul(spb_ctx* ctx, spb_fr* a, const spb_fr* b, size_t n) {
  if (!ctx || !a || !b) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, a, a}, {"poly_b", n * 32, b, nullptr}},
                    [&](void* const* p) { return dev_vec_mul(ctx, d, (Fr*)p[0], (const Fr*)p[1], n); });
}
int spb_vec_axpy(spb_ctx* ctx, spb_fr* y, const spb_fr* alpha, const spb_fr* x, size_t n) {
  if (!ctx || !y || !alpha || !x) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, y, y}, {"poly_b", n * 32, x, nullptr}},
                    [&](void* const* p) { return dev_vec_axpy(ctx, d, (Fr*)p[0], fr_load(alpha), (const Fr*)p[1], n); });
}
int spb_vec_scale(spb_ctx* ctx, spb_fr* a, const spb_fr* alpha, size_t n) {
  if (!ctx || !a || !alpha) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, a, a}}, [&](void* const* p) { return dev_vec_scale(ctx, d, (Fr*)p[0], fr_load(alpha), n); });
}

// ---- scans --------------------------------------------------------------------------------------------------------
int spb_grand_product_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, spb_fr* d_z) {
  if (!ctx || !d_a || !d_z) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_grand_product(ctx, d, (const Fr*)d_a, n, (Fr*)d_z, fp_one<FrParams>()));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_grand_product(spb_ctx* ctx, const spb_fr* a, size_t n, spb_fr* z) {
  if (!ctx || !a || !z) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, a, nullptr}, {"poly_b", n * 32, nullptr, z}},
                    [&](void* const* p) { return dev_grand_product(ctx, d, (const Fr*)p[0], n, (Fr*)p[1], fp_one<FrParams>()); });
}

int spb_grand_product_seeded_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, const spb_fr* init, spb_fr* d_z) {
  if (!ctx || !d_a || !d_z || !init) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_grand_product(ctx, d, (const Fr*)d_a, n, (Fr*)d_z, fr_load(init)));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_product_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, spb_fr* out) {
  if (!ctx || !out || (n && !d_a)) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  Fr total = fp_one<FrParams>();
  if (n) {
    Fr* dt = nullptr;
    SPB_TRY(dev_product_enqueue(ctx, d, (const Fr*)d_a, n, &dt));
    SPB_CUDA(ctx, cudaMemcpyAsync(&total, dt, 32, cudaMemcpyDeviceToHost, d.stream));
    SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  }
  memcpy(out, &total, 32);
  return 0;
}

int spb_kate_division_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, const spb_fr* b, spb_fr* d_q) {
  if (!ctx || !d_a || !b || !d_q || n < 1) return SPB_ERR_ARG;
  if (n == 1) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_kate_division(ctx, d, (const Fr*)d_a, n, fr_load(b), (Fr*)d_q));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_kate_division(spb_ctx* ctx, const spb_fr* a, size_t n, const spb_fr* b, spb_fr* q) {
  if (!ctx || !a || !b || !q || n < 1) return SPB_ERR_ARG;
  if (n == 1) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, a, nullptr}, {"poly_b", n * 32, nullptr, q, 0, (n - 1) * 32}},
                    [&](void* const* p) { return dev_kate_division(ctx, d, (const Fr*)p[0], n, fr_load(b), (Fr*)p[1]); });
}

int spb_batch_invert_dev(spb_ctx* ctx, spb_fr* d_a, size_t n) {
  if (!ctx || !d_a) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  SPB_TRY(dev_batch_invert(ctx, d, (Fr*)d_a, n));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int spb_batch_invert(spb_ctx* ctx, spb_fr* a, size_t n) {
  if (!ctx || !a) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"poly_a", n * 32, a, a}}, [&](void* const* p) { return dev_batch_invert(ctx, d, (Fr*)p[0], n); });
}

int spb_eval_polynomial_dev(spb_ctx* ctx, const spb_fr* d_poly, size_t n, const spb_fr* point, spb_fr* out) {
  if (!ctx || !point || !out || (n && !d_poly)) return SPB_ERR_ARG;
  Fr acc = fp_zero<FrParams>();
  if (n) {
    SPB_ENTER(ctx);
    SPB_TRY(dev_eval_polynomial(ctx, d, (const Fr*)d_poly, n, fr_load(point), &acc));
  }
  memcpy(out, &acc, 32);
  return 0;
}
int spb_eval_polynomial_many_dev(spb_ctx* ctx, const spb_fr* const* d_polys, size_t n, const spb_fr* points, size_t count, spb_fr* out) {
  if (!ctx || (count && (!d_polys || !points || !out)) || !n) return SPB_ERR_ARG;
  if (!count) return 0;
  if (count > 65535) return set_error(ctx, SPB_ERR_ARG, "spb_eval_polynomial_many_dev: more than 65535 queries");
  SPB_ENTER(ctx);
  uint32_t T = 256;
  while (T < 16384 && (uint64_t)T * 64 < n) T <<= 1;     // many queries fill the machine: longer Horner chains, fewer partials
  const uint32_t blocks = T / 256;
  const Fr* const* dptr = (const Fr* const*)slot(ctx, d, "evm_ptrs", count * sizeof(void*));
  Fr* dxs = (Fr*)slot(ctx, d, "evm_xs", 2 * count * sizeof(Fr));
  Fr* dpart = (Fr*)slot(ctx, d, "evm_partial", count * blocks * sizeof(Fr));
  if (!dptr || !dxs || !dpart) return SPB_ERR_OOM;
  std::vector<Fr> xs(2 * count);
  for (size_t q = 0; q < count; q++) { xs[2 * q] = fr_load(&points[q]); xs[2 * q + 1] = fp_pow_u64(xs[2 * q], T); }
  SPB_CUDA(ctx, cudaMemcpyAsync((void*)dptr, d_polys, count * sizeof(void*), cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(dxs, xs.data(), xs.size() * sizeof(Fr), cudaMemcpyHostToDevice, d.stream));
  SPB_TRY(launch(ctx, d.stream, dim3(blocks, (unsigned)count), 256, 0, eval_many_kernel, dptr, dxs, n, T, dpart));
  std::vector<Fr> part(count * blocks);
  SPB_CUDA(ctx, cudaMemcpyAsync(part.data(), dpart, part.size() * sizeof(Fr), cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  for (size_t q = 0; q < count; q++) {
    Fr acc = fp_zero<FrParams>();
    for (uint32_t t = 0; t < blocks; t++) acc = fp_add(acc, part[q * blocks + t]);
    memcpy(&out[q], &acc, 32);
  }
  return 0;
}
int spb_eval_polynomial(spb_ctx* ctx, const spb_fr* poly, size_t n, const spb_fr* point, spb_fr* out) {
  if (!ctx || !point || !out || (n && !poly)) return SPB_ERR_ARG;
  Fr acc = fp_zero<FrParams>();
  if (n) {
    SPB_ENTER(ctx);
    SPB_TRY(run_staged(ctx, d, {{"poly_a", n * 32, poly, nullptr}},
                       [&](void* const* p) { return dev_eval_polynomial(ctx, d, (const Fr*)p[0], n, fr_load(point), &acc); }));
  }
  memcpy(out, &acc, 32);
  return 0;
}

int spb_fr_random_chacha_dev(spb_ctx* ctx, const uint8_t seed[32], uint64_t first, spb_fr* d_out, size_t n) {
  if (!ctx || !seed || (n && !d_out)) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  ChaChaKey key; memcpy(key.w, seed, 32);
  SPB_TRY(launch(ctx, d.stream, nblk(n, 256), 256, 0, fr_random_chacha_kernel, key, first, n, (Fr*)d_out));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

}  // extern "C"
