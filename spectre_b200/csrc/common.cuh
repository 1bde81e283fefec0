// Internal plumbing shared by the translation units of libspectre_b200.so (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include "curve.cuh"
#include "../../include/spectre_b200.h"

namespace spb {


// Grow-only device buffer (workspace slots live for the lifetime of the context: no malloc in the hot path).
struct DevBuf {
  void* ptr = nullptr;
  size_t cap = 0;
};

struct NttTables {
  Fr omega;
  uint32_t k, h;
  Fr* tw_lo = nullptr;  // 2^h
  Fr* tw_hi = nullptr;  // 2^(k-h)
  Fr* tw_full = nullptr;  // 2^k (optional)
};

// One MSM lane of a device: own stream, workspace slots (named "...#lane"), events and pinned result area. Consecutive MSMs of a
// batch cycle over the lanes so the latency-bound tail of one overlaps the sort and accumulation of the next (msm.cu).
struct MsmLane {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // 0-7 stage bounds, 8 start, 9 entry count on the host
  void* pinned = nullptr;
  bool ready = false;
};
// Lanes a batch cycles through: while one MSM accumulates, the latency-bound reduction tail of the previous one and the sort of
// the next one fill the gaps.
static const int kMaxMsmLanes = 3;

struct DeviceState {
  int device = 0;
  int sm_count = 0;
  size_t total_mem = 0;  // bytes of device memory
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t dep_ev = nullptr;  // recorded on `stream` when other streams (MSM lanes, peer devices) must wait for it
  cudaEvent_t stage_ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // MSM stage boundaries
  std::map<std::string, DevBuf> slots;
  MsmLane lanes[kMaxMsmLanes];   // created on first use, released with the context (all access under the context lock)
  std::vector<NttTables> ntt_tables;
  std::vector<NttTables> ntt_pre_tables;  // power tables of coset generators (NttOpts::pre_generator; never a full table)
  void* pinned = nullptr;  // small pinned staging area for results
  size_t pinned_cap = 0;
  void* stage[2] = {nullptr, nullptr};              // two pinned 16 MiB buffers for file <-> device streaming (lazily allocated)
  cudaEvent_t stage_done[2] = {nullptr, nullptr};
};

}  // namespace spb

struct spb_ctx {
  std::vector<spb::DeviceState> dev;
  std::mutex mu;
  std::string last_error;
  bool peer_access = false;  // every device of the context can load from every other one (NVLink P2P enabled)
  // counters (SURVEY.md section 5: per-call instrumentation behind the C ABI)
  uint64_t n_kernel_launches = 0;
  float last_kernel_ms = 0.f;
  uint64_t last_msm_adds = 0;  // G1 additions of the last MSM call / batch
  bool shplonk_slots_busy = false;  // the context's SHPLONK workspace slots are held by an open spb_shplonk handle
  float msm_stage_ms[7] = {0, 0, 0, 0, 0, 0, 0};  // digits, sort, offsets, accumulate, stitch, groups, rowcol + weighted (device 0)
};

// EvaluationDomain (capi.cu builds it; quotient.cu reads its sizes)
struct spb_domain {
  uint32_t j, k, extended_k, quotient_poly_degree;
  spb::Fr omega, omega_inv, extended_omega, extended_omega_inv, g_coset, g_coset_inv, ifft_divisor, extended_ifft_divisor;
  uint32_t t_len;
  spb::Fr* d_t_evaluations;  // device, t_len values
  int device;
};

namespace spb {

int set_error(spb_ctx* ctx, int code, const char* fmt, ...);
// returns nullptr (and sets the error) on failure
void* slot(spb_ctx* ctx, DeviceState& d, const char* name, size_t bytes);

#define SPB_CUDA(ctx, call)                                                                      \
  do {                                                                                           \
    cudaError_t e_ = (call);                                                                     \
    if (e_ != cudaSuccess) return spb::set_error(ctx, SPB_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
  } while (0)
#define SPB_TRY(expr)            \
  do {                           \
    int rc_ = (expr);            \
    if (rc_ != 0) return rc_;    \
  } while (0)

// Prologue of an entry point that works on the first device of the context: takes the context lock, binds `d`.
#define SPB_ENTER(ctx)                          \
  std::lock_guard<std::mutex> lk((ctx)->mu);    \
  DeviceState& d = (ctx)->dev[0];               \
  SPB_CUDA(ctx, cudaSetDevice(d.device));

inline unsigned nblk(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// Every kernel of the library is launched through here. An empty grid launches nothing and returns 0. Otherwise the launch is
// checked, so no launch error is left pending for a later, unrelated call, and counted: the context's launch counter
// (spb_kernel_launches) counts the library's own __global__ launches, not CUB's internal ones, memsets or copies.
template <class... P, class... A>
int launch(spb_ctx* ctx, cudaStream_t stream, dim3 grid, dim3 block, size_t smem, void (*kernel)(P...), const A&... args) {
  if (!grid.x || !grid.y || !grid.z) return 0;
  kernel<<<grid, block, smem, stream>>>(args...);
  ctx->n_kernel_launches++;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return set_error(ctx, SPB_ERR_CUDA, "kernel launch (grid %ux%ux%u, block %u, %zu B shared memory): %s", grid.x, grid.y, grid.z,
                     block.x * block.y * block.z, smem, cudaGetErrorString(e));
  return 0;
}

// Lowest index i < n with bad(i), folded into *first (all ones before the launch). Only a thread that finds a bad element
// touches the atomic, and it stops there: its later indices are larger. The params check (msm.cu) and the proving-key check
// (witness.cu) each pass their own predicate.
template <class Bad>
__global__ void __launch_bounds__(256) first_bad_kernel(Bad bad, uint64_t n, unsigned long long* first) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    if (bad(i)) { atomicMin(first, (unsigned long long)i); return; }
}
// One grid-stride launch of first_bad_kernel over n elements on d.stream, at most 8 blocks per SM; *first must hold all ones.
template <class Bad>
int first_bad_launch(spb_ctx* ctx, DeviceState& d, const Bad& bad, uint64_t n, unsigned long long* first) {
  const unsigned tb = 256;
  const uint64_t blocks = (n + tb - 1) / tb, cap = (uint64_t)(d.sm_count > 0 ? d.sm_count : 1) * 8;
  return launch(ctx, d.stream, (unsigned)(blocks < cap ? blocks : cap), tb, 0, first_bad_kernel<Bad>, bad, n, first);
}

// One device buffer of a host-buffer entry point: slot `slot` of `bytes` bytes. Before the device core runs, its first
// `in_bytes` are copied from `in`; after it, its first `out_bytes` are copied to `out` (a null pointer: no copy).
struct Staging {
  const char* slot;
  size_t bytes;
  const void* in;
  void* out;
  size_t in_bytes = bytes, out_bytes = bytes;
};
// The host-buffer form of a device core: stages every buffer in its slot, uploads, runs core(device pointers, in the order of
// `bufs`) on d.stream, downloads and synchronises.
template <class Core>
int run_staged(spb_ctx* ctx, DeviceState& d, std::initializer_list<Staging> bufs, Core&& core) {
  std::vector<void*> p;
  for (const Staging& b : bufs) {
    p.push_back(slot(ctx, d, b.slot, b.bytes));
    if (!p.back()) return SPB_ERR_OOM;
  }
  size_t i = 0;
  for (const Staging& b : bufs) {
    if (b.in) SPB_CUDA(ctx, cudaMemcpyAsync(p[i], b.in, b.in_bytes, cudaMemcpyHostToDevice, d.stream));
    i++;
  }
  SPB_TRY(core(p.data()));
  i = 0;
  for (const Staging& b : bufs) {
    if (b.out) SPB_CUDA(ctx, cudaMemcpyAsync(b.out, p[i], b.out_bytes, cudaMemcpyDeviceToHost, d.stream));
    i++;
  }
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

// ---- capi.cu: multi-device sharding of one pass ----
// Row ranges of a pass over `rows` rows, one per device, starting at multiples of 256 rows; a single range on the first device
// when the context has one device, no peer access, or the pass is short enough to be launch-bound.
struct RowRange { int dev_index; uint64_t lo, hi; };
std::vector<RowRange> row_ranges(spb_ctx* ctx, uint64_t rows);

// ---- capi.cu: file <-> device streaming through two pinned staging buffers (read of chunk i+1 overlaps the DMA of chunk i) ----
int stream_file_to_device(spb_ctx* ctx, DeviceState& d, FILE* f, void* d_dst, size_t bytes, const char* what);
int stream_device_to_file(spb_ctx* ctx, DeviceState& d, FILE* f, const void* d_src, size_t bytes, const char* what);

// ---- msm.cu ----
void msm_release_ctx(spb_ctx* ctx);

// ---- pairing.cu: out = t in for a G2 point of a params trailer (128 bytes, Montgomery limbs; t Montgomery), on the host ----
void g2_trailer_mul(unsigned char out[128], const unsigned char in[128], const Fr& t);

// ---- ntt.cu ----
struct NttOpts {
  uint64_t n_in = 0, n_out = 0;  // 0 = n
  const Fr* pre3 = nullptr;      // host pointers to 3 factors, or nullptr
  const Fr* post3 = nullptr;
  const Fr* pre_generator = nullptr;  // host pointer to g, or nullptr: input i multiplied by g^i (power tables cached per (k, g))
};
// free every table of a device's NTT caches (the caller has synchronised the device)
void ntt_free_tables(DeviceState& d);
// d_src/d_dst device pointers (may alias); omega host value (Montgomery)
int ntt_device(spb_ctx* ctx, DeviceState& d, const Fr* d_src, Fr* d_dst, uint32_t log_n, const Fr& omega, const NttOpts& opts);
// several devices in the context: six-step across devices with one all-to-all (host buffers)
bool ntt_multi_applicable(spb_ctx* ctx, uint32_t log_n);
int ntt_multi_host(spb_ctx* ctx, const Fr* in, Fr* out, uint32_t log_n, const Fr& omega, const NttOpts& opts, float* ev_ms);

// ---- poly.cu: device-resident cores (pointers on device d, work enqueued on d.stream, no synchronisation unless noted) ----
int dev_grand_product(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, Fr* dz, const Fr& init);  // z[i] = init * prod_{j<i} a[j]
int dev_kate_division(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, const Fr& b, Fr* dq);
int dev_batch_invert(spb_ctx* ctx, DeviceState& d, Fr* da, size_t n);
int dev_product_enqueue(spb_ctx* ctx, DeviceState& d, const Fr* da, size_t n, Fr** d_total);  // *d_total: one Fr on device d, valid after the enqueued work
int dev_eval_polynomial(spb_ctx* ctx, DeviceState& d, const Fr* dp, size_t n, const Fr& x, Fr* out_host);  // synchronises

// ---- lookup.cu: the workspace of permute_expression_pair over n rows (context slots "lk_*") and its canonical sort ----
struct LookupWork {
  Fr *canon, *sin, *stb;                        // n each
  uint32_t *idx_a, *idx_b;                      // n each
  unsigned long long *keys_a, *keys_b;          // n each
  uint32_t* flags;                              // 4 n + 8
  int* err;
  uint32_t *rs_hist, *rs_tile;                  // radix-sort histograms
  void* tmp; size_t tmp_bytes;                  // cub scan temp, enough for n + 1 u32
};
int lookup_work(spb_ctx* ctx, DeviceState& d, uint64_t n, LookupWork* w);
// sorted[i] = the canonical values of src's n rows in ascending order (w.canon, w.idx_*, w.keys_* and the histograms are
// overwritten; sorted may be w.sin or w.stb)
int sort_canonical(spb_ctx* ctx, DeviceState& d, const LookupWork& w, const Fr* src, Fr* sorted, uint64_t n);

// ---- host field helpers (64-bit path) ----
inline Fr fr_from_u64(uint64_t v) {
  Fr a = fp_zero<FrParams>(); a.l[0] = (uint32_t)v; a.l[1] = (uint32_t)(v >> 32);
  return fp_to_mont(a);
}
inline Fr fr_load(const spb_fr* p) { Fr a; memcpy(&a, p, 32); return a; }
inline Fr fr_const(const uint32_t (&v)[8]) { Fr a; for (int i = 0; i < 8; i++) a.l[i] = v[i]; return a; }
// primitive 2^k-th root of unity (Montgomery form)
inline Fr fr_root_of_unity(uint32_t k) {
  constexpr uint32_t v[8] = SPB_FR_ROOT_OF_UNITY_MONT;
  Fr w = fr_const(v);
  for (uint32_t i = k; i < SPB_FR_S; i++) w = fp_sqr(w);
  return w;
}
inline Fr fr_zeta() { constexpr uint32_t v[8] = SPB_FR_ZETA_MONT; return fr_const(v); }
inline Fr fr_delta() { constexpr uint32_t v[8] = SPB_FR_DELTA_MONT; return fr_const(v); }

}  // namespace spb
