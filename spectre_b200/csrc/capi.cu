// C ABI of libspectre_b200.so: context, NTT, EvaluationDomain. (MSM entry points are in msm.cu, batch
// polynomial ops in poly.cu.) See include/spectre_b200.h for the contract of every function.
#include "common.cuh"
#include "ntt.cuh"
#include "../../include/spectre_b200.h"
#include <stdarg.h>
#include <stdio.h>
#include <sys/types.h>
#include <stdlib.h>
#include <string.h>

using namespace spb;

static_assert(sizeof(spb_fr) == sizeof(Fr) && sizeof(spb_g1_affine) == sizeof(G1Affine) && sizeof(spb_g1) == sizeof(G1Jac),
              "C ABI structs must match the device structs byte for byte");

namespace spb {

int set_error(spb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  if (ctx) ctx->last_error = buf;
  return code;
}

void* slot(spb_ctx* ctx, DeviceState& d, const char* name, size_t bytes) {
  DevBuf& b = d.slots[name];
  if (b.cap >= bytes && b.ptr) return b.ptr;
  if (b.ptr) { cudaStreamSynchronize(d.stream); cudaFree(b.ptr); b.ptr = nullptr; b.cap = 0; }
  size_t want = bytes + bytes / 8;  // a little headroom so growing sizes do not realloc every call
  cudaError_t e = cudaMalloc(&b.ptr, want);
  if (e != cudaSuccess) {
    cudaGetLastError();  // the failed headroom allocation must not be reported by the next launch check
    want = bytes; e = cudaMalloc(&b.ptr, want);
  }
  if (e != cudaSuccess) { set_error(ctx, SPB_ERR_OOM, "cudaMalloc(%zu) for slot %s: %s", want, name, cudaGetErrorString(e)); b.ptr = nullptr; return nullptr; }
  b.cap = want;
  return b.ptr;
}

// Below these sizes a pass is launch-bound and stays on the first device. The environment may lower them (SPB_SHARD_MIN_ROWS,
// SPB_SHARD_MIN_LOGN) so that a small circuit runs the multi-device paths; read on every call, as a test sets them at run time.
static uint64_t shard_threshold(const char* var, uint64_t dflt, uint64_t least) {
  const char* e = getenv(var);
  const long long v = e ? atoll(e) : 0;
  return v >= (long long)least ? (uint64_t)v : dflt;
}

std::vector<RowRange> row_ranges(spb_ctx* ctx, uint64_t rows) {
  const size_t D = ctx->dev.size();
  if (D < 2 || !ctx->peer_access || rows < shard_threshold("SPB_SHARD_MIN_ROWS", (uint64_t)1 << 16, 256)) return {RowRange{0, 0, rows}};
  std::vector<RowRange> v;
  const uint64_t per = ((rows + D - 1) / D + 255) / 256 * 256;
  for (size_t i = 0; i < D; i++) {
    const uint64_t lo = per * i, hi = lo + per < rows ? lo + per : rows;
    if (lo < hi) v.push_back(RowRange{(int)i, lo, hi});
  }
  return v;
}

// Double-buffered staging: two pinned 16 MiB buffers per device (slot-like, allocated once). While the DMA of one buffer is
// in flight (cudaMemcpyAsync + an event), the host fills / drains the other, so the file system and the PCIe copy overlap
// instead of alternating as a synchronous cudaMemcpy loop does. (cuFile / GDS would remove the bounce buffer altogether; the
// pool's boxes expose no nvidia-fs, where cuFile itself falls back to exactly this scheme.)
static const size_t kStageBytes = (size_t)16 << 20;
static int stage_buffers(spb_ctx* ctx, DeviceState& d, char** a, char** b, cudaEvent_t* ea, cudaEvent_t* eb) {
  if (!d.stage[0]) {
    SPB_CUDA(ctx, cudaMallocHost(&d.stage[0], kStageBytes));
    SPB_CUDA(ctx, cudaMallocHost(&d.stage[1], kStageBytes));
    SPB_CUDA(ctx, cudaEventCreateWithFlags(&d.stage_done[0], cudaEventDisableTiming));
    SPB_CUDA(ctx, cudaEventCreateWithFlags(&d.stage_done[1], cudaEventDisableTiming));
  }
  *a = (char*)d.stage[0]; *b = (char*)d.stage[1]; *ea = d.stage_done[0]; *eb = d.stage_done[1];
  return 0;
}
int stream_file_to_device(spb_ctx* ctx, DeviceState& d, FILE* f, void* d_dst, size_t bytes, const char* what) {
  char* buf[2]; cudaEvent_t ev[2];
  SPB_TRY(stage_buffers(ctx, d, &buf[0], &buf[1], &ev[0], &ev[1]));
  bool busy[2] = {false, false};
  int cur = 0;
  for (size_t off = 0; off < bytes; off += kStageBytes, cur ^= 1) {
    const size_t cnt = bytes - off < kStageBytes ? bytes - off : kStageBytes;
    if (busy[cur]) SPB_CUDA(ctx, cudaEventSynchronize(ev[cur]));          // the DMA that last used this buffer has drained it
    if (fread(buf[cur], 1, cnt, f) != cnt) return set_error(ctx, SPB_ERR_ARG, "%s: file is truncated", what);
    SPB_CUDA(ctx, cudaMemcpyAsync((char*)d_dst + off, buf[cur], cnt, cudaMemcpyHostToDevice, d.stream));
    SPB_CUDA(ctx, cudaEventRecord(ev[cur], d.stream));
    busy[cur] = true;
  }
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}
int stream_device_to_file(spb_ctx* ctx, DeviceState& d, FILE* f, const void* d_src, size_t bytes, const char* what) {
  char* buf[2]; cudaEvent_t ev[2];
  SPB_TRY(stage_buffers(ctx, d, &buf[0], &buf[1], &ev[0], &ev[1]));
  size_t pending_cnt[2] = {0, 0};
  int cur = 0;
  for (size_t off = 0; off < bytes || pending_cnt[0] || pending_cnt[1]; cur ^= 1) {
    if (pending_cnt[cur]) {                                               // drain the buffer whose D2H was issued two steps ago
      SPB_CUDA(ctx, cudaEventSynchronize(ev[cur]));
      if (fwrite(buf[cur], 1, pending_cnt[cur], f) != pending_cnt[cur]) return set_error(ctx, SPB_ERR_ARG, "%s: short write", what);
      pending_cnt[cur] = 0;
    }
    if (off < bytes) {
      const size_t cnt = bytes - off < kStageBytes ? bytes - off : kStageBytes;
      SPB_CUDA(ctx, cudaMemcpyAsync(buf[cur], (const char*)d_src + off, cnt, cudaMemcpyDeviceToHost, d.stream));
      SPB_CUDA(ctx, cudaEventRecord(ev[cur], d.stream));
      pending_cnt[cur] = cnt; off += cnt;
    }
  }
  return 0;
}

}  // namespace spb

// The test kernels below inline the field / curve primitives under their own register allocation; the test suite runs them on
// operand corpora against Python integers and against the same code built for the host (tests/hostemu/hostemu.cpp).
template <class P>
__global__ void field_op_kernel(int op, const Fp<P>* a, const Fp<P>* b, Fp<P>* o, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fp<P> x = a[i], y = b[i];
  Fp<P> r;
  switch (op) {
    case 0: r = fp_mul(x, y); break;
    case 1: r = fp_add(x, y); break;
    case 2: r = fp_sub(x, y); break;
    case 3: r = fp_sqr(x); break;
    case 4: r = fp_neg(x); break;
    case 5: r = fp_dbl(x); break;
    case 6: r = fp_inv(x); break;
    case 7: r = fp_to_mont(x); break;
    case 8: r = fp_from_mont(x); break;
    case 9: r = fp_zero<P>(); r.l[0] = fp_is_canonical(x) ? 1u : 0u; break;
    case 10: r = fp_pow(x, y.l); break;
    default: r = fp_pow_u64(x, ((uint64_t)y.l[1] << 32) | y.l[0]); break;
  }
  o[i] = r;
}
template <class P>
__global__ void field_mul_sub_mul_kernel(const Fp<P>* a, const Fp<P>* b, const Fp<P>* c, const Fp<P>* d, Fp<P>* o, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) o[i] = fp_mul_sub_mul(a[i], b[i], c[i], d[i]);
}
__device__ __forceinline__ G1Affine xyzz_xy(const G1Xyzz& p) { G1Affine r; r.x = p.x; r.y = p.y; return r; }
__global__ void curve_op_kernel(int op, const G1Xyzz* p, const G1Xyzz* q, const uint32_t* k, G1Xyzz* o, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Xyzz r = p[i];
  switch (op) {
    case 0: xyzz_add_mixed(r, xyzz_xy(q[i])); break;
    case 1: xyzz_add(r, q[i]); break;
    case 2: r = xyzz_dbl(r); break;
    case 3: r = xyzz_dbl_affine(xyzz_xy(r)); break;
    case 4: { G1Affine a = xyzz_to_affine(r); r.x = a.x; r.y = a.y; r.zz = fp_zero<FqParams>(); r.zzz = fp_zero<FqParams>(); break; }
    case 5: r = xyzz_mul_u32(r, k[i]); break;
    default: { const int v = affine_check(xyzz_xy(r)); r = G1Xyzz{}; r.x.l[0] = (uint32_t)v; break; }
  }
  o[i] = r;
}

// ILP independent multiply chains per thread; result folded and written so nothing is optimised away
template <class P, int ILP, bool SQR = false>
__global__ void modmul_bench_kernel(Fp<P>* out, uint32_t iters) {
  Fp<P> x[ILP], y;
  uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
  for (int j = 0; j < ILP; j++) { x[j] = fp_one<P>(); x[j].l[0] ^= tid * 2654435761u + j; x[j].l[7] &= 0x0fffffffu; }
  y = x[0]; y.l[1] ^= 0x9e3779b9u;
  for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
    for (int j = 0; j < ILP; j++) x[j] = SQR ? fp_sqr(x[j]) : fp_mul(x[j], y);
  }
  Fp<P> acc = x[0];
#pragma unroll
  for (int j = 1; j < ILP; j++) acc = fp_add(acc, x[j]);
  out[tid] = acc;
}

extern "C" {

int spb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

spb_ctx* spb_init(const int* device_ids, int n_dev) {
  int avail = spb_device_count();
  if (n_dev <= 0) n_dev = 1;
  if (avail <= 0) { fprintf(stderr, "spectre_b200: no CUDA device visible; this library has no CPU fallback\n"); return nullptr; }
  spb_ctx* ctx = new spb_ctx();
  for (int i = 0; i < n_dev; i++) {
    int id = device_ids ? device_ids[i] : i;
    if (id < 0 || id >= avail) { fprintf(stderr, "spectre_b200: device id %d out of range (have %d)\n", id, avail); delete ctx; return nullptr; }
    DeviceState d; d.device = id;
    if (cudaSetDevice(id) != cudaSuccess) { delete ctx; return nullptr; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, id) != cudaSuccess) { delete ctx; return nullptr; }
    d.sm_count = prop.multiProcessorCount;
    d.total_mem = prop.totalGlobalMem;
    if (cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return nullptr; }
    cudaEventCreate(&d.ev0); cudaEventCreate(&d.ev1);
    cudaEventCreateWithFlags(&d.dep_ev, cudaEventDisableTiming);
    for (int e = 0; e < 8; e++) cudaEventCreate(&d.stage_ev[e]);
    d.pinned_cap = 1 << 20;
    if (cudaMallocHost(&d.pinned, d.pinned_cap) != cudaSuccess) { delete ctx; return nullptr; }
    ctx->dev.push_back(d);
  }
  // several devices: direct NVLink peer copies for the NTT all-to-all and the sharded-MSM scalar scatter. Two entries that
  // name the same device (one device, several shards) need no peer access: a device always reaches its own memory.
  ctx->peer_access = ctx->dev.size() > 1;
  for (size_t i = 0; i < ctx->dev.size(); i++)
    for (size_t j = 0; j < ctx->dev.size(); j++) {
      if (ctx->dev[i].device == ctx->dev[j].device) continue;
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, ctx->dev[i].device, ctx->dev[j].device) != cudaSuccess) can = 0;
      if (!can) { ctx->peer_access = false; cudaGetLastError(); continue; }
      cudaSetDevice(ctx->dev[i].device);
      cudaError_t e = cudaDeviceEnablePeerAccess(ctx->dev[j].device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ctx->peer_access = false;
      cudaGetLastError();  // a peer-access failure is tolerated and must not be reported by the next launch check
    }
  if (!ctx->dev.empty()) cudaSetDevice(ctx->dev[0].device);
  return ctx;
}

void spb_shutdown(spb_ctx* ctx) {
  if (!ctx) return;
  msm_release_ctx(ctx);
  for (auto& d : ctx->dev) {
    cudaSetDevice(d.device);
    cudaStreamSynchronize(d.stream);
    for (auto& kv : d.slots) if (kv.second.ptr) cudaFree(kv.second.ptr);
    ntt_free_tables(d);
    if (d.pinned) cudaFreeHost(d.pinned);
    for (int i = 0; i < 2; i++) { if (d.stage[i]) cudaFreeHost(d.stage[i]); if (d.stage_done[i]) cudaEventDestroy(d.stage_done[i]); }
    cudaEventDestroy(d.ev0); cudaEventDestroy(d.ev1); cudaEventDestroy(d.dep_ev);
    for (int e = 0; e < 8; e++) cudaEventDestroy(d.stage_ev[e]);
    cudaStreamDestroy(d.stream);
  }
  delete ctx;
}

int spb_release_workspace(spb_ctx* ctx) {
  if (!ctx) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->shplonk_slots_busy) return set_error(ctx, SPB_ERR_STATE, "spb_release_workspace: an spb_shplonk handle is open");
  for (auto& d : ctx->dev) {
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaDeviceSynchronize());
    for (auto& kv : d.slots) if (kv.second.ptr) cudaFree(kv.second.ptr);
    d.slots.clear();
    ntt_free_tables(d);
  }
  if (!ctx->dev.empty()) cudaSetDevice(ctx->dev[0].device);
  return 0;
}

const char* spb_last_error(spb_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }
uint64_t spb_kernel_launches(spb_ctx* ctx) { return ctx ? ctx->n_kernel_launches : 0; }
float spb_last_device_ms(spb_ctx* ctx) { return ctx ? ctx->last_kernel_ms : 0.f; }

void* spb_stream(spb_ctx* ctx, int dev_index) {
  if (!ctx || dev_index < 0 || (size_t)dev_index >= ctx->dev.size()) return nullptr;
  return (void*)ctx->dev[dev_index].stream;
}

// ---- file <-> device (params / proving-key files: SURVEY.md 8f rank 4) -----------------------------------------------------
int spb_read_file_dev(spb_ctx* ctx, const char* path, uint64_t offset, void* d_dst, size_t bytes) {
  if (!ctx || !path || (bytes && !d_dst)) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  FILE* f = fopen(path, "rb");
  if (!f) return set_error(ctx, SPB_ERR_ARG, "spb_read_file_dev: cannot open %s", path);
  int rc = fseeko(f, (off_t)offset, SEEK_SET) == 0 ? stream_file_to_device(ctx, d, f, d_dst, bytes, "spb_read_file_dev") : set_error(ctx, SPB_ERR_ARG, "spb_read_file_dev: seek failed");
  fclose(f);
  return rc;
}
int spb_write_file_dev(spb_ctx* ctx, const char* path, int append, const void* d_src, size_t bytes) {
  if (!ctx || !path || (bytes && !d_src)) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  FILE* f = fopen(path, append ? "ab" : "wb");
  if (!f) return set_error(ctx, SPB_ERR_ARG, "spb_write_file_dev: cannot open %s", path);
  int rc = stream_device_to_file(ctx, d, f, d_src, bytes, "spb_write_file_dev");
  if (fclose(f) != 0 && rc == 0) rc = set_error(ctx, SPB_ERR_ARG, "spb_write_file_dev: close failed");
  return rc;
}

int spb_host_register(spb_ctx* ctx, void* ptr, size_t bytes) {
  SPB_CUDA(ctx, cudaHostRegister(ptr, bytes, cudaHostRegisterPortable));
  return 0;
}
int spb_host_unregister(spb_ctx* ctx, void* ptr) {
  SPB_CUDA(ctx, cudaHostUnregister(ptr));
  return 0;
}

// host-only fold of partial MSM results (multi-rank all-gather + local add; EC addition is not an NCCL op)
int spb_g1_sum(const spb_g1* pts, size_t n, spb_g1* out) {
  if (!out || (n && !pts)) return SPB_ERR_ARG;
  G1Xyzz acc = xyzz_identity();
  for (size_t i = 0; i < n; i++) { G1Jac j; memcpy(&j, &pts[i], sizeof j); xyzz_add(acc, xyzz_from_jac(j)); }
  G1Jac r = jac_from_affine(xyzz_to_affine(acc));
  memcpy(out, &r, sizeof r);
  return 0;
}

// out[i] = sum_g pts[g * count + i]: the fold of a whole batch of sharded MSMs after ONE all-gather (groups = ranks)
int spb_g1_sum_batch(const spb_g1* pts, size_t groups, size_t count, spb_g1* out) {
  if (!out || (groups && count && !pts)) return SPB_ERR_ARG;
  for (size_t i = 0; i < count; i++) {
    G1Xyzz acc = xyzz_identity();
    for (size_t g = 0; g < groups; g++) { G1Jac j; memcpy(&j, &pts[g * count + i], sizeof j); xyzz_add(acc, xyzz_from_jac(j)); }
    G1Jac r = jac_from_affine(xyzz_to_affine(acc));
    memcpy(&out[i], &r, sizeof r);
  }
  return 0;
}

// ---- NTT ---------------------------------------------------------------------------------------------------
static int ntt_timed(spb_ctx* ctx, DeviceState& d, const Fr* src, Fr* dst, uint32_t k, const Fr& omega, const NttOpts& o) {
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
  SPB_TRY(ntt_device(ctx, d, src, dst, k, omega, o));
  SPB_CUDA(ctx, cudaEventRecord(d.ev1, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  SPB_CUDA(ctx, cudaEventElapsedTime(&ctx->last_kernel_ms, d.ev0, d.ev1));
  return 0;
}

int spb_ntt_dev(spb_ctx* ctx, spb_fr* d_a, uint32_t log_n, const spb_fr* omega) {
  if (!ctx || !d_a || !omega) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  return ntt_timed(ctx, d, (const Fr*)d_a, (Fr*)d_a, log_n, fr_load(omega), NttOpts());
}

// host-buffer transform through a device staging slot
static int ntt_host(spb_ctx* ctx, const Fr* in, size_t n_in_copy, Fr* out, size_t n_out_copy, uint32_t k, const Fr& omega, const NttOpts& o) {
  if (ntt_multi_applicable(ctx, k)) {
    NttOpts o2 = o;
    if (!o2.n_in) o2.n_in = n_in_copy;
    if (!o2.n_out) o2.n_out = n_out_copy;
    return ntt_multi_host(ctx, in, out, k, omega, o2, nullptr);
  }
  DeviceState& d = ctx->dev[0];
  SPB_CUDA(ctx, cudaSetDevice(d.device));
  return run_staged(ctx, d, {{"ntt_io", ((size_t)1 << k) * sizeof(Fr), in, out, n_in_copy * sizeof(Fr), n_out_copy * sizeof(Fr)}},
                    [&](void* const* p) { return ntt_timed(ctx, d, (Fr*)p[0], (Fr*)p[0], k, omega, o); });
}

int spb_ntt(spb_ctx* ctx, spb_fr* a, uint32_t log_n, const spb_fr* omega) {
  if (!ctx || !a || !omega) return SPB_ERR_ARG;
  if (log_n > 28) return set_error(ctx, SPB_ERR_ARG, "spb_ntt: log_n %u > 28", log_n);
  std::lock_guard<std::mutex> lk(ctx->mu);
  size_t n = (size_t)1 << log_n;
  return ntt_host(ctx, (const Fr*)a, n, (Fr*)a, n, log_n, fr_load(omega), NttOpts());
}

// ---- EvaluationDomain --------------------------------------------------------------------------------------
__global__ void vanishing_table_kernel(Fr* t, Fr cur0, Fr step, uint32_t len) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  Fr cur = fp_mul(cur0, fp_pow_u64(step, i));
  t[i] = fp_inv(fp_sub(cur, fp_one<FrParams>()));
}
__global__ void mul_periodic_kernel(Fr* a, const Fr* t, uint64_t n, uint32_t mask) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr v = ntt_ld_stream(a + i);
  ntt_stg(a + i, fp_mul(v, ntt_ldg(t + (i & mask))));
}

int spb_domain_new(spb_ctx* ctx, uint32_t j, uint32_t k, spb_domain** out) {
  if (!ctx || !out || j < 2) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  spb_domain* dm = new spb_domain();
  dm->j = j; dm->k = k; dm->quotient_poly_degree = j - 1;
  uint64_t n = 1ull << k;
  uint32_t ek = k;
  while ((1ull << ek) < n * dm->quotient_poly_degree) ek++;
  if (ek > 28) { delete dm; return set_error(ctx, SPB_ERR_ARG, "domain: extended_k %u > 28", ek); }
  dm->extended_k = ek;
  dm->extended_omega = fr_root_of_unity(ek); dm->extended_omega_inv = fp_inv(dm->extended_omega);
  dm->omega = fr_root_of_unity(k); dm->omega_inv = fp_inv(dm->omega);
  dm->g_coset = fr_zeta();
  dm->g_coset_inv = fp_sqr(dm->g_coset);
  dm->ifft_divisor = fp_inv(fr_from_u64(n));
  dm->extended_ifft_divisor = fp_inv(fr_from_u64(1ull << ek));
  dm->t_len = 1u << (ek - k);
  DeviceState& d = ctx->dev[0];
  dm->device = d.device;
  SPB_CUDA(ctx, cudaSetDevice(d.device));
  SPB_CUDA(ctx, cudaMalloc(&dm->d_t_evaluations, dm->t_len * sizeof(Fr)));
  Fr cur0 = fp_pow_u64(dm->g_coset, n), step = fp_pow_u64(dm->extended_omega, n);
  SPB_TRY(launch(ctx, d.stream, nblk(dm->t_len, 64), 64, 0, vanishing_table_kernel, dm->d_t_evaluations, cur0, step, dm->t_len));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  *out = dm;
  return 0;
}

void spb_domain_free(spb_ctx* ctx, spb_domain* dm) {
  if (!dm) return;
  if (ctx) { std::lock_guard<std::mutex> lk(ctx->mu); cudaSetDevice(dm->device); cudaFree(dm->d_t_evaluations); }
  delete dm;
}
uint32_t spb_domain_extended_k(const spb_domain* d) { return d ? d->extended_k : 0; }
void spb_domain_constants(const spb_domain* d, spb_fr out[8]) {
  if (!d || !out) return;
  const Fr* src[8] = {&d->omega, &d->omega_inv, &d->extended_omega, &d->extended_omega_inv, &d->g_coset, &d->g_coset_inv, &d->ifft_divisor, &d->extended_ifft_divisor};
  for (int i = 0; i < 8; i++) memcpy(&out[i], src[i], 32);
}

static void l2c_opts(const spb_domain* dm, Fr post[3], NttOpts& o) { for (int i = 0; i < 3; i++) post[i] = dm->ifft_divisor; o.post3 = post; }
static void c2e_opts(const spb_domain* dm, Fr pre[3], NttOpts& o) {
  pre[0] = fp_one<FrParams>(); pre[1] = dm->g_coset; pre[2] = dm->g_coset_inv;
  o.pre3 = pre; o.n_in = 1ull << dm->k;
}
static void e2c_opts(const spb_domain* dm, Fr post[3], NttOpts& o) {
  post[0] = dm->extended_ifft_divisor;
  post[1] = fp_mul(dm->extended_ifft_divisor, dm->g_coset_inv);
  post[2] = fp_mul(dm->extended_ifft_divisor, dm->g_coset);
  o.post3 = post; o.n_out = (1ull << dm->k) * dm->quotient_poly_degree;
}

int spb_lagrange_to_coeff(spb_ctx* ctx, const spb_domain* dm, spb_fr* a) {
  if (!ctx || !dm || !a) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  Fr post[3]; NttOpts o; l2c_opts(dm, post, o);
  size_t n = (size_t)1 << dm->k;
  return ntt_host(ctx, (const Fr*)a, n, (Fr*)a, n, dm->k, dm->omega_inv, o);
}
int spb_coeff_to_lagrange(spb_ctx* ctx, const spb_domain* dm, spb_fr* a) {
  if (!ctx || !dm || !a) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  size_t n = (size_t)1 << dm->k;
  return ntt_host(ctx, (const Fr*)a, n, (Fr*)a, n, dm->k, dm->omega, NttOpts());
}
int spb_coeff_to_extended(spb_ctx* ctx, const spb_domain* dm, const spb_fr* in, spb_fr* out) {
  if (!ctx || !dm || !in || !out) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  Fr pre[3]; NttOpts o; c2e_opts(dm, pre, o);
  return ntt_host(ctx, (const Fr*)in, (size_t)1 << dm->k, (Fr*)out, (size_t)1 << dm->extended_k, dm->extended_k, dm->extended_omega, o);
}
int spb_extended_to_coeff(spb_ctx* ctx, const spb_domain* dm, const spb_fr* in, spb_fr* out) {
  if (!ctx || !dm || !in || !out) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  Fr post[3]; NttOpts o; e2c_opts(dm, post, o);
  return ntt_host(ctx, (const Fr*)in, (size_t)1 << dm->extended_k, (Fr*)out, ((size_t)1 << dm->k) * dm->quotient_poly_degree, dm->extended_k, dm->extended_omega_inv, o);
}
static int div_vanishing_device(spb_ctx* ctx, DeviceState& d, const spb_domain* dm, Fr* d_a) {
  uint64_t e = 1ull << dm->extended_k;
  return launch(ctx, d.stream, nblk(e, 256), 256, 0, mul_periodic_kernel, d_a, dm->d_t_evaluations, e, dm->t_len - 1);
}
int spb_divide_by_vanishing(spb_ctx* ctx, const spb_domain* dm, spb_fr* a) {
  if (!ctx || !dm || !a) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"ntt_io", ((size_t)1 << dm->extended_k) * sizeof(Fr), a, a}},
                    [&](void* const* p) { return div_vanishing_device(ctx, d, dm, (Fr*)p[0]); });
}
int spb_lagrange_to_coeff_dev(spb_ctx* ctx, const spb_domain* dm, spb_fr* d_a) {
  if (!ctx || !dm || !d_a) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  Fr post[3]; NttOpts o; l2c_opts(dm, post, o);
  return ntt_timed(ctx, d, (const Fr*)d_a, (Fr*)d_a, dm->k, dm->omega_inv, o);
}
int spb_coeff_to_extended_dev(spb_ctx* ctx, const spb_domain* dm, const spb_fr* d_in, spb_fr* d_out) {
  if (!ctx || !dm || !d_in || !d_out) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  Fr pre[3]; NttOpts o; c2e_opts(dm, pre, o);
  return ntt_timed(ctx, d, (const Fr*)d_in, (Fr*)d_out, dm->extended_k, dm->extended_omega, o);
}
int spb_extended_to_coeff_dev(spb_ctx* ctx, const spb_domain* dm, const spb_fr* d_in, spb_fr* d_out) {
  if (!ctx || !dm || !d_in || !d_out) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  Fr post[3]; NttOpts o; e2c_opts(dm, post, o);
  return ntt_timed(ctx, d, (const Fr*)d_in, (Fr*)d_out, dm->extended_k, dm->extended_omega_inv, o);
}
// `count` transforms with the same options, polynomial i on device i mod D of the context (SURVEY.md 8e: "shard by polynomial
// for the NTTs"): the buffers stay on the first device; the other devices read the first pass's input and write the last
// pass's output through NVLink peer access, intermediate passes run in their own HBM.
static int ntt_batch_devices(spb_ctx* ctx, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count, uint32_t k, const Fr& omega, const NttOpts& o) {
  DeviceState& d0 = ctx->dev[0];
  const size_t D = (ctx->peer_access && ctx->dev.size() > 1 && k >= shard_threshold("SPB_SHARD_MIN_LOGN", 16, 1)) ? ctx->dev.size() : 1;
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  SPB_CUDA(ctx, cudaEventRecord(d0.ev0, d0.stream));
  if (D > 1) SPB_CUDA(ctx, cudaEventRecord(d0.dep_ev, d0.stream));
  for (size_t i = 0; i < count; i++) {
    if (!d_in[i] || !d_out[i]) return SPB_ERR_ARG;
    DeviceState& d = ctx->dev[i % D];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    if (i < D && i > 0) SPB_CUDA(ctx, cudaStreamWaitEvent(d.stream, d0.dep_ev, 0));
    SPB_TRY(ntt_device(ctx, d, (const Fr*)d_in[i], (Fr*)d_out[i], k, omega, o));
  }
  for (size_t i = 1; i < D && i < count; i++) {
    DeviceState& d = ctx->dev[i];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaEventRecord(d.dep_ev, d.stream));
    SPB_CUDA(ctx, cudaStreamWaitEvent(d0.stream, d.dep_ev, 0));
  }
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  SPB_CUDA(ctx, cudaEventRecord(d0.ev1, d0.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d0.stream));
  SPB_CUDA(ctx, cudaEventElapsedTime(&ctx->last_kernel_ms, d0.ev0, d0.ev1));
  return 0;
}
int spb_lagrange_to_coeff_batch_dev(spb_ctx* ctx, const spb_domain* dm, spb_fr* const* d_a, size_t count) {
  if (!ctx || !dm || (count && !d_a)) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  Fr post[3]; NttOpts o; l2c_opts(dm, post, o);
  return ntt_batch_devices(ctx, (const spb_fr* const*)d_a, d_a, count, dm->k, dm->omega_inv, o);
}
int spb_coeff_to_extended_batch_dev(spb_ctx* ctx, const spb_domain* dm, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count) {
  if (!ctx || !dm || (count && (!d_in || !d_out))) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  Fr pre[3]; NttOpts o; c2e_opts(dm, pre, o);
  return ntt_batch_devices(ctx, d_in, d_out, count, dm->extended_k, dm->extended_omega, o);
}
// Coset part `part` of the extended coset: the extended rows part + R m (R = 2^(extended_k - k)) are the values at
// g omega^m with g = zeta extended_omega^part, so they are the n-point transform of the coefficients pre-scaled by g^a.
int spb_coeff_to_extended_part_batch_dev(spb_ctx* ctx, const spb_domain* dm, uint32_t part, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count) {
  if (!ctx || !dm || (count && (!d_in || !d_out))) return SPB_ERR_ARG;
  if (part >= dm->t_len) return set_error(ctx, SPB_ERR_ARG, "spb_coeff_to_extended_part_batch_dev: part %u of %u", part, dm->t_len);
  std::lock_guard<std::mutex> lk(ctx->mu);
  const Fr g = fp_mul(dm->g_coset, fp_pow_u64(dm->extended_omega, part));
  NttOpts o; o.pre_generator = &g;
  return ntt_batch_devices(ctx, d_in, d_out, count, dm->k, dm->omega, o);
}
int spb_divide_by_vanishing_dev(spb_ctx* ctx, const spb_domain* dm, spb_fr* d_a) {
  if (!ctx || !dm || !d_a) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  SPB_TRY(div_vanishing_device(ctx, d, dm, (Fr*)d_a));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

// ---- test utilities ----------------------------------------------------------------------------------------
int spb_test_field_op(spb_ctx* ctx, int field, int op, const spb_fr* a, const spb_fr* b, spb_fr* out, size_t n) {
  if (!ctx || !a || !b || !out) return SPB_ERR_ARG;
  if (op < 0 || op > 11) return set_error(ctx, SPB_ERR_ARG, "spb_test_field_op: op %d", op);
  SPB_ENTER(ctx);
  Fr* buf = (Fr*)slot(ctx, d, "test_io", 3 * n * sizeof(Fr));
  if (!buf) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaMemcpyAsync(buf, a, n * 32, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(buf + n, b, n * 32, cudaMemcpyHostToDevice, d.stream));
  if (field == 0) SPB_TRY(launch(ctx, d.stream, nblk(n, 128), 128, 0, field_op_kernel<FrParams>, op, (const Fr*)buf, (const Fr*)(buf + n), (Fr*)(buf + 2 * n), n));
  else SPB_TRY(launch(ctx, d.stream, nblk(n, 128), 128, 0, field_op_kernel<FqParams>, op, (const Fq*)buf, (const Fq*)(buf + n), (Fq*)(buf + 2 * n), n));
  SPB_CUDA(ctx, cudaMemcpyAsync(out, buf + 2 * n, n * 32, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

int spb_test_field_mul_sub_mul(spb_ctx* ctx, int field, const spb_fr* a, const spb_fr* b, const spb_fr* c, const spb_fr* dd, spb_fr* out, size_t n) {
  if (!ctx || !a || !b || !c || !dd || !out) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  Fr* buf = (Fr*)slot(ctx, d, "test_io", 5 * n * sizeof(Fr));
  if (!buf) return SPB_ERR_OOM;
  const spb_fr* in[4] = {a, b, c, dd};
  for (int j = 0; j < 4; j++) SPB_CUDA(ctx, cudaMemcpyAsync(buf + j * n, in[j], n * 32, cudaMemcpyHostToDevice, d.stream));
  if (field == 0) SPB_TRY(launch(ctx, d.stream, nblk(n, 128), 128, 0, field_mul_sub_mul_kernel<FrParams>, (const Fr*)buf, (const Fr*)(buf + n), (const Fr*)(buf + 2 * n),
                                 (const Fr*)(buf + 3 * n), (Fr*)(buf + 4 * n), n));
  else SPB_TRY(launch(ctx, d.stream, nblk(n, 128), 128, 0, field_mul_sub_mul_kernel<FqParams>, (const Fq*)buf, (const Fq*)(buf + n), (const Fq*)(buf + 2 * n),
                      (const Fq*)(buf + 3 * n), (Fq*)(buf + 4 * n), n));
  SPB_CUDA(ctx, cudaMemcpyAsync(out, buf + 4 * n, n * 32, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

int spb_test_curve_op(spb_ctx* ctx, int op, const spb_fr* p, const spb_fr* q, const uint32_t* k, spb_fr* out, size_t n) {
  if (!ctx || !p || !q || !out || (op == 5 && !k)) return SPB_ERR_ARG;
  if (op < 0 || op > 6) return set_error(ctx, SPB_ERR_ARG, "spb_test_curve_op: op %d", op);
  SPB_ENTER(ctx);
  const size_t pb = n * sizeof(G1Xyzz);
  char* buf = (char*)slot(ctx, d, "test_io", 3 * pb + n * sizeof(uint32_t));
  if (!buf) return SPB_ERR_OOM;
  G1Xyzz* dp = (G1Xyzz*)buf; G1Xyzz* dq = dp + n; G1Xyzz* dout = dq + n; uint32_t* dk = (uint32_t*)(dout + n);
  SPB_CUDA(ctx, cudaMemcpyAsync(dp, p, pb, cudaMemcpyHostToDevice, d.stream));
  SPB_CUDA(ctx, cudaMemcpyAsync(dq, q, pb, cudaMemcpyHostToDevice, d.stream));
  if (k) SPB_CUDA(ctx, cudaMemcpyAsync(dk, k, n * sizeof(uint32_t), cudaMemcpyHostToDevice, d.stream));
  SPB_TRY(launch(ctx, d.stream, nblk(n, 128), 128, 0, curve_op_kernel, op, (const G1Xyzz*)dp, (const G1Xyzz*)dq, (const uint32_t*)(k ? dk : nullptr), dout, n));
  SPB_CUDA(ctx, cudaMemcpyAsync(out, dout, pb, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return 0;
}

int spb_bench_modmul(spb_ctx* ctx, int field, uint32_t threads, uint32_t iters, int ilp, float* ms) {
  if (!ctx || !ms) return SPB_ERR_ARG;
  SPB_ENTER(ctx);
  threads = (threads + 255) / 256 * 256;
  Fr* buf = (Fr*)slot(ctx, d, "test_io", (size_t)threads * sizeof(Fr));
  if (!buf) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
  // ilp & 0x100: squaring chains (two independent ones per thread)
  void (*fr)(Fr*, uint32_t) = (ilp & 0x100) ? modmul_bench_kernel<FrParams, 2, true> : ilp == 1 ? modmul_bench_kernel<FrParams, 1>
                              : ilp == 2 ? modmul_bench_kernel<FrParams, 2> : modmul_bench_kernel<FrParams, 4>;
  void (*fq)(Fq*, uint32_t) = (ilp & 0x100) ? modmul_bench_kernel<FqParams, 2, true> : ilp == 1 ? modmul_bench_kernel<FqParams, 1>
                              : ilp == 2 ? modmul_bench_kernel<FqParams, 2> : modmul_bench_kernel<FqParams, 4>;
  SPB_TRY(field == 0 ? launch(ctx, d.stream, threads / 256, 256, 0, fr, (Fr*)buf, iters) : launch(ctx, d.stream, threads / 256, 256, 0, fq, (Fq*)buf, iters));
  SPB_CUDA(ctx, cudaEventRecord(d.ev1, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  SPB_CUDA(ctx, cudaEventElapsedTime(ms, d.ev0, d.ev1));
  return 0;
}

}  // extern "C"
