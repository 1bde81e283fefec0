// Host side of the MSM and of the device-resident ParamsKZG (SRS) handle. Kernels: msm.cuh.
#define SPB_MSM_KERNELS 1
#include "common.cuh"
#include "msm.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <string.h>

using namespace spb;

struct SrsShard {
  int dev_index = 0;
  size_t start = 0, count = 0;
  // row 0 = the basis itself; with tables, rows 1..W-1 hold 2^(c*j) * P (row stride = count)
  G1Affine* g = nullptr;
  G1Affine* g_lagrange = nullptr;
};
struct spb_srs {
  uint32_t k = 0;
  size_t n = 0;
  unsigned char g2[128] = {0}, s_g2[128] = {0};  // carried through read/write only (the prover never touches G2)
  uint32_t table_c = 0;  // 0: no precomputed tables
  std::vector<SrsShard> shards;  // one per device of the context, contiguous point ranges
};


namespace spb {

// The lanes of a device (common.cuh: MsmLane) live in its DeviceState, i.e. in the context: nothing here is process-wide.
typedef MsmLane Lane;
static const size_t kLanePinnedBytes = 256 * 1024;  // window partials of one MSM (<= 128 windows x a few points)
// call with the context lock held (every entry point that runs an MSM holds it)
static int get_lane(spb_ctx* ctx, int dev_index, int lane_index, Lane** out) {
  Lane& l = ctx->dev[dev_index].lanes[lane_index];
  if (!l.ready) {
    SPB_CUDA(ctx, cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking));
    for (int i = 0; i < 10; i++) SPB_CUDA(ctx, cudaEventCreate(&l.ev[i]));
    SPB_CUDA(ctx, cudaMallocHost(&l.pinned, kLanePinnedBytes));
    l.ready = true;
  }
  *out = &l;
  return 0;
}

void msm_release_ctx(spb_ctx* ctx) {
  for (auto& d : ctx->dev) {
    cudaSetDevice(d.device);
    for (auto& l : d.lanes) {
      if (!l.ready) continue;
      cudaStreamSynchronize(l.stream);
      for (int i = 0; i < 10; i++) cudaEventDestroy(l.ev[i]);
      cudaFreeHost(l.pinned);
      cudaStreamDestroy(l.stream);
      l = Lane();
    }
  }
}

static void* lane_slot(spb_ctx* ctx, DeviceState& d, int lane, const char* name, size_t bytes) {
  char buf[64];
  snprintf(buf, sizeof buf, "%s#%d", name, lane);
  return slot(ctx, d, buf, bytes);
}

// chunk length such that the accumulation grid is close to a whole number of waves (sm_count SMs x 512 resident threads)
static uint32_t choose_chunk(const DeviceState& d, uint64_t est_entries) {
  const double wave = (double)d.sm_count * 512.0;
  // long entry lists: the chunk pieces (two 128-byte points per chunk, 8 B per entry at L = 32) no longer fit the L2 and the
  // stitch pass becomes DRAM-latency bound; with hundreds of waves the tail of the last wave does not matter
  if (est_entries >= kLongChunkMinEntries) return kLongChunk;
  double waves = (double)est_entries / 32.0 / wave;
  if (waves < 1.0) return 32;
  double w = waves < 1.5 ? 1.0 : (double)(uint64_t)(waves + 0.5);
  uint32_t L = (uint32_t)((double)est_entries / (w * wave)) + 1;
  if (L < 24) L = 24;
  if (L > 48) L = 48;
  return L;
}

// Workspace of one MSM on a lane: the slots are named per lane, so both halves of msm_enqueue_* find the same buffers.
struct MsmWork {
  uint32_t* total;          // entry count M, counted by the digit kernel
  MsmEntry* ent[2];         // unsorted entries | the radix sort's other buffer
  void* sort_tmp; size_t sort_bytes;
};
static int msm_work(spb_ctx* ctx, DeviceState& d, int lane, Lane& ln, uint64_t n, MsmGeom g, MsmWork& w) {
  const uint64_t cap = n * g.W;                 // upper bound on entries
  if (cap >= 0x7fffffffull) return set_error(ctx, SPB_ERR_ARG, "msm: %llu entries exceed the 31-bit sort index", (unsigned long long)cap);
  w.total = (uint32_t*)lane_slot(ctx, d, lane, "msm_total", 16);
  w.ent[0] = (MsmEntry*)lane_slot(ctx, d, lane, "msm_entries", (cap + 1) * sizeof(MsmEntry));
  w.ent[1] = (MsmEntry*)lane_slot(ctx, d, lane, "msm_entries_alt", (cap + 1) * sizeof(MsmEntry));
  // temporary storage for the longest list this MSM can have; a shorter sort uses a prefix of it
  cub::DoubleBuffer<uint64_t> keys((uint64_t*)w.ent[0], (uint64_t*)w.ent[1]);
  w.sort_bytes = 0;
  SPB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(nullptr, w.sort_bytes, keys, (int)cap, 0, msm_key_bits(g), ln.stream));
  w.sort_tmp = lane_slot(ctx, d, lane, "msm_sort_tmp", w.sort_bytes ? w.sort_bytes : 16);
  if (!w.total || !w.ent[0] || !w.ent[1] || !w.sort_tmp) return SPB_ERR_OOM;
  return 0;
}

// First half of one MSM on lane `ln` of device `d`: the digit kernel writes the unsorted entries and counts them; the count
// is copied to the lane's pinned area (after the window partials) and ln.ev[9] marks its arrival.
static int msm_enqueue_digits(spb_ctx* ctx, DeviceState& d, int lane, Lane& ln, const Fr* d_scalars, uint64_t n, MsmGeom g) {
  MsmWork w; SPB_TRY(msm_work(ctx, d, lane, ln, n, g, w));
  const uint32_t per = msm_tail_partials(msm_tail_shape(g.c));
  if ((size_t)g.BW * per * sizeof(G1Xyzz) + 16 > kLanePinnedBytes) return set_error(ctx, SPB_ERR_STATE, "msm: %u window partials exceed the pinned staging area", g.BW * per);
  cudaStream_t st = ln.stream;
  SPB_CUDA(ctx, cudaMemsetAsync(w.total, 0, 4, st));
  cudaEventRecord(ln.ev[0], st);
  SPB_TRY(launch(ctx, st, nblk(n, kDigitsThreads), kDigitsThreads, 0, msm_digits_kernel, n, d_scalars, g, w.total, w.ent[0]));
  cudaEventRecord(ln.ev[1], st);
  SPB_CUDA(ctx, cudaMemcpyAsync((char*)ln.pinned + (size_t)g.BW * per * sizeof(G1Xyzz), w.total, 4, cudaMemcpyDeviceToHost, st));
  SPB_CUDA(ctx, cudaEventRecord(ln.ev[9], st));
  return 0;
}

// Second half: waits for the entry count M on the host (the device keeps running whatever the other lanes have queued), then
// enqueues the sort of exactly M entries and the rest of the MSM. The BW window sums land in the lane's pinned area.
static int msm_enqueue_rest(spb_ctx* ctx, DeviceState& d, int lane, Lane& ln, const G1Affine* d_bases, uint64_t n, MsmGeom g) {
  MsmWork w; SPB_TRY(msm_work(ctx, d, lane, ln, n, g, w));
  const uint64_t nb = (uint64_t)g.BW * g.B;
  const uint64_t cap = n * g.W;
  const uint32_t Lmin = g.L == kLongChunk ? kShortChunk : g.L;   // the kernels may fall back to the short chunk (msm_effective_chunk)
  const uint64_t Tmax = (cap + Lmin - 1) / Lmin;  // upper bound on chunks
  uint32_t* offsets = (uint32_t*)lane_slot(ctx, d, lane, "msm_offsets", (nb + 1) * 4);
  G1Xyzz* buckets = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_buckets", nb * sizeof(G1Xyzz));
  uint32_t* head_key = (uint32_t*)lane_slot(ctx, d, lane, "msm_head_key", (Tmax + 1) * 4);
  uint32_t* tail_key = (uint32_t*)lane_slot(ctx, d, lane, "msm_tail_key", (Tmax + 1) * 4);
  G1Xyzz* head = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_head", (Tmax + 1) * sizeof(G1Xyzz));
  G1Xyzz* tail = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_tail", (Tmax + 1) * sizeof(G1Xyzz));
  uint32_t* giant = (uint32_t*)lane_slot(ctx, d, lane, "msm_giant", (Tmax + 2) * 4);  // [0] = count, [1..] = queue
  const uint64_t max_huge = Tmax / kHugeChain + 1;
  uint32_t* huge = (uint32_t*)lane_slot(ctx, d, lane, "msm_huge", (2 * max_huge + 2) * 4);  // [0] = count, [2..] = (t0, end) pairs
  G1Xyzz* huge_part = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_huge_part", max_huge * kHugeBlocks * sizeof(G1Xyzz));
  const MsmTail tl = msm_tail_shape(g.c);
  const uint32_t R = 1u << tl.r_log, C = 1u << tl.c_log, per = msm_tail_partials(tl);
  const uint32_t T1 = g.B >> tl.m_log;                       // group sums per bucket set
  const uint64_t ngroups = (uint64_t)g.BW * T1;
  G1Xyzz* grp = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_groups", 2 * ngroups * sizeof(G1Xyzz));   // S1 | W1
  G1Xyzz* seg_out = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_rowcol", (uint64_t)g.BW * (2 * R + C) * sizeof(G1Xyzz));   // rows | columns | W rows
  G1Xyzz* win_out = (G1Xyzz*)lane_slot(ctx, d, lane, "msm_partials", (uint64_t)g.BW * per * sizeof(G1Xyzz));
  if (!offsets || !buckets || !head_key || !tail_key || !head || !tail || !giant || !huge || !huge_part || !grp || !seg_out || !win_out)
    return SPB_ERR_OOM;

  SPB_CUDA(ctx, cudaEventSynchronize(ln.ev[9]));
  uint32_t M; memcpy(&M, (const char*)ln.pinned + (size_t)g.BW * per * sizeof(G1Xyzz), 4);
  cudaStream_t st = ln.stream;
  // the bucket array is NOT cleared: every non-empty bucket is written exactly once (accumulate / stitch / giant paths) and
  // the reduction reads a bucket only where the offsets say it has entries
  SPB_CUDA(ctx, cudaMemsetAsync(giant, 0, 4, st));
  SPB_CUDA(ctx, cudaMemsetAsync(huge, 0, 4, st));
  // Sorting M entries rather than the n * W upper bound keeps a sparse (witness) column as cheap as its entries. A pass
  // moves whole 8-byte entries but looks only at key bits: the value in the upper half rides along.
  cub::DoubleBuffer<uint64_t> keys((uint64_t*)w.ent[0], (uint64_t*)w.ent[1]);
  SPB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(w.sort_tmp, w.sort_bytes, keys, (int)M, 0, msm_key_bits(g), st));
  const MsmEntry* ent = (const MsmEntry*)keys.Current();
  const uint32_t* total = w.total;
  cudaEventRecord(ln.ev[2], st);
  SPB_TRY(launch(ctx, st, nblk(nb + 1, 256), 256, 0, msm_offsets_kernel, total, nb, ent, offsets));
  cudaEventRecord(ln.ev[3], st);
  SPB_TRY(launch(ctx, st, nblk(Tmax, 128), 128, 0, msm_accumulate_kernel, total, g, ent, d_bases, buckets, head_key, head, tail_key, tail));
  cudaEventRecord(ln.ev[4], st);
  SPB_TRY(launch(ctx, st, nblk(Tmax, 128), 128, 0, msm_stitch_kernel, total, g.L, 24, head_key, head, tail_key, tail, buckets, giant, giant + 1));
  SPB_TRY(launch(ctx, st, 256, 128, 0, msm_giant_kernel, total, g.L, giant, giant + 1, head_key, head, tail_key, tail, buckets, huge, huge + 2));
  SPB_TRY(launch(ctx, st, kHugeBlocks, 128, 0, msm_huge_kernel, huge, huge + 2, head, huge_part));
  SPB_TRY(launch(ctx, st, 64, 128, 0, msm_huge_finish_kernel, huge, huge + 2, kHugeBlocks, huge_part, tail_key, tail, buckets));
  cudaEventRecord(ln.ev[5], st);
  G1Xyzz *rows = seg_out, *cols = seg_out + (uint64_t)g.BW * R, *wrows = seg_out + (uint64_t)g.BW * (R + C);
  SPB_TRY(launch(ctx, st, nblk(ngroups, 128), 128, 0, msm_group_kernel, ngroups, tl.m_log, offsets, buckets, grp, grp + ngroups));
  cudaEventRecord(ln.ev[6], st);
  SPB_TRY(launch(ctx, st, g.BW * (2 * R + C), 64, 0, msm_rowcol_kernel, T1, tl, grp, grp + ngroups, rows, cols, wrows));
  SPB_TRY(launch(ctx, st, g.BW * (2 * tl.nbr + tl.nbc), 128, 0, msm_weighted_kernel, tl, rows, cols, wrows, win_out));
  cudaEventRecord(ln.ev[7], st);
  SPB_CUDA(ctx, cudaMemcpyAsync(ln.pinned, win_out, (size_t)g.BW * per * sizeof(G1Xyzz), cudaMemcpyDeviceToHost, st));
  return 0;
}

static G1Xyzz msm_finish(Lane& ln, MsmGeom g, uint64_t* adds) {
  const MsmTail tl = msm_tail_shape(g.c);
  const uint32_t per = msm_tail_partials(tl);
  const G1Xyzz* P = (const G1Xyzz*)ln.pinned;
  uint32_t M; memcpy(&M, (const char*)ln.pinned + (size_t)g.BW * per * sizeof(G1Xyzz), 4);
  if (adds) *adds += (uint64_t)M + 2ull * g.BW * g.B;
  std::vector<G1Xyzz> S(g.BW);
  for (uint32_t w = 0; w < g.BW; w++) S[w] = msm_tail_finish(g, P + (size_t)w * per);
  return msm_combine_windows(S.data(), g.BW, g.c);
}

static void write_result(const G1Xyzz& r, spb_g1* out) {
  G1Affine a = xyzz_to_affine(r);
  G1Jac j = jac_from_affine(a);
  memcpy(out, &j, sizeof(G1Jac));
}

struct MsmPart {
  int dev_index;
  const Fr* d_scalars;      // device pointer on that device (nullptr: copy from h_scalars on the lane's stream)
  const Fr* h_scalars;      // host pointer for this part, or nullptr
  int peer_src_device;      // >= 0: d_scalars lives on that device and must be peer-copied
  const G1Affine* d_bases;  // device pointer on that device
  uint64_t n;
  MsmGeom g;
};

// One job = one MSM = one part per device, all on lane `lane`. enqueue -> (later) collect. The enqueue returns once every
// part's entry count has reached the host and the rest of the part is queued.
static int job_enqueue(spb_ctx* ctx, int lane, std::vector<MsmPart>& parts) {
  for (auto& p : parts) {
    if (!p.n) continue;
    DeviceState& d = ctx->dev[p.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    Lane* ln; SPB_TRY(get_lane(ctx, p.dev_index, lane, &ln));
    p.g.L = choose_chunk(d, p.n * p.g.W);
    const Fr* ds = p.d_scalars;
    // stream contract (spectre_b200.h): scalars produced on the context stream of the device they live on are ready for the lane
    DeviceState& src = p.peer_src_device >= 0 ? ctx->dev[0] : d;
    if (&src != &d) SPB_CUDA(ctx, cudaSetDevice(src.device));
    SPB_CUDA(ctx, cudaEventRecord(src.dep_ev, src.stream));
    if (&src != &d) SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaStreamWaitEvent(ln->stream, src.dep_ev, 0));
    SPB_CUDA(ctx, cudaEventRecord(ln->ev[8], ln->stream));
    if (p.h_scalars || p.peer_src_device >= 0) {
      Fr* buf = (Fr*)lane_slot(ctx, d, lane, "msm_scalars", p.n * sizeof(Fr));
      if (!buf) return SPB_ERR_OOM;
      if (p.h_scalars) SPB_CUDA(ctx, cudaMemcpyAsync(buf, p.h_scalars, p.n * sizeof(Fr), cudaMemcpyHostToDevice, ln->stream));
      else SPB_CUDA(ctx, cudaMemcpyPeerAsync(buf, d.device, p.d_scalars, p.peer_src_device, p.n * sizeof(Fr), ln->stream));
      ds = buf;
    }
    SPB_TRY(msm_enqueue_digits(ctx, d, lane, *ln, ds, p.n, p.g));
  }
  // every part's digit kernel is queued before the first wait for an entry count
  for (auto& p : parts) {
    if (!p.n) continue;
    DeviceState& d = ctx->dev[p.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    Lane* ln; SPB_TRY(get_lane(ctx, p.dev_index, lane, &ln));
    SPB_TRY(msm_enqueue_rest(ctx, d, lane, *ln, p.d_bases, p.n, p.g));
  }
  return 0;
}

static int job_collect(spb_ctx* ctx, int lane, const std::vector<MsmPart>& parts, spb_g1* out) {
  G1Xyzz acc = xyzz_identity();
  float worst = 0.f;
  for (auto& p : parts) {
    if (!p.n) continue;
    DeviceState& d = ctx->dev[p.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    Lane* ln; SPB_TRY(get_lane(ctx, p.dev_index, lane, &ln));
    SPB_CUDA(ctx, cudaStreamSynchronize(ln->stream));
    float ms = 0.f;
    SPB_CUDA(ctx, cudaEventElapsedTime(&ms, ln->ev[8], ln->ev[7]));
    if (ms > worst) worst = ms;
    if (p.dev_index == 0) for (int e = 0; e < 7; e++) cudaEventElapsedTime(&ctx->msm_stage_ms[e], ln->ev[e], ln->ev[e + 1]);
    G1Xyzz r = msm_finish(*ln, p.g, &ctx->last_msm_adds);
    xyzz_add(acc, r);
  }
  ctx->last_kernel_ms = worst;
  write_result(acc, out);
  return 0;
}

// out[i] = scalars[i] * G1 generator, affine
static int g1_fixed_base_mul(spb_ctx* ctx, DeviceState& d, const Fr* scalars, size_t n, G1Affine* out) {
  return launch(ctx, d.stream, nblk(n, 128), 128, 0, g1_fixed_base_mul_kernel, scalars, n, out);
}

}  // namespace spb

extern "C" {

uint64_t spb_last_msm_adds(spb_ctx* ctx) { return ctx ? ctx->last_msm_adds : 0; }
void spb_last_msm_stage_ms(spb_ctx* ctx, float out[7]) { if (!out) return; for (int i = 0; i < 7; i++) out[i] = ctx ? ctx->msm_stage_ms[i] : 0.f; }
void spb_msm_geometry(size_t n, int tables, uint32_t* c, uint32_t* windows) {
  MsmGeom g = msm_make_geometry(msm_choose_c(n ? n : 1, tables != 0), tables != 0, 0);
  if (c) *c = g.c;
  if (windows) *windows = g.W;
}

// ---- ParamsKZG ---------------------------------------------------------------------------------------------
static spb_srs* srs_alloc(spb_ctx* ctx, uint32_t k) {
  spb_srs* s = new spb_srs();
  s->k = k; s->n = (size_t)1 << k;
  size_t D = ctx->dev.size();
  for (size_t i = 0; i < D; i++) {
    SrsShard sh; sh.dev_index = (int)i;
    sh.start = s->n * i / D; sh.count = s->n * (i + 1) / D - sh.start;
    s->shards.push_back(sh);
  }
  return s;
}

void spb_srs_free(spb_ctx* ctx, spb_srs* srs) {
  if (!srs) return;
  if (ctx) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    for (auto& sh : srs->shards) {
      cudaSetDevice(ctx->dev[sh.dev_index].device);
      if (sh.g) cudaFree(sh.g);
      if (sh.g_lagrange) cudaFree(sh.g_lagrange);
    }
  }
  delete srs;
}

int spb_srs_upload(spb_ctx* ctx, uint32_t k, const spb_g1_affine* g, const spb_g1_affine* g_lagrange, spb_srs** out) {
  if (!ctx || !out || k > 28) return SPB_ERR_ARG;
  spb_srs* s;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    s = srs_alloc(ctx, k);
    for (auto& sh : s->shards) {
      DeviceState& d = ctx->dev[sh.dev_index];
      cudaError_t e = cudaSetDevice(d.device);
      if (e == cudaSuccess && g && sh.count) {
        e = cudaMalloc(&sh.g, sh.count * sizeof(G1Affine));
        if (e == cudaSuccess) e = cudaMemcpyAsync(sh.g, (const G1Affine*)g + sh.start, sh.count * sizeof(G1Affine), cudaMemcpyHostToDevice, d.stream);
      }
      if (e == cudaSuccess && g_lagrange && sh.count) {
        e = cudaMalloc(&sh.g_lagrange, sh.count * sizeof(G1Affine));
        if (e == cudaSuccess) e = cudaMemcpyAsync(sh.g_lagrange, (const G1Affine*)g_lagrange + sh.start, sh.count * sizeof(G1Affine), cudaMemcpyHostToDevice, d.stream);
      }
      if (e == cudaSuccess) e = cudaStreamSynchronize(d.stream);
      if (e != cudaSuccess) { set_error(ctx, SPB_ERR_CUDA, "spb_srs_upload: %s", cudaGetErrorString(e)); goto fail; }
    }
    *out = s;
    return 0;
  }
fail:
  spb_srs_free(ctx, s);
  return SPB_ERR_CUDA;
}

// Arbitrary bases kept resident: what a caller of best_multiexp that reuses one base vector (any length) uploads once instead of
// paying 64 B x n of PCIe per call through spb_msm_raw. The handle is an SRS handle with only `g` set and n = the given length.
int spb_bases_upload(spb_ctx* ctx, const spb_g1_affine* bases, size_t n, spb_srs** out) {
  if (!ctx || !out || !bases || !n || n > ((size_t)1 << 28)) return SPB_ERR_ARG;
  uint32_t k = 0; while (((size_t)1 << k) < n) k++;
  spb_srs* s;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    s = srs_alloc(ctx, k);
    s->n = n;
    const size_t D = ctx->dev.size();
    for (size_t i = 0; i < D; i++) { s->shards[i].start = n * i / D; s->shards[i].count = n * (i + 1) / D - s->shards[i].start; }
    for (auto& sh : s->shards) {
      if (!sh.count) continue;
      DeviceState& d = ctx->dev[sh.dev_index];
      cudaError_t e = cudaSetDevice(d.device);
      if (e == cudaSuccess) e = cudaMalloc(&sh.g, sh.count * sizeof(G1Affine));
      if (e == cudaSuccess) e = cudaMemcpyAsync(sh.g, (const G1Affine*)bases + sh.start, sh.count * sizeof(G1Affine), cudaMemcpyHostToDevice, d.stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(d.stream);
      if (e != cudaSuccess) { set_error(ctx, SPB_ERR_CUDA, "spb_bases_upload: %s", cudaGetErrorString(e)); goto fail; }
    }
    *out = s;
    return 0;
  }
fail:
  spb_srs_free(ctx, s);
  return SPB_ERR_CUDA;
}

int spb_srs_setup(spb_ctx* ctx, uint32_t k, const spb_fr* secret, spb_srs** out) {
  if (!ctx || !out || !secret || k > 28) return SPB_ERR_ARG;
  spb_srs* s;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    s = srs_alloc(ctx, k);
    const Fr tau = fr_load(secret), w = fr_root_of_unity(k);
    const uint64_t n = 1ull << k;
    Fr coef = fp_mul(fp_sub(fp_pow_u64(tau, n), fp_one<FrParams>()), fp_inv(fr_from_u64(n)));
    for (auto& sh : s->shards) {
      if (!sh.count) continue;
      DeviceState& d = ctx->dev[sh.dev_index];
      cudaError_t e = cudaSetDevice(d.device);
      Fr* sc = (Fr*)slot(ctx, d, "srs_scalars", sh.count * sizeof(Fr));
      if (!sc) goto fail;
      if (e == cudaSuccess) e = cudaMalloc(&sh.g, sh.count * sizeof(G1Affine));
      if (e == cudaSuccess) e = cudaMalloc(&sh.g_lagrange, sh.count * sizeof(G1Affine));
      if (e != cudaSuccess) { set_error(ctx, SPB_ERR_CUDA, "spb_srs_setup: %s", cudaGetErrorString(e)); goto fail; }
      const unsigned blocks = nblk(sh.count, 128);
      if (launch(ctx, d.stream, blocks, 128, 0, srs_scalars_kernel, 0, tau, w, coef, sh.start, sh.count, sc) ||
          g1_fixed_base_mul(ctx, d, sc, sh.count, sh.g) ||
          launch(ctx, d.stream, blocks, 128, 0, srs_scalars_kernel, 1, tau, w, coef, sh.start, sh.count, sc) ||
          g1_fixed_base_mul(ctx, d, sc, sh.count, sh.g_lagrange))
        goto fail;
      e = cudaStreamSynchronize(d.stream);
      if (e != cudaSuccess) { set_error(ctx, SPB_ERR_CUDA, "spb_srs_setup: %s", cudaGetErrorString(e)); goto fail; }
    }
    *out = s;
    return 0;
  }
fail:
  spb_srs_free(ctx, s);
  return SPB_ERR_CUDA;
}

// ParamsKZG::downsize(k) ([UPSTREAM] halo2_proofs/src/poly/kzg/commitment.rs; the reference keeps a degree -> params map "for
// params downsize", prover/src/prover.rs:34): g truncated to 2^k points, g_lagrange recomputed for the smaller domain as
// g_to_lagrange(g) = the inverse DFT over the group (log2 n stages of n/2 butterflies, each one point addition, one
// subtraction and one 254-bit scalar multiple by a power of omega^-1; then 1/n and affine normalisation). Works for any SRS
// (no knowledge of the secret). Returns a NEW handle (no window tables); the caller frees the old one when it is done with it.
//
// g_to_lagrange of the first n = 2^k points of src's g (complete before the call), on the context's first device: the points
// gathered into slot "ds_g", the result in slot "ds_lag". Enqueued on that device's stream, not waited for.
static int srs_g_to_lagrange(spb_ctx* ctx, const spb_srs* src, uint32_t k, const char* who, G1Affine** g_out, G1Affine** lag_out) {
  const uint64_t n = 1ull << k;
  DeviceState& d = ctx->dev[0];
  SPB_CUDA(ctx, cudaSetDevice(d.device));
  G1Affine* g0 = (G1Affine*)slot(ctx, d, "ds_g", n * sizeof(G1Affine));          // the first n points of g, gathered on device 0
  G1Xyzz* pts = (G1Xyzz*)slot(ctx, d, "ds_pts", n * sizeof(G1Xyzz));
  G1Affine* lag = (G1Affine*)slot(ctx, d, "ds_lag", n * sizeof(G1Affine));
  Fr* tw = (Fr*)slot(ctx, d, "ds_tw", (n / 2 ? n / 2 : 1) * sizeof(Fr));
  if (!g0 || !pts || !lag || !tw) return SPB_ERR_OOM;
  for (auto& sh : src->shards) {
    if (sh.start >= n || !sh.count) continue;
    if (!sh.g) return set_error(ctx, SPB_ERR_STATE, "%s: basis g not resident", who);
    const size_t cnt = (n - sh.start) < sh.count ? (n - sh.start) : sh.count;
    SPB_CUDA(ctx, cudaMemcpyPeerAsync(g0 + sh.start, d.device, sh.g, ctx->dev[sh.dev_index].device, cnt * sizeof(G1Affine), d.stream));
  }
  const Fr w_inv = fp_inv(fr_root_of_unity(k)), n_inv = fp_inv(fr_from_u64(n));
  const unsigned tb = 128;
  SPB_TRY(launch(ctx, d.stream, nblk(n, tb), tb, 0, ec_lift_kernel, n, g0, pts));
  if (n >= 2) {
    SPB_TRY(launch(ctx, d.stream, nblk(n / 2, 256), 256, 0, fr_powers_kernel, tw, w_inv, n / 2));
    for (uint64_t half = n / 2; half >= 1; half >>= 1) SPB_TRY(launch(ctx, d.stream, nblk(n / 2, tb), tb, 0, ec_ntt_stage_kernel, n, half, tw, pts));
  }
  SPB_TRY(launch(ctx, d.stream, nblk(n, tb), tb, 0, ec_ntt_finish_kernel, n, k, n_inv, pts, lag));
  *g_out = g0; *lag_out = lag;
  return 0;
}

// Give every shard of s its g_lagrange (and its g, when g is not null) from the first device's buffers, and wait for the copies.
static int srs_fill_shards(spb_ctx* ctx, spb_srs* s, const G1Affine* g, const G1Affine* lag, const char* who) {
  DeviceState& d = ctx->dev[0];
  cudaError_t e = cudaSuccess;
  for (auto& sh : s->shards) {
    if (!sh.count) continue;
    DeviceState& dd = ctx->dev[sh.dev_index];
    e = cudaSetDevice(dd.device);
    if (e == cudaSuccess && g) e = cudaMalloc(&sh.g, sh.count * sizeof(G1Affine));
    if (e == cudaSuccess) e = cudaMalloc(&sh.g_lagrange, sh.count * sizeof(G1Affine));
    if (e != cudaSuccess) break;
    cudaSetDevice(d.device);
    if (g) e = cudaMemcpyPeerAsync(sh.g, dd.device, g + sh.start, d.device, sh.count * sizeof(G1Affine), d.stream);
    if (e == cudaSuccess) e = cudaMemcpyPeerAsync(sh.g_lagrange, dd.device, lag + sh.start, d.device, sh.count * sizeof(G1Affine), d.stream);
    if (e != cudaSuccess) break;
  }
  cudaSetDevice(d.device);
  if (e == cudaSuccess) e = cudaStreamSynchronize(d.stream);
  if (e != cudaSuccess) return set_error(ctx, SPB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
  return 0;
}

static int srs_downsize_locked(spb_ctx* ctx, const spb_srs* srs, uint32_t k, spb_srs** made) {
  G1Affine *g0, *lag;
  SPB_TRY(srs_g_to_lagrange(ctx, srs, k, "spb_srs_downsize", &g0, &lag));
  spb_srs* s = srs_alloc(ctx, k);
  *made = s;
  memcpy(s->g2, srs->g2, 128); memcpy(s->s_g2, srs->s_g2, 128);
  return srs_fill_shards(ctx, s, g0, lag, "spb_srs_downsize");
}

// ParamsKZG::setup run by several parties: one powers-of-tau update by the secret t. Each shard scales its own points on its own
// device (srs_scale_kernel, global index start + j), g_lagrange is g_to_lagrange of the new g at the handle's own k (the path
// of downsize), and s_g2 = t s_g2 on the host. last_kernel_ms: first scaling launch to the end of g_to_lagrange, on the first
// device's clock.
static int srs_contribute_locked(spb_ctx* ctx, const spb_srs* srs, const Fr& t, spb_srs** made) {
  spb_srs* s = srs_alloc(ctx, srs->k);
  *made = s;
  DeviceState& d0 = ctx->dev[0];
  SPB_CUDA(ctx, cudaSetDevice(d0.device));
  SPB_CUDA(ctx, cudaEventRecord(d0.ev0, d0.stream));
  for (size_t i = 0; i < s->shards.size(); i++) {
    const SrsShard& from = srs->shards[i];
    SrsShard& to = s->shards[i];
    if (!to.count) continue;
    if (!from.g) return set_error(ctx, SPB_ERR_STATE, "spb_srs_contribute: basis g not resident");
    DeviceState& d = ctx->dev[to.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaMalloc(&to.g, to.count * sizeof(G1Affine)));
    SPB_TRY(launch(ctx, d.stream, nblk(to.count, 128), 128, 0, srs_scale_kernel, (uint64_t)to.start, (uint64_t)to.count, t, (const G1Affine*)from.g, to.g));
  }
  for (auto& sh : s->shards) {
    if (!sh.count) continue;
    SPB_CUDA(ctx, cudaSetDevice(ctx->dev[sh.dev_index].device));
    SPB_CUDA(ctx, cudaStreamSynchronize(ctx->dev[sh.dev_index].stream));
  }
  G1Affine *g0, *lag;
  SPB_TRY(srs_g_to_lagrange(ctx, s, s->k, "spb_srs_contribute", &g0, &lag));
  SPB_CUDA(ctx, cudaEventRecord(d0.ev1, d0.stream));
  SPB_TRY(srs_fill_shards(ctx, s, nullptr, lag, "spb_srs_contribute"));
  SPB_CUDA(ctx, cudaEventElapsedTime(&ctx->last_kernel_ms, d0.ev0, d0.ev1));
  memcpy(s->g2, srs->g2, 128);
  g2_trailer_mul(s->s_g2, srs->s_g2, t);
  return 0;
}
int spb_srs_downsize(spb_ctx* ctx, const spb_srs* srs, uint32_t k, spb_srs** out) {
  if (!ctx || !srs || !out || k > srs->k) return SPB_ERR_ARG;
  if (srs->n != ((size_t)1 << srs->k)) return set_error(ctx, SPB_ERR_STATE, "spb_srs_downsize: the handle holds %zu plain bases (spb_bases_upload), not a 2^k SRS", srs->n);
  if (srs->table_c) return set_error(ctx, SPB_ERR_STATE, "spb_srs_downsize: call before spb_srs_precompute (the table rows replaced the plain basis layout)");
  spb_srs* made = nullptr;
  int rc;
  { std::lock_guard<std::mutex> lk(ctx->mu); rc = srs_downsize_locked(ctx, srs, k, &made); }
  if (rc != 0) { if (made) spb_srs_free(ctx, made); return rc; }
  *out = made;
  return 0;
}

int spb_srs_contribute(spb_ctx* ctx, const spb_srs* srs, const spb_fr* t, spb_srs** out) {
  if (!ctx || !srs || !t || !out) return SPB_ERR_ARG;
  const Fr tm = fr_load(t);
  if (fp_is_zero(tm)) return set_error(ctx, SPB_ERR_ARG, "spb_srs_contribute: t = 0 would erase every point after g[0]");
  if (!fp_is_canonical(tm)) return set_error(ctx, SPB_ERR_ARG, "spb_srs_contribute: t is not less than r");
  if (srs->n != ((size_t)1 << srs->k)) return set_error(ctx, SPB_ERR_STATE, "spb_srs_contribute: the handle holds %zu plain bases (spb_bases_upload), not a 2^k SRS", srs->n);
  if (srs->table_c) return set_error(ctx, SPB_ERR_STATE, "spb_srs_contribute: call before spb_srs_precompute (the table rows replaced the plain basis layout)");
  static const unsigned char zero[128] = {0};
  if (!memcmp(srs->g2, zero, 128) || !memcmp(srs->s_g2, zero, 128))
    return set_error(ctx, SPB_ERR_STATE, "spb_srs_contribute: the handle's G2 trailer is zero (give it with spb_srs_set_g2 first)");
  spb_srs* made = nullptr;
  int rc;
  { std::lock_guard<std::mutex> lk(ctx->mu); rc = srs_contribute_locked(ctx, srs, tm, &made); }
  if (rc != 0) { if (made) spb_srs_free(ctx, made); return rc; }
  *out = made;
  return 0;
}

}  // extern "C"

namespace spb {

// a point that fails affine_check (first_bad_kernel's predicate for the params check)
struct PointBad {
  const G1Affine* pts;
  __device__ bool operator()(uint64_t i) const { return affine_check(pts[i]) != kPointValid; }
};

static const char* point_check_reason(int verdict) {
  switch (verdict) {
    case kPointXNotCanonical: return "x is not less than the field modulus";
    case kPointYNotCanonical: return "y is not less than the field modulus";
    case kPointOffCurve: return "not on the curve";
    default: return "rejected by the device check but valid on the host";
  }
}

// Check `count` resident points of device d (one grid-stride launch on d's stream). *bad = index of the first invalid point, or
// count when every point is valid; *ms accumulates the kernel's device time.
static int srs_check_points(spb_ctx* ctx, DeviceState& d, const G1Affine* pts, size_t count, size_t* bad, float* ms) {
  unsigned long long* first = (unsigned long long*)slot(ctx, d, "srs_check", sizeof(unsigned long long));
  if (!first) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaMemsetAsync(first, 0xff, sizeof(unsigned long long), d.stream));
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
  SPB_TRY(first_bad_launch(ctx, d, PointBad{pts}, count, first));
  SPB_CUDA(ctx, cudaEventRecord(d.ev1, d.stream));
  unsigned long long h = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&h, first, sizeof h, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  float t = 0.f;
  SPB_CUDA(ctx, cudaEventElapsedTime(&t, d.ev0, d.ev1));
  *ms += t;
  *bad = h < count ? (size_t)h : count;
  return 0;
}

// The shard's first invalid point, downloaded and classified again on the host for the error text.
static int srs_point_error(spb_ctx* ctx, DeviceState& d, const char* path, const char* basis, const G1Affine* pts, size_t local, size_t global) {
  G1Affine p;
  SPB_CUDA(ctx, cudaMemcpyAsync(&p, pts + local, sizeof p, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  return set_error(ctx, SPB_ERR_DATA, "spb_srs_read_file: %s: %s[%zu]: %s", path, basis, global, point_check_reason(affine_check(p)));
}

}  // namespace spb

extern "C" {

// ParamsKZG::read_custom / write: k (u32 LE) | g[n] | g_lagrange[n] | g2 | s_g2, every coordinate as its in-memory Montgomery
// limbs -- the file halo2-base's gen_srs caches as params/kzg_bn254_{k}.srs ([UPSTREAM] halo2_proofs/src/poly/kzg/commitment.rs;
// reference .gitignore:36 `params/`). Streamed through two pinned staging buffers straight into device memory, file read and
// DMA overlapped (K = 24: 2 GiB). SPB_SERDE_RAW_BYTES checks every point as halo2curves' read_raw does: the G1 points of each
// shard with one kernel on its own device once the shard is resident, the G2 trailer on the host. Shards are read in file
// order, so the first shard that reports a bad point holds the first one of the file. (The check is not fused into the
// staging loop: on an H100 80GB HBM3 at a 400 W power limit its kernels took 0.9 ms of a 270-300 ms page-cached K = 23 read,
// tools/srs_read_probe.py.)
int spb_srs_read_file_custom(spb_ctx* ctx, const char* path, int format, spb_srs** out) {
  if (!ctx || !path || !out) return SPB_ERR_ARG;
  if (format != SPB_SERDE_RAW_BYTES && format != SPB_SERDE_RAW_BYTES_UNCHECKED)
    return set_error(ctx, SPB_ERR_ARG, "spb_srs_read_file_custom: unknown format %d (SPB_SERDE_RAW_BYTES or SPB_SERDE_RAW_BYTES_UNCHECKED)", format);
  const bool checked = format == SPB_SERDE_RAW_BYTES;
  FILE* f = fopen(path, "rb");
  if (!f) return set_error(ctx, SPB_ERR_ARG, "spb_srs_read_file: cannot open %s", path);
  uint32_t k = 0;
  if (fread(&k, 4, 1, f) != 1 || k > 28) { fclose(f); return set_error(ctx, SPB_ERR_ARG, "spb_srs_read_file: bad header in %s", path); }
  spb_srs* s;
  int rc = 0;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    s = srs_alloc(ctx, k);
    float check_ms = 0.f;
    for (int which = 0; which < 2 && rc == 0; which++) {
      for (auto& sh : s->shards) {
        DeviceState& d = ctx->dev[sh.dev_index];
        cudaSetDevice(d.device);
        G1Affine** dst = which == 0 ? &sh.g : &sh.g_lagrange;
        if (sh.count && cudaMalloc(dst, sh.count * sizeof(G1Affine)) != cudaSuccess) { rc = set_error(ctx, SPB_ERR_OOM, "spb_srs_read_file: cudaMalloc"); break; }
        if (sh.count) rc = stream_file_to_device(ctx, d, f, *dst, sh.count * sizeof(G1Affine), "spb_srs_read_file");
        if (rc == 0 && checked && sh.count) {
          size_t bad = sh.count;
          rc = srs_check_points(ctx, d, *dst, sh.count, &bad, &check_ms);
          if (rc == 0 && bad < sh.count) rc = srs_point_error(ctx, d, path, which == 0 ? "g" : "g_lagrange", *dst, bad, sh.start + bad);
        }
        if (rc) break;
      }
    }
    if (rc == 0 && (fread(s->g2, 128, 1, f) != 1 || fread(s->s_g2, 128, 1, f) != 1)) rc = set_error(ctx, SPB_ERR_ARG, "spb_srs_read_file: %s has no G2 trailer", path);
    for (int i = 0; i < 2 && rc == 0 && checked; i++) {
      static_assert(sizeof(G2Affine) == 128, "a G2 point of the trailer is 128 bytes");
      G2Affine q;
      memcpy(&q, i == 0 ? s->g2 : s->s_g2, sizeof q);
      const int v = g2_affine_check(q);
      if (v != kPointValid) rc = set_error(ctx, SPB_ERR_DATA, "spb_srs_read_file: %s: %s: %s", path, i == 0 ? "g2" : "s_g2", point_check_reason(v));
    }
    if (rc == 0 && checked) ctx->last_kernel_ms = check_ms;
  }
  fclose(f);
  if (rc) { spb_srs_free(ctx, s); return rc; }
  *out = s;
  return 0;
}

int spb_srs_read_file(spb_ctx* ctx, const char* path, spb_srs** out) { return spb_srs_read_file_custom(ctx, path, SPB_SERDE_RAW_BYTES_UNCHECKED, out); }

int spb_srs_write_file(spb_ctx* ctx, const spb_srs* srs, const char* path) {
  if (!ctx || !srs || !path) return SPB_ERR_ARG;
  if (srs->n != ((size_t)1 << srs->k)) return set_error(ctx, SPB_ERR_STATE, "spb_srs_write_file: the handle holds %zu plain bases (spb_bases_upload), not a 2^k SRS", srs->n);
  if (srs->table_c) return set_error(ctx, SPB_ERR_STATE, "spb_srs_write_file: call before spb_srs_precompute (rows 1.. are derived data)");
  FILE* f = fopen(path, "wb");
  if (!f) return set_error(ctx, SPB_ERR_ARG, "spb_srs_write_file: cannot create %s", path);
  int rc = 0;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    fwrite(&srs->k, 4, 1, f);
    for (int which = 0; which < 2 && rc == 0; which++)
      for (auto& sh : srs->shards) {
        const G1Affine* src = which == 0 ? sh.g : sh.g_lagrange;
        if (!src && sh.count) { rc = set_error(ctx, SPB_ERR_STATE, "spb_srs_write_file: basis %d not resident", which); break; }
        DeviceState& d = ctx->dev[sh.dev_index];
        cudaSetDevice(d.device);
        if (sh.count) rc = stream_device_to_file(ctx, d, f, src, sh.count * sizeof(G1Affine), "spb_srs_write_file");
        if (rc) break;
      }
    if (rc == 0) { fwrite(srs->g2, 128, 1, f); fwrite(srs->s_g2, 128, 1, f); }
  }
  fclose(f);
  return rc;
}

// G2 trailer of the params file (x.c0, x.c1, y.c0, y.c1 Montgomery limbs each): g2 and s_g2; set by the caller after
// spb_srs_setup / spb_srs_upload when the handle will be written out.
int spb_srs_set_g2(spb_ctx* ctx, spb_srs* srs, const unsigned char g2[128], const unsigned char s_g2[128]) {
  if (!ctx || !srs || !g2 || !s_g2) return SPB_ERR_ARG;
  memcpy(srs->g2, g2, 128); memcpy(srs->s_g2, s_g2, 128);
  return 0;
}
int spb_srs_get_g2(spb_ctx* ctx, const spb_srs* srs, unsigned char g2[128], unsigned char s_g2[128]) {
  if (!ctx || !srs || !g2 || !s_g2) return SPB_ERR_ARG;
  memcpy(g2, srs->g2, 128); memcpy(s_g2, srs->s_g2, 128);
  return 0;
}
uint32_t spb_srs_k(const spb_srs* srs) { return srs ? srs->k : 0; }

int spb_srs_download(spb_ctx* ctx, const spb_srs* srs, int basis, size_t start, size_t count, spb_g1_affine* out) {
  if (!ctx || !srs || !out || start + count > srs->n) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (auto& sh : srs->shards) {
    size_t lo = start > sh.start ? start : sh.start;
    size_t hi = (start + count) < (sh.start + sh.count) ? (start + count) : (sh.start + sh.count);
    if (lo >= hi) continue;
    const G1Affine* src = basis == SPB_BASIS_G ? sh.g : sh.g_lagrange;
    if (!src) return set_error(ctx, SPB_ERR_STATE, "spb_srs_download: basis %d not resident", basis);
    DeviceState& d = ctx->dev[sh.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    SPB_CUDA(ctx, cudaMemcpy((G1Affine*)out + (lo - start), src + (lo - sh.start), (hi - lo) * sizeof(G1Affine), cudaMemcpyDeviceToHost));
  }
  return 0;
}

// ---- MSM ---------------------------------------------------------------------------------------------------
int spb_msm_raw(spb_ctx* ctx, const spb_fr* scalars, const spb_g1_affine* bases, size_t n, spb_g1* out) {
  if (!ctx || !out || (n && (!scalars || !bases))) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->last_msm_adds = 0;
  std::vector<MsmPart> parts;
  size_t D = ctx->dev.size();
  for (size_t i = 0; i < D; i++) {
    size_t lo = n * i / D, cnt = n * (i + 1) / D - lo;
    if (!cnt) continue;
    DeviceState& d = ctx->dev[i];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    Lane* ln; SPB_TRY(get_lane(ctx, (int)i, 0, &ln));
    G1Affine* db = (G1Affine*)slot(ctx, d, "msm_raw_bases", cnt * sizeof(G1Affine));
    if (!db) return SPB_ERR_OOM;
    SPB_CUDA(ctx, cudaMemcpyAsync(db, (const G1Affine*)bases + lo, cnt * sizeof(G1Affine), cudaMemcpyHostToDevice, ln->stream));
    MsmPart p; p.dev_index = (int)i; p.d_scalars = nullptr; p.h_scalars = (const Fr*)scalars + lo; p.peer_src_device = -1;
    p.d_bases = db; p.n = cnt; p.g = msm_choose_geometry(cnt);
    parts.push_back(p);
  }
  SPB_TRY(job_enqueue(ctx, 0, parts));
  return job_collect(ctx, 0, parts, out);
}

// parts of one SRS-backed MSM (one per shard that intersects [0, n))
static int srs_parts(spb_ctx* ctx, const spb_srs* srs, int basis, const Fr* scalars, bool on_device, size_t n, std::vector<MsmPart>& parts) {
  if (n > srs->n) return set_error(ctx, SPB_ERR_ARG, "spb_msm: %zu scalars but the SRS has %zu points", n, srs->n);
  for (auto& sh : srs->shards) {
    if (sh.start >= n) continue;
    size_t cnt = (n - sh.start) < sh.count ? (n - sh.start) : sh.count;
    const G1Affine* b = basis == SPB_BASIS_G ? sh.g : sh.g_lagrange;
    if (!b) return set_error(ctx, SPB_ERR_STATE, "spb_msm: basis %d not resident", basis);
    MsmPart p; p.dev_index = sh.dev_index; p.d_bases = b; p.n = cnt; p.h_scalars = nullptr; p.d_scalars = nullptr; p.peer_src_device = -1;
    if (!on_device) p.h_scalars = scalars + sh.start;
    else { p.d_scalars = scalars + sh.start; if (sh.dev_index != 0) p.peer_src_device = ctx->dev[0].device; }
    p.g = srs->table_c ? msm_make_geometry(srs->table_c, true, (uint32_t)sh.count) : msm_choose_geometry(cnt);
    parts.push_back(p);
  }
  return 0;
}

static int msm_batch_common(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* scalars, bool on_device, size_t n, size_t count, spb_g1* out) {
  if (!ctx || !srs || !out || (count && !scalars)) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->last_msm_adds = 0;
  // every lane holds a workspace sized for these MSMs (the entries and the sort's second buffer, chunk pieces, buckets); lanes
  // beyond the first are used only while their workspaces together stay within a tenth of the device's memory (H100, 80 GB:
  // three lanes for a K = 23 SRS with tables, 2.7 GB each; one for K = 24 without, 6.2 GB), so a large proof keeps its memory
  // for its polynomials. (The sort's temporary storage, a few MB, is left out.)
  const MsmGeom lg = srs->table_c ? msm_make_geometry(srs->table_c, true, 0) : msm_choose_geometry(n ? n : 1);
  const uint64_t ents = (uint64_t)n * lg.W;
  const uint64_t lane_bytes = 2 * ents * sizeof(MsmEntry) + 2 * (ents / kShortChunk + 1) * (sizeof(G1Xyzz) + 4) + (uint64_t)lg.BW * lg.B * sizeof(G1Xyzz);
  const uint64_t fit = ctx->dev[0].total_mem / 10 / (lane_bytes ? lane_bytes : 1);
  const size_t NL = std::max<size_t>(1, std::min<size_t>((size_t)kMaxMsmLanes, (size_t)fit));
  std::vector<MsmPart> jobs[kMaxMsmLanes];
  for (size_t i = 0; i < count; i++) {
    int lane = (int)(i % NL);
    if (i >= NL) SPB_TRY(job_collect(ctx, lane, jobs[lane], &out[i - NL]));  // MSM i-NL ran on this lane
    if (n && !scalars[i]) return SPB_ERR_ARG;
    jobs[lane].clear();
    SPB_TRY(srs_parts(ctx, srs, basis, (const Fr*)scalars[i], on_device, n, jobs[lane]));
    SPB_TRY(job_enqueue(ctx, lane, jobs[lane]));
  }
  for (size_t i = count >= NL ? count - NL : 0; i < count; i++) SPB_TRY(job_collect(ctx, (int)(i % NL), jobs[i % NL], &out[i]));
  return 0;
}

int spb_msm(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* scalars, size_t n, spb_g1* out) {
  const spb_fr* one[1] = {scalars};
  if (n && !scalars) return SPB_ERR_ARG;
  return msm_batch_common(ctx, srs, basis, one, false, n, 1, out);
}
int spb_msm_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* d_scalars, size_t n, spb_g1* out) {
  const spb_fr* one[1] = {d_scalars};
  if (n && !d_scalars) return SPB_ERR_ARG;
  return msm_batch_common(ctx, srs, basis, one, true, n, 1, out);
}
int spb_msm_batch(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* scalars, size_t n, size_t count, spb_g1* out) {
  return msm_batch_common(ctx, srs, basis, scalars, false, n, count, out);
}
int spb_msm_batch_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* d_scalars, size_t n, size_t count, spb_g1* out) {
  return msm_batch_common(ctx, srs, basis, d_scalars, true, n, count, out);
}

// Build the 2^(c*j) multiples of both resident bases (c chosen for the full SRS length). Costs W x the basis
// memory; every later spb_msm* on this SRS then uses ONE bucket set for all windows (fewer, larger windows:
// W = 13 instead of 16 at k = 20) and needs no window Horner.
int spb_srs_precompute(spb_ctx* ctx, spb_srs* srs) {
  if (!ctx || !srs) return SPB_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (srs->table_c) return 0;
  size_t per_dev = srs->shards.empty() ? srs->n : srs->shards[0].count;
  uint32_t c = msm_choose_c(per_dev ? per_dev : 1, true);
  uint32_t W = (255 + c - 1) / c;
  // The tables are built only while they take at most a quarter of each device's memory: on an 80 GB H100 that keeps them
  // for both bases of a K = 23 SRS (12 GiB) but not of K = 24 (24 GiB), which would leave too little for the proof's
  // polynomials. Without tables the SRS keeps one bucket set per window; results are the same either way.
  for (auto& sh : srs->shards) {
    if (!sh.count) continue;
    SPB_CUDA(ctx, cudaSetDevice(ctx->dev[sh.dev_index].device));
    size_t free_b = 0, total_b = 0;
    SPB_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    const size_t bases = (sh.g ? 1 : 0) + (sh.g_lagrange ? 1 : 0);
    if ((size_t)W * sh.count * sizeof(G1Affine) * bases > total_b / 4) return 0;
  }
  for (auto& sh : srs->shards) {
    if (!sh.count) continue;
    DeviceState& d = ctx->dev[sh.dev_index];
    SPB_CUDA(ctx, cudaSetDevice(d.device));
    if ((uint64_t)W * sh.count >= 0x7fffffffull) return set_error(ctx, SPB_ERR_ARG, "spb_srs_precompute: table index exceeds 31 bits");
    for (int which = 0; which < 2; which++) {
      G1Affine** slotp = which == 0 ? &sh.g : &sh.g_lagrange;
      if (!*slotp) continue;
      G1Affine* tab = nullptr;
      cudaError_t e = cudaMalloc(&tab, (size_t)W * sh.count * sizeof(G1Affine));
      if (e != cudaSuccess) return set_error(ctx, SPB_ERR_OOM, "spb_srs_precompute: cudaMalloc(%zu): %s", (size_t)W * sh.count * sizeof(G1Affine), cudaGetErrorString(e));
      SPB_CUDA(ctx, cudaMemcpyAsync(tab, *slotp, sh.count * sizeof(G1Affine), cudaMemcpyDeviceToDevice, d.stream));
      SPB_TRY(launch(ctx, d.stream, nblk(sh.count, 128), 128, 0, msm_precompute_kernel, sh.count, c, W, tab));
      SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
      cudaFree(*slotp);
      *slotp = tab;
    }
  }
  srs->table_c = c;
  return 0;
}

int spb_g1_fixed_base_mul(spb_ctx* ctx, const spb_fr* scalars, size_t n, spb_g1_affine* out) {
  if (!ctx || !scalars || !out) return SPB_ERR_ARG;
  if (!n) return 0;
  SPB_ENTER(ctx);
  return run_staged(ctx, d, {{"srs_scalars", n * sizeof(Fr), scalars, nullptr}, {"fbm_out", n * sizeof(G1Affine), nullptr, out}},
                    [&](void* const* p) { return g1_fixed_base_mul(ctx, d, (const Fr*)p[0], n, (G1Affine*)p[1]); });
}

}  // extern "C"
