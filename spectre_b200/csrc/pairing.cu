// C ABI of the BN254 pairing: spb_pairing and spb_pairing_check_batch (include/spectre_b200.h). The arithmetic is in
// pairing.cuh; here are the three kernels and the staging around them.
//
// One call is one launch sequence on the context's first device: the input check (first_bad_launch: element 2i is pair i's
// G1 point, 2i + 1 its G2 point, so the lowest bad index is the first bad input in the order p[0], q[0], p[1], ...), then
// pairing_miller_kernel (one thread per pair, its Fq12 into the workspace) and pairing_final_kernel (one thread per check:
// the product of the check's Miller values, the final exponentiation, and the Gt value or the verdict). The launch count does
// not depend on the number of pairs or checks. One thread carries a whole Miller loop or final exponentiation: the kernels are
// latency-bound by design, and a batch of checks fills the GPU with independent threads.
#include "common.cuh"
#include "pairing.cuh"

using namespace spb;

static_assert(sizeof(spb_g2_affine) == sizeof(G2Affine) && sizeof(spb_gt) == sizeof(Fq12), "C ABI structs must match the device structs byte for byte");

namespace spb {

// an input of the pair list that fails its check: 2i = p[i] (affine_check), 2i + 1 = q[i] (g2_pairing_check)
struct PairInputBad {
  const G1Affine* p;
  const G2Affine* q;
  __device__ bool operator()(uint64_t i) const {
    return (i & 1) ? g2_pairing_check(q[i >> 1]) != kPointValid : affine_check(p[i >> 1]) != kPointValid;
  }
};

__global__ void __launch_bounds__(32) pairing_miller_kernel(const G1Affine* p, const G2Affine* q, Fq12* f, uint64_t n) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) {
    Fq12 r;
    miller_loop(r, p[i], q[i]);
    f[i] = r;
  }
}

// check j: final_exponentiation(prod_{i < m} f[j m + i]); gt (when not null) gets the value, ok (when not null) 1 iff it is one
__global__ void __launch_bounds__(32) pairing_final_kernel(const Fq12* f, uint64_t m, uint64_t n_checks, Fq12* gt, int32_t* ok) {
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j >= n_checks) return;
  Fq12 acc = f[j * m];
  for (uint64_t i = 1; i < m; i++) fq12_mul(acc, acc, f[j * m + i]);
  final_exponentiation(acc, acc);
  if (gt) gt[j] = acc;
  if (ok) ok[j] = fq12_is_one(acc) ? 1 : 0;
}

void g2_trailer_mul(unsigned char out[128], const unsigned char in[128], const Fr& t) {
  G2Affine q;
  memcpy(&q, in, sizeof q);
  q = g2_mul_scalar(q, fp_from_mont(t));
  memcpy(out, &q, sizeof q);
}

static const unsigned kPairingThreads = 32;  // small blocks: a few hundred pairs already spread over every SM

static const char* pairing_point_reason(int verdict) {
  switch (verdict) {
    case kPointXNotCanonical: return "x is not less than the field modulus";
    case kPointYNotCanonical: return "y is not less than the field modulus";
    case kPointOffCurve: return "not on the curve";
    case kPointNotInSubgroup: return "not in the r-torsion subgroup";
    default: return "rejected by the device check but valid on the host";
  }
}

// n pairs staged on device d -> (n / m) checks. gt or ok (device pointers) receive the result. Returns SPB_ERR_DATA naming the
// first invalid input, classified again on the host, before any Miller loop runs.
static int pairing_device(spb_ctx* ctx, DeviceState& d, const char* what, const G1Affine* dp, const G2Affine* dq, uint64_t n, uint64_t m, Fq12* dgt, int32_t* dok) {
  unsigned long long* first = (unsigned long long*)slot(ctx, d, "pairing_first", sizeof(unsigned long long));
  Fq12* f = (Fq12*)slot(ctx, d, "pairing_miller", n * sizeof(Fq12));
  if (!first || !f) return SPB_ERR_OOM;
  SPB_CUDA(ctx, cudaEventRecord(d.ev0, d.stream));
  SPB_CUDA(ctx, cudaMemsetAsync(first, 0xff, sizeof(unsigned long long), d.stream));
  SPB_TRY(first_bad_launch(ctx, d, PairInputBad{dp, dq}, 2 * n, first));
  unsigned long long bad = 0;
  SPB_CUDA(ctx, cudaMemcpyAsync(&bad, first, sizeof bad, cudaMemcpyDeviceToHost, d.stream));
  SPB_CUDA(ctx, cudaStreamSynchronize(d.stream));
  if (bad < 2 * n) {
    const uint64_t i = bad >> 1;
    int v;
    if (bad & 1) {
      G2Affine q;
      SPB_CUDA(ctx, cudaMemcpy(&q, dq + i, sizeof q, cudaMemcpyDeviceToHost));
      v = g2_pairing_check(q);
    } else {
      G1Affine p;
      SPB_CUDA(ctx, cudaMemcpy(&p, dp + i, sizeof p, cudaMemcpyDeviceToHost));
      v = affine_check(p);
    }
    return set_error(ctx, SPB_ERR_DATA, "%s: %s[%llu]: %s", what, (bad & 1) ? "q" : "p", (unsigned long long)i, pairing_point_reason(v));
  }
  SPB_TRY(launch(ctx, d.stream, nblk(n, kPairingThreads), kPairingThreads, 0, pairing_miller_kernel, dp, dq, f, n));
  const uint64_t n_checks = n / m;
  SPB_TRY(launch(ctx, d.stream, nblk(n_checks, kPairingThreads), kPairingThreads, 0, pairing_final_kernel, (const Fq12*)f, m, n_checks, dgt, dok));
  SPB_CUDA(ctx, cudaEventRecord(d.ev1, d.stream));
  return 0;
}

// Stage the n pairs, run pairing_device, download its n / m results (Gt values, or verdicts) into out.
static int pairing_host(spb_ctx* ctx, const char* what, const spb_g1_affine* p, const spb_g2_affine* q, uint64_t n, uint64_t m, void* out, bool verdicts) {
  SPB_ENTER(ctx);
  const uint64_t n_checks = n / m;
  const size_t out_bytes = n_checks * (verdicts ? sizeof(int32_t) : sizeof(Fq12));
  SPB_TRY(run_staged(ctx, d, {{"pairing_p", n * sizeof(G1Affine), p, nullptr}, {"pairing_q", n * sizeof(G2Affine), q, nullptr}, {"pairing_out", out_bytes, nullptr, out}},
                     [&](void* const* b) {
                       return pairing_device(ctx, d, what, (const G1Affine*)b[0], (const G2Affine*)b[1], n, m, verdicts ? nullptr : (Fq12*)b[2],
                                             verdicts ? (int32_t*)b[2] : nullptr);
                     }));
  SPB_CUDA(ctx, cudaEventElapsedTime(&ctx->last_kernel_ms, d.ev0, d.ev1));
  return 0;
}

}  // namespace spb

extern "C" {

int spb_pairing(spb_ctx* ctx, const spb_g1_affine* p, const spb_g2_affine* q, size_t n, spb_gt* out) {
  if (!ctx || !out || (n && (!p || !q))) return SPB_ERR_ARG;
  if (n == 0) {  // the empty product
    const Fq12 one = fq12_one();
    memcpy(out, &one, sizeof one);
    ctx->last_kernel_ms = 0.f;
    return 0;
  }
  return pairing_host(ctx, "spb_pairing", p, q, n, n, out, false);
}

int spb_pairing_check_batch(spb_ctx* ctx, const spb_g1_affine* p, const spb_g2_affine* q, size_t m, size_t n_checks, int32_t* ok) {
  if (!ctx || (n_checks && !ok) || (m && n_checks && (!p || !q))) return SPB_ERR_ARG;
  if (m && n_checks > SIZE_MAX / 2 / m / sizeof(Fq12)) return set_error(ctx, SPB_ERR_ARG, "spb_pairing_check_batch: %zu checks of %zu pairs is too many", n_checks, m);
  if (n_checks == 0 || m == 0) {  // no checks, or checks of empty products: all hold
    for (size_t j = 0; j < n_checks; j++) ok[j] = 1;
    ctx->last_kernel_ms = 0.f;
    return 0;
  }
  return pairing_host(ctx, "spb_pairing_check_batch", p, q, (uint64_t)m * n_checks, m, ok, true);
}

}  // extern "C"
