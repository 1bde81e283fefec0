// Host build of a powers-of-tau update's bodies for tests/test_hostemu_params_update.py: the per-point scale of
// spb_srs_contribute's kernel (spectre_b200/csrc/msm.cuh, srs_scale_thread) and the G2 multiple of its trailer
// (spectre_b200/csrc/pairing.cuh, g2_mul_scalar). Compiled with -DSPB_EMULATE_PTX (the 32-bit-limb carry chains the device
// runs) and without it (the 64-bit host path the trailer takes in the library).
#include "../../spectre_b200/csrc/msm.cuh"
#include "../../spectre_b200/csrc/pairing.cuh"
using namespace spb;

extern "C" {
// out[j] = t^(start + j) in[j] for j < n: every thread of the kernel's grid, one past the end included (it writes nothing)
void he_srs_scale(const G1Affine* in, G1Affine* out, uint64_t start, uint64_t n, const Fr* t) {
  for (uint64_t j = 0; j <= n; j++) srs_scale_thread(j, start, n, *t, in, out);
}
// out = t q for t in Montgomery limbs, as the library's trailer update takes it
void he_g2_mul(const G2Affine* q, const Fr* t, G2Affine* out) { *out = g2_mul_scalar(*q, fp_from_mont(*t)); }
}
