// Host build of the params-file point checks (spectre_b200/csrc/{field,curve}.cuh), for tests/test_hostemu_srs_check.py.
// Compiled twice: with -DSPB_EMULATE_PTX (the 32-bit-limb PTX carry chains the device runs) and without (the 64-bit host
// path the library's G2 trailer check takes).
#include "../../spectre_b200/csrc/curve.cuh"
using namespace spb;
extern "C" {
// verdicts of the params-file point checks (0 valid, 1 x not canonical, 2 y not canonical, 3 off the curve)
void he_g1_check(int* out, const G1Affine* p, size_t n) { for (size_t i = 0; i < n; i++) out[i] = affine_check(p[i]); }
void he_g2_check(int* out, const G2Affine* p, size_t n) { for (size_t i = 0; i < n; i++) out[i] = g2_affine_check(p[i]); }
}
