// Host build of the pairing's device bodies (spectre_b200/csrc/pairing.cuh), for tests/test_hostemu_pairing.py. Compiled
// twice: with -DSPB_EMULATE_PTX (the 32-bit-limb PTX carry chains the device runs) and without (the 64-bit host path).
#include "../../spectre_b200/csrc/pairing.cuh"
using namespace spb;
extern "C" {
// op 0 mul, 1 sqr, 2 inv (b unread for 1 and 2)
void he_fq6_op(int op, const Fq6* a, const Fq6* b, Fq6* out, size_t n) {
  for (size_t i = 0; i < n; i++) out[i] = op == 0 ? fq6_mul(a[i], b[i]) : op == 1 ? fq6_sqr(a[i]) : fq6_inv(a[i]);
}
// op 0 mul, 1 sqr, 2 inv, 3..5 the Frobenius maps p, p^2, p^3, 6 mul_by_034 with the line (b.c0.c0, b.c1.c0, b.c1.c1)
void he_fq12_op(int op, const Fq12* a, const Fq12* b, Fq12* out, size_t n) {
  for (size_t i = 0; i < n; i++) {
    switch (op) {
      case 0: fq12_mul(out[i], a[i], b[i]); break;
      case 1: fq12_sqr(out[i], a[i]); break;
      case 2: fq12_inv(out[i], a[i]); break;
      case 3: case 4: case 5: fq12_frobenius(out[i], a[i], op - 2); break;
      default: out[i] = a[i]; fq12_mul_by_034(out[i], b[i].c0.c0, b[i].c1.c0, b[i].c1.c1); break;
    }
  }
}
// out = final_exponentiation(prod_i miller_loop(p[i], q[i]))
void he_pairing(const G1Affine* p, const G2Affine* q, size_t n, Fq12* out) {
  Fq12 f = fq12_one(), m;
  for (size_t i = 0; i < n; i++) {
    miller_loop(m, p[i], q[i]);
    fq12_mul(f, f, m);
  }
  final_exponentiation(*out, f);
}
// g2_pairing_check verdicts: 0 valid, 1 x not canonical, 2 y not canonical, 3 off the twist, 4 not in the r-torsion subgroup
void he_g2_pairing_check(int* out, const G2Affine* q, size_t n) { for (size_t i = 0; i < n; i++) out[i] = g2_pairing_check(q[i]); }
}
