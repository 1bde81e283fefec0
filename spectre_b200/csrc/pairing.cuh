// BN254 optimal ate pairing: the tower Fq2 / Fq6 / Fq12, the Miller loop, the final exponentiation and the G2 subgroup check.
//
// Replaces halo2curves::bn256::{Fq6, Fq12, Gt, multi_miller_loop, final_exponentiation} ([UPSTREAM] halo2curves
// src/bn256/{fq6,fq12,engine}.rs), which halo2's KZG verifier reaches through `Bn256::multi_miller_loop` in
// poly/kzg/strategy.rs. Tower as upstream: Fq2 = Fq[u]/(u^2 + 1), Fq6 = Fq2[v]/(v^3 - xi) with xi = 9 + u,
// Fq12 = Fq6[w]/(w^2 - v); an Fq12 is 12 Montgomery Fq values in the order c0.c0.c0, c0.c0.c1, ..., c1.c2.c1 (384 B).
//
// Every function is SPB_HD so tests/hostemu/pairing.cpp compiles the same bodies for the host. The large ones are
// SPB_HD_NOINLINE: on the device one thread runs a whole Miller loop or final exponentiation, and inlining every Fq6 product
// would only multiply the code size of a latency-bound kernel. The Fq12 ones write their result through an out-parameter
// (which may alias an input: it is written last). A call that returned its 384 B by value would take a stack slot of its own
// at every call site, and the driver reserves the deepest per-thread stack for every thread the GPU can hold.
//
//   * Miller loop: 6u + 2 in NAF, G2 accumulator in homogeneous projective coordinates on the twist, each line evaluated at P
//     and multiplied in sparse form (three non-zero Fq2 coefficients, at w^0, w^1 and w^3), then the two extra steps at
//     pi(Q) and -pi^2(Q). Lines are scaled by Fq2 factors, which the final exponentiation removes.
//   * Final exponentiation: (p^6 - 1)(p^2 + 1) with one inversion, then exactly (p^4 - p^2 + 1) / r written in base p,
//     l0 + l1 p + l2 p^2 + l3 p^3 with l3 = 1, l2 = 6u^2 + 1, l1 = -36u^3 - 18u^2 - 12u + 1, l0 = -36u^3 - 30u^2 - 18u - 2
//     (tools/gen_constants.py asserts the identity): three exponentiations by u and short chains for the small multiples.
//     The result is f^((p^12 - 1) / r), not a power of it.
#pragma once
#include "curve.cuh"

#if defined(__CUDACC__)
#define SPB_HD_NOINLINE __host__ __device__ __noinline__
#else
#define SPB_HD_NOINLINE inline
#endif

namespace spb {

struct alignas(16) Fq6 { Fq2 c0, c1, c2; };
struct alignas(16) Fq12 { Fq6 c0, c1; };
struct alignas(16) G2Proj { Fq2 x, y, z; };  // homogeneous projective on the twist: (x/z, y/z), identity z = 0

// a G2 input that is on the twist but not in the order-r subgroup (extends PointCheck, curve.cuh)
static const int kPointNotInSubgroup = 4;

// ---- Fq2 -------------------------------------------------------------------------------------------------------------
SPB_HD Fq2 fq2_zero() { Fq2 r; r.c0 = fp_zero<FqParams>(); r.c1 = fp_zero<FqParams>(); return r; }
SPB_HD Fq2 fq2_one() { Fq2 r; r.c0 = fp_one<FqParams>(); r.c1 = fp_zero<FqParams>(); return r; }
SPB_HD Fq2 fq2_const(const uint32_t (&c0)[8], const uint32_t (&c1)[8]) {
  Fq2 r;
  for (int i = 0; i < 8; i++) { r.c0.l[i] = c0[i]; r.c1.l[i] = c1[i]; }
  return r;
}
SPB_HD bool fq2_is_zero(const Fq2& a) { return fp_is_zero(a.c0) && fp_is_zero(a.c1); }
SPB_HD bool fq2_eq(const Fq2& a, const Fq2& b) { return fp_eq(a.c0, b.c0) && fp_eq(a.c1, b.c1); }
SPB_HD Fq2 fq2_add(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = fp_add(a.c0, b.c0); r.c1 = fp_add(a.c1, b.c1); return r; }
SPB_HD Fq2 fq2_sub(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = fp_sub(a.c0, b.c0); r.c1 = fp_sub(a.c1, b.c1); return r; }
SPB_HD Fq2 fq2_neg(const Fq2& a) { Fq2 r; r.c0 = fp_neg(a.c0); r.c1 = fp_neg(a.c1); return r; }
SPB_HD Fq2 fq2_dbl(const Fq2& a) { return fq2_add(a, a); }
SPB_HD Fq2 fq2_conj(const Fq2& a) { Fq2 r; r.c0 = a.c0; r.c1 = fp_neg(a.c1); return r; }
SPB_HD Fq2 fq2_mul_fq(const Fq2& a, const Fq& s) { Fq2 r; r.c0 = fp_mul(a.c0, s); r.c1 = fp_mul(a.c1, s); return r; }
// (a0 + a1)(a0 - a1) + 2 a0 a1 u
SPB_HD Fq2 fq2_sqr(const Fq2& a) {
  Fq2 r;
  r.c0 = fp_mul(fp_add(a.c0, a.c1), fp_sub(a.c0, a.c1));
  r.c1 = fp_dbl(fp_mul(a.c0, a.c1));
  return r;
}
// (9 + u)(a0 + a1 u) = (9 a0 - a1) + (9 a1 + a0) u
SPB_HD Fq2 fq2_mul_xi(const Fq2& a) {
  Fq2 t = fq2_dbl(fq2_dbl(fq2_dbl(a)));
  t = fq2_add(t, a);
  Fq2 r;
  r.c0 = fp_sub(t.c0, a.c1);
  r.c1 = fp_add(t.c1, a.c0);
  return r;
}
// (a0 - a1 u) / (a0^2 + a1^2); inverse of zero is zero
SPB_HD Fq2 fq2_inv(const Fq2& a) {
  const Fq t = fp_inv(fp_add(fp_sqr(a.c0), fp_sqr(a.c1)));
  Fq2 r;
  r.c0 = fp_mul(a.c0, t);
  r.c1 = fp_neg(fp_mul(a.c1, t));
  return r;
}

// ---- Fq6 -------------------------------------------------------------------------------------------------------------
SPB_HD Fq6 fq6_zero() { Fq6 r; r.c0 = fq2_zero(); r.c1 = fq2_zero(); r.c2 = fq2_zero(); return r; }
SPB_HD Fq6 fq6_one() { Fq6 r; r.c0 = fq2_one(); r.c1 = fq2_zero(); r.c2 = fq2_zero(); return r; }
SPB_HD Fq6 fq6_add(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = fq2_add(a.c0, b.c0); r.c1 = fq2_add(a.c1, b.c1); r.c2 = fq2_add(a.c2, b.c2); return r; }
SPB_HD Fq6 fq6_sub(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = fq2_sub(a.c0, b.c0); r.c1 = fq2_sub(a.c1, b.c1); r.c2 = fq2_sub(a.c2, b.c2); return r; }
SPB_HD Fq6 fq6_neg(const Fq6& a) { Fq6 r; r.c0 = fq2_neg(a.c0); r.c1 = fq2_neg(a.c1); r.c2 = fq2_neg(a.c2); return r; }
// a v = xi a2 + a0 v + a1 v^2
SPB_HD Fq6 fq6_mul_v(const Fq6& a) { Fq6 r; r.c0 = fq2_mul_xi(a.c2); r.c1 = a.c0; r.c2 = a.c1; return r; }

// Karatsuba over three coefficients: 6 Fq2 products
SPB_HD_NOINLINE Fq6 fq6_mul(const Fq6& a, const Fq6& b) {
  const Fq2 v0 = fq2_mul(a.c0, b.c0), v1 = fq2_mul(a.c1, b.c1), v2 = fq2_mul(a.c2, b.c2);
  Fq6 r;
  r.c0 = fq2_add(v0, fq2_mul_xi(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c1, a.c2), fq2_add(b.c1, b.c2)), v1), v2)));
  r.c1 = fq2_add(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c0, a.c1), fq2_add(b.c0, b.c1)), v0), v1), fq2_mul_xi(v2));
  r.c2 = fq2_add(fq2_sub(fq2_sub(fq2_mul(fq2_add(a.c0, a.c2), fq2_add(b.c0, b.c2)), v0), v2), v1);
  return r;
}
// Chung-Hasan SQR2: s0 = a0^2, s1 = 2 a0 a1, s2 = (a0 - a1 + a2)^2, s3 = 2 a1 a2, s4 = a2^2
SPB_HD_NOINLINE Fq6 fq6_sqr(const Fq6& a) {
  const Fq2 s0 = fq2_sqr(a.c0), s1 = fq2_dbl(fq2_mul(a.c0, a.c1)), s2 = fq2_sqr(fq2_add(fq2_sub(a.c0, a.c1), a.c2));
  const Fq2 s3 = fq2_dbl(fq2_mul(a.c1, a.c2)), s4 = fq2_sqr(a.c2);
  Fq6 r;
  r.c0 = fq2_add(s0, fq2_mul_xi(s3));
  r.c1 = fq2_add(s1, fq2_mul_xi(s4));
  r.c2 = fq2_sub(fq2_sub(fq2_add(fq2_add(s1, s2), s3), s0), s4);
  return r;
}
// a (b0 + b1 v): the sparse Fq6 factor of a line
SPB_HD Fq6 fq6_mul_by_01(const Fq6& a, const Fq2& b0, const Fq2& b1) {
  Fq6 r;
  r.c0 = fq2_add(fq2_mul(a.c0, b0), fq2_mul_xi(fq2_mul(a.c2, b1)));
  r.c1 = fq2_add(fq2_mul(a.c0, b1), fq2_mul(a.c1, b0));
  r.c2 = fq2_add(fq2_mul(a.c1, b1), fq2_mul(a.c2, b0));
  return r;
}
// (A + B v + C v^2) / F with A = a0^2 - xi a1 a2, B = xi a2^2 - a0 a1, C = a1^2 - a0 a2, F = a0 A + xi (a2 B + a1 C): one Fq2 inversion
SPB_HD_NOINLINE Fq6 fq6_inv(const Fq6& a) {
  const Fq2 A = fq2_sub(fq2_sqr(a.c0), fq2_mul_xi(fq2_mul(a.c1, a.c2)));
  const Fq2 B = fq2_sub(fq2_mul_xi(fq2_sqr(a.c2)), fq2_mul(a.c0, a.c1));
  const Fq2 C = fq2_sub(fq2_sqr(a.c1), fq2_mul(a.c0, a.c2));
  const Fq2 F = fq2_add(fq2_mul(a.c0, A), fq2_mul_xi(fq2_add(fq2_mul(a.c2, B), fq2_mul(a.c1, C))));
  const Fq2 fi = fq2_inv(F);
  Fq6 r;
  r.c0 = fq2_mul(A, fi);
  r.c1 = fq2_mul(B, fi);
  r.c2 = fq2_mul(C, fi);
  return r;
}

// ---- Fq12 ------------------------------------------------------------------------------------------------------------
SPB_HD Fq12 fq12_one() { Fq12 r; r.c0 = fq6_one(); r.c1 = fq6_zero(); return r; }
SPB_HD bool fq12_is_one(const Fq12& a) {
  const Fq12 one = fq12_one();
  const Fq2* x = &a.c0.c0;
  const Fq2* y = &one.c0.c0;
  bool eq = true;
  for (int i = 0; i < 6; i++) eq = eq && fq2_eq(x[i], y[i]);
  return eq;
}
SPB_HD Fq12 fq12_conj(const Fq12& a) { Fq12 r; r.c0 = a.c0; r.c1 = fq6_neg(a.c1); return r; }

// Karatsuba: (a0 + a1 w)(b0 + b1 w) = a0 b0 + v a1 b1 + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) w
SPB_HD_NOINLINE void fq12_mul(Fq12& r, const Fq12& a, const Fq12& b) {
  const Fq6 aa = fq6_mul(a.c0, b.c0), bb = fq6_mul(a.c1, b.c1);
  r.c1 = fq6_sub(fq6_sub(fq6_mul(fq6_add(a.c0, a.c1), fq6_add(b.c0, b.c1)), aa), bb);
  r.c0 = fq6_add(aa, fq6_mul_v(bb));
}
// complex squaring: c0 = (a0 + a1)(a0 + v a1) - t - v t, c1 = 2 t, t = a0 a1
SPB_HD_NOINLINE void fq12_sqr(Fq12& r, const Fq12& a) {
  const Fq6 t = fq6_mul(a.c0, a.c1);
  r.c0 = fq6_sub(fq6_sub(fq6_mul(fq6_add(a.c0, a.c1), fq6_add(a.c0, fq6_mul_v(a.c1))), t), fq6_mul_v(t));
  r.c1 = fq6_add(t, t);
}
// (a0 - a1 w) / (a0^2 - v a1^2): one Fq6 inversion
SPB_HD_NOINLINE void fq12_inv(Fq12& r, const Fq12& a) {
  const Fq6 d = fq6_inv(fq6_sub(fq6_sqr(a.c0), fq6_mul_v(fq6_sqr(a.c1))));
  const Fq6 c1 = fq6_neg(fq6_mul(a.c1, d));
  r.c0 = fq6_mul(a.c0, d);
  r.c1 = c1;
}
// f *= a line l0 + l1 w + l3 w^3 (l0 at c0.c0, l1 at c1.c0, l3 at c1.c1): 15 Fq2 products instead of a full product's 18
SPB_HD_NOINLINE void fq12_mul_by_034(Fq12& f, const Fq2& l0, const Fq2& l1, const Fq2& l3) {
  Fq6 aa;
  aa.c0 = fq2_mul(f.c0.c0, l0); aa.c1 = fq2_mul(f.c0.c1, l0); aa.c2 = fq2_mul(f.c0.c2, l0);
  const Fq6 bb = fq6_mul_by_01(f.c1, l1, l3);
  f.c1 = fq6_sub(fq6_sub(fq6_mul_by_01(fq6_add(f.c0, f.c1), fq2_add(l0, l1), l3), aa), bb);
  f.c0 = fq6_add(aa, fq6_mul_v(bb));
}

// xi^(i (p^k - 1) / 6) for k = 1, 2, 3 and i = 1..5 (tools/gen_constants.py); gamma(k, 0) = 1. One table in constant memory on
// the device (a local copy would be rebuilt in every calling thread's stack), a static one on the host.
#define SPB_FQ12_GAMMA_TABLE                                                                                                   \
  {{{SPB_FQ12_GAMMA_1_1_C0_MONT, SPB_FQ12_GAMMA_1_1_C1_MONT}, {SPB_FQ12_GAMMA_1_2_C0_MONT, SPB_FQ12_GAMMA_1_2_C1_MONT},       \
    {SPB_FQ12_GAMMA_1_3_C0_MONT, SPB_FQ12_GAMMA_1_3_C1_MONT}, {SPB_FQ12_GAMMA_1_4_C0_MONT, SPB_FQ12_GAMMA_1_4_C1_MONT},       \
    {SPB_FQ12_GAMMA_1_5_C0_MONT, SPB_FQ12_GAMMA_1_5_C1_MONT}},                                                               \
   {{SPB_FQ12_GAMMA_2_1_C0_MONT, SPB_FQ12_GAMMA_2_1_C1_MONT}, {SPB_FQ12_GAMMA_2_2_C0_MONT, SPB_FQ12_GAMMA_2_2_C1_MONT},       \
    {SPB_FQ12_GAMMA_2_3_C0_MONT, SPB_FQ12_GAMMA_2_3_C1_MONT}, {SPB_FQ12_GAMMA_2_4_C0_MONT, SPB_FQ12_GAMMA_2_4_C1_MONT},       \
    {SPB_FQ12_GAMMA_2_5_C0_MONT, SPB_FQ12_GAMMA_2_5_C1_MONT}},                                                               \
   {{SPB_FQ12_GAMMA_3_1_C0_MONT, SPB_FQ12_GAMMA_3_1_C1_MONT}, {SPB_FQ12_GAMMA_3_2_C0_MONT, SPB_FQ12_GAMMA_3_2_C1_MONT},       \
    {SPB_FQ12_GAMMA_3_3_C0_MONT, SPB_FQ12_GAMMA_3_3_C1_MONT}, {SPB_FQ12_GAMMA_3_4_C0_MONT, SPB_FQ12_GAMMA_3_4_C1_MONT},       \
    {SPB_FQ12_GAMMA_3_5_C0_MONT, SPB_FQ12_GAMMA_3_5_C1_MONT}}}
#if defined(__CUDACC__)
static __constant__ uint32_t kFq12GammaDev[3][5][2][8] = SPB_FQ12_GAMMA_TABLE;
#endif
static const uint32_t kFq12GammaHost[3][5][2][8] = SPB_FQ12_GAMMA_TABLE;
SPB_HD Fq2 fq12_gamma(int k, int i) {
#if defined(__CUDA_ARCH__)
  const uint32_t(&t)[2][8] = kFq12GammaDev[k - 1][i - 1];
#else
  const uint32_t(&t)[2][8] = kFq12GammaHost[k - 1][i - 1];
#endif
  return fq2_const(t[0], t[1]);
}
// a^(p^k), k = 1, 2, 3: the coefficient of w^i (c0.cj: i = 2j, c1.cj: i = 2j + 1) goes to frob^k(c) gamma(k, i)
SPB_HD_NOINLINE void fq12_frobenius(Fq12& r, const Fq12& a, int k) {
  const Fq2* src = &a.c0.c0;
  Fq2* dst = &r.c0.c0;
  for (int j = 0; j < 6; j++) {  // slot j reads only slot j: r may alias a
    const int i = j < 3 ? 2 * j : 2 * (j - 3) + 1;  // power of w of tower slot j
    const Fq2 c = (k & 1) ? fq2_conj(src[j]) : src[j];
    dst[j] = i == 0 ? c : fq2_mul(c, fq12_gamma(k, i));
  }
}

// ---- G2 on the twist y^2 = x^3 + b', b' = 3 / xi -------------------------------------------------------------------------
SPB_HD bool g2_affine_is_identity(const G2Affine& q) { return fq2_is_zero(q.x) && fq2_is_zero(q.y); }
SPB_HD Fq2 g2_twist_b() {
  constexpr uint32_t c0[8] = SPB_FQ2_TWIST_B_C0_MONT, c1[8] = SPB_FQ2_TWIST_B_C1_MONT;
  return fq2_const(c0, c1);
}
SPB_HD Fq fq_two_inv() { constexpr uint32_t v[8] = SPB_FQ_TWO_INV_MONT; Fq r; for (int i = 0; i < 8; i++) r.l[i] = v[i]; return r; }

// 2T for T = (X, Y, Z) with a = 0 (Costello-Lange-Naehrig 2010, as in Aranha et al. 2011 eq. 10):
//   A = XY/2, B = Y^2, C = Z^2, E = 3b'C, F = 3E, G = (B + F)/2, H = (Y + Z)^2 - B - C, I = E - B, J = X^2
//   X3 = A (B - F), Y3 = G^2 - 3E^2, Z3 = B H.
// The tangent at T evaluated at P = (xP, yP), scaled by -2YZ: l = -H yP + 3J xP w + I w^3. T = O or a point of order 2 gives Z3 = 0.
SPB_HD void g2_dbl_step(G2Proj& t, Fq2* l0, Fq2* l1, Fq2* l3, const Fq& xp, const Fq& yp) {
  const Fq two_inv = fq_two_inv();
  const Fq2 A = fq2_mul_fq(fq2_mul(t.x, t.y), two_inv);
  const Fq2 B = fq2_sqr(t.y), C = fq2_sqr(t.z);
  const Fq2 bC = fq2_mul(g2_twist_b(), C);
  const Fq2 E = fq2_add(fq2_dbl(bC), bC);
  const Fq2 F = fq2_add(fq2_dbl(E), E);
  const Fq2 G = fq2_mul_fq(fq2_add(B, F), two_inv);
  const Fq2 H = fq2_sub(fq2_sqr(fq2_add(t.y, t.z)), fq2_add(B, C));
  const Fq2 J = fq2_sqr(t.x);
  const Fq2 E2 = fq2_sqr(E);
  if (l0) {
    *l0 = fq2_neg(fq2_mul_fq(H, yp));
    *l1 = fq2_mul_fq(fq2_add(fq2_dbl(J), J), xp);
    *l3 = fq2_sub(E, B);
  }
  t.x = fq2_mul(A, fq2_sub(B, F));
  t.y = fq2_sub(fq2_sqr(G), fq2_add(fq2_dbl(E2), E2));
  t.z = fq2_mul(B, H);
}
// T + Q for affine Q = (x2, y2), T != +-Q, neither the identity (Aranha et al. 2011 eq. 12):
//   theta = Y - y2 Z, lambda = X - x2 Z, C = theta^2, D = lambda^2, E = lambda D, F = Z C, G = X D, H = E + F - 2G
//   X3 = lambda H, Y3 = theta (G - H) - Y E, Z3 = Z E.
// The chord evaluated at P, scaled by lambda: l = lambda yP - theta xP w + (theta x2 - lambda y2) w^3.
SPB_HD void g2_add_step(G2Proj& t, const G2Affine& q, Fq2* l0, Fq2* l1, Fq2* l3, const Fq& xp, const Fq& yp) {
  const Fq2 theta = fq2_sub(t.y, fq2_mul(q.y, t.z));
  const Fq2 lambda = fq2_sub(t.x, fq2_mul(q.x, t.z));
  const Fq2 C = fq2_sqr(theta), D = fq2_sqr(lambda);
  const Fq2 E = fq2_mul(lambda, D), F = fq2_mul(t.z, C), G = fq2_mul(t.x, D);
  const Fq2 H = fq2_sub(fq2_add(E, F), fq2_dbl(G));
  if (l0) {
    *l0 = fq2_mul_fq(lambda, yp);
    *l1 = fq2_neg(fq2_mul_fq(theta, xp));
    *l3 = fq2_sub(fq2_mul(theta, q.x), fq2_mul(lambda, q.y));
  }
  const Fq2 ye = fq2_mul(t.y, E);
  t.x = fq2_mul(lambda, H);
  t.y = fq2_sub(fq2_mul(theta, fq2_sub(G, H)), ye);
  t.z = fq2_mul(t.z, E);
}

// T + Q with every exceptional case resolved (for the subgroup check, where T may meet +-Q or the identity)
SPB_HD void g2_add_complete(G2Proj& t, const G2Affine& q) {
  if (fq2_is_zero(t.z)) { t.x = q.x; t.y = q.y; t.z = fq2_one(); return; }
  const Fq2 theta = fq2_sub(t.y, fq2_mul(q.y, t.z));
  const Fq2 lambda = fq2_sub(t.x, fq2_mul(q.x, t.z));
  if (fq2_is_zero(lambda)) {
    if (fq2_is_zero(theta)) g2_dbl_step(t, nullptr, nullptr, nullptr, fp_zero<FqParams>(), fp_zero<FqParams>());
    else { t.x = fq2_zero(); t.y = fq2_one(); t.z = fq2_zero(); }
    return;
  }
  g2_add_step(t, q, nullptr, nullptr, nullptr, fp_zero<FqParams>(), fp_zero<FqParams>());
}

// [r]Q == O for a point already known to be on the twist: double-and-add over the bits of r
SPB_HD_NOINLINE bool g2_in_subgroup(const G2Affine& q) {
  if (g2_affine_is_identity(q)) return true;
  G2Proj t; t.x = q.x; t.y = q.y; t.z = fq2_one();
  for (int i = 252; i >= 0; i--) {  // r < 2^254, bit 253 set: it is the starting T = Q
    g2_dbl_step(t, nullptr, nullptr, nullptr, fp_zero<FqParams>(), fp_zero<FqParams>());
    if ((FrParams::mod(i >> 5) >> (i & 31)) & 1) g2_add_complete(t, q);
  }
  return fq2_is_zero(t.z);
}

// k Q for a canonical (non-Montgomery) scalar k, as an affine point (identity (0, 0)): MSB-first double-and-add over the steps
// of g2_in_subgroup, then one Fq2 inversion. The G2 trailer of a powers-of-tau update (spb_srs_contribute), run on the host.
SPB_HD_NOINLINE G2Affine g2_mul_scalar(const G2Affine& q, const Fr& k) {
  G2Proj t; t.x = fq2_zero(); t.y = fq2_one(); t.z = fq2_zero();
  if (!g2_affine_is_identity(q))
    for (int i = 255; i >= 0; i--) {
      if (!fq2_is_zero(t.z)) g2_dbl_step(t, nullptr, nullptr, nullptr, fp_zero<FqParams>(), fp_zero<FqParams>());
      if ((k.l[i >> 5] >> (i & 31)) & 1) g2_add_complete(t, q);
    }
  G2Affine r; r.x = fq2_zero(); r.y = fq2_zero();
  if (fq2_is_zero(t.z)) return r;
  const Fq2 zi = fq2_inv(t.z);
  r.x = fq2_mul(t.x, zi);
  r.y = fq2_mul(t.y, zi);
  return r;
}

// The input check of a pairing's G2 point: g2_affine_check (canonical, on the twist), then membership in the order-r subgroup.
SPB_HD int g2_pairing_check(const G2Affine& q) {
  const int v = g2_affine_check(q);
  if (v != kPointValid) return v;
  return g2_in_subgroup(q) ? kPointValid : kPointNotInSubgroup;
}

// ---- the pairing -----------------------------------------------------------------------------------------------------
// f_{6u+2,Q}(P) l_{[6u+2]Q, pi(Q)}(P) l_{[6u+2]Q + pi(Q), -pi^2(Q)}(P) for P in G1 and Q in G2 (both checked); 1 when either is
// the identity, as upstream's multi_miller_loop and EIP-197 treat such a pair.
SPB_HD_NOINLINE void miller_loop(Fq12& f, const G1Affine& p, const G2Affine& q) {
  f = fq12_one();
  if (affine_is_identity(p) || g2_affine_is_identity(q)) return;
  G2Affine nq; nq.x = q.x; nq.y = fq2_neg(q.y);
  G2Proj t; t.x = q.x; t.y = q.y; t.z = fq2_one();
  constexpr int8_t naf[SPB_BN_ATE_NAF_LEN] = SPB_BN_ATE_NAF;
  Fq2 l0, l1, l3;
  for (int i = SPB_BN_ATE_NAF_LEN - 2; i >= 0; i--) {
    fq12_sqr(f, f);
    g2_dbl_step(t, &l0, &l1, &l3, p.x, p.y);
    fq12_mul_by_034(f, l0, l1, l3);
    if (naf[i]) {
      g2_add_step(t, naf[i] > 0 ? q : nq, &l0, &l1, &l3, p.x, p.y);
      fq12_mul_by_034(f, l0, l1, l3);
    }
  }
  // pi(Q) = (conj(x) gamma_1_2, conj(y) gamma_1_3), -pi^2(Q) = (x gamma_2_2, -y gamma_2_3)
  G2Affine q1, q2;
  q1.x = fq2_mul(fq2_conj(q.x), fq12_gamma(1, 2));
  q1.y = fq2_mul(fq2_conj(q.y), fq12_gamma(1, 3));
  q2.x = fq2_mul(q.x, fq12_gamma(2, 2));
  q2.y = fq2_neg(fq2_mul(q.y, fq12_gamma(2, 3)));
  g2_add_step(t, q1, &l0, &l1, &l3, p.x, p.y);
  fq12_mul_by_034(f, l0, l1, l3);
  g2_add_step(t, q2, &l0, &l1, &l3, p.x, p.y);
  fq12_mul_by_034(f, l0, l1, l3);
}

// r = a^u, u = SPB_BN_U (positive, 63 bits): square-and-multiply from the top bit. r must not alias a.
SPB_HD_NOINLINE void fq12_pow_u(Fq12& r, const Fq12& a) {
  const uint64_t u = SPB_BN_U;
  r = a;
  for (int i = 61; i >= 0; i--) {  // bit 62 is the top bit of u
    fq12_sqr(r, r);
    if ((u >> i) & 1) fq12_mul(r, r, a);
  }
}

// r = f^((p^12 - 1) / r), r may alias f. f must be non-zero (a Miller value of checked points is). Eight named Fq12 values,
// each result written into one of them.
SPB_HD_NOINLINE void final_exponentiation(Fq12& r, const Fq12& f) {
  Fq12 g, t, a, b, c, a6, b6, t1;
  // easy part: g = f^((p^6 - 1)(p^2 + 1)); g lies in the cyclotomic subgroup, where the inverse is the conjugate
  fq12_inv(t, f);
  g = fq12_conj(f);
  fq12_mul(g, g, t);
  fq12_frobenius(t, g, 2);
  fq12_mul(g, t, g);
  // hard part: g^(l0 + l1 p + l2 p^2 + p^3)
  fq12_pow_u(a, g);                                           // g^u
  fq12_pow_u(b, a);                                           // g^(u^2)
  fq12_pow_u(c, b);                                           // g^(u^3)
  fq12_sqr(t, a); fq12_mul(t, t, a); fq12_sqr(a6, t);         // g^(6u)
  fq12_sqr(a, a6);                                            // g^(12u)
  fq12_sqr(t, b); fq12_mul(t, t, b); fq12_sqr(b6, t);         // g^(6u^2)
  fq12_sqr(b, b6);                                            // g^(12u^2)
  fq12_sqr(t, c); fq12_sqr(t, t); fq12_sqr(t, t); fq12_mul(c, t, c);
  fq12_sqr(c, c); fq12_sqr(c, c);                             // g^(36u^3)
  fq12_mul(t1, c, b); fq12_mul(t1, t1, b6); fq12_mul(t1, t1, a);   // g^(36u^3 + 18u^2 + 12u) = g^(1 - l1)
  fq12_mul(c, t1, b); fq12_mul(c, c, a6);
  fq12_sqr(t, g); fq12_mul(c, c, t);                          // g^(36u^3 + 30u^2 + 18u + 2) = g^(-l0)
  t1 = fq12_conj(t1); fq12_mul(t1, t1, g); fq12_frobenius(t1, t1, 1);   // (g^l1)^p
  c = fq12_conj(c); fq12_mul(c, c, t1);                       // g^(l0 + l1 p)
  fq12_mul(b6, b6, g); fq12_frobenius(b6, b6, 2); fq12_mul(c, c, b6);   // (g^(6u^2 + 1))^(p^2) = (g^l2)^(p^2)
  fq12_frobenius(t, g, 3);
  fq12_mul(r, c, t);
}

}  // namespace spb
