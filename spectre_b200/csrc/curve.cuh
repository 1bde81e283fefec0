// BN254 G1 (y^2 = x^3 + 3 over Fq) group law, and the validity checks of stored G1 / G2 points.
//
// Replaces halo2curves::bn256::{G1, G1Affine} ([UPSTREAM] halo2curves src/bn256/curve.rs + src/derive/curve.rs;
// types named by the reference at lightclient-circuits/src/util/circuit.rs:12). Conventions kept:
//   * G1Affine = {x, y} Montgomery Fq, 64 bytes, identity encoded as x = y = 0;
//   * G1 (what best_multiexp returns) = Jacobian {x, y, z}, affine = (x/z^2, y/z^3), identity z = 0.
// Internally the MSM accumulates in extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ,
// ZZ^3 = ZZZ^2): a mixed add costs 8M + 2S instead of Jacobian's 7M + 4S and needs no field doubling
// chains, which is what an IMAD-bound kernel wants. Formulas: Explicit-Formulas Database,
// short Weierstrass / xyzz: madd-2008-s, add-2008-s, dbl-2008-s-1, mdbl-2008-s-1 (a = 0).
// Everything here is exact for every input, including P + P, P + (-P), identity operands and affine (0,0).
#pragma once
#include "field.cuh"

namespace spb {

struct alignas(16) G1Affine { Fq x, y; };          // 64 B, identity = (0,0)
struct alignas(16) G1Jac    { Fq x, y, z; };       // 96 B, identity z = 0
struct alignas(16) G1Xyzz   { Fq x, y, zz, zzz; }; // 128 B, identity zz = 0

SPB_HD bool affine_is_identity(const G1Affine& p) { return fp_is_zero(p.x) && fp_is_zero(p.y); }
SPB_HD bool xyzz_is_identity(const G1Xyzz& p) { return fp_is_zero(p.zz); }
SPB_HD G1Xyzz xyzz_identity() {
  G1Xyzz r; r.x = fp_zero<FqParams>(); r.y = fp_one<FqParams>(); r.zz = fp_zero<FqParams>(); r.zzz = fp_zero<FqParams>();
  return r;
}
SPB_HD G1Xyzz xyzz_from_affine(const G1Affine& p) {
  if (affine_is_identity(p)) return xyzz_identity();
  G1Xyzz r; r.x = p.x; r.y = p.y; r.zz = fp_one<FqParams>(); r.zzz = fp_one<FqParams>();
  return r;
}
SPB_HD G1Affine affine_neg(const G1Affine& p) { G1Affine r; r.x = p.x; r.y = fp_neg(p.y); return r; }
SPB_HD G1Xyzz xyzz_neg(const G1Xyzz& p) { G1Xyzz r = p; r.y = fp_neg(p.y); return r; }

// 2*(x,y) for a finite affine point: mdbl-2008-s-1
SPB_HD G1Xyzz xyzz_dbl_affine(const G1Affine& p) {
  Fq u = fp_dbl(p.y);
  Fq v = fp_sqr(u);
  Fq w = fp_mul(u, v);
  Fq s = fp_mul(p.x, v);
  Fq xx = fp_sqr(p.x);
  Fq m = fp_add(fp_dbl(xx), xx);
  G1Xyzz r;
  r.x = fp_sub(fp_sqr(m), fp_dbl(s));
  r.y = fp_mul_sub_mul(m, fp_sub(s, r.x), w, p.y);
  r.zz = v;
  r.zzz = w;
  return r;  // y = 0 cannot occur on a prime-order curve, so zz != 0
}

// 2*P: dbl-2008-s-1
SPB_HD G1Xyzz xyzz_dbl(const G1Xyzz& p) {
  if (xyzz_is_identity(p)) return p;
  Fq u = fp_dbl(p.y);
  Fq v = fp_sqr(u);
  Fq w = fp_mul(u, v);
  Fq s = fp_mul(p.x, v);
  Fq xx = fp_sqr(p.x);
  Fq m = fp_add(fp_dbl(xx), xx);
  G1Xyzz r;
  r.x = fp_sub(fp_sqr(m), fp_dbl(s));
  r.y = fp_mul_sub_mul(m, fp_sub(s, r.x), w, p.y);
  r.zz = fp_mul(v, p.zz);
  r.zzz = fp_mul(w, p.zzz);
  return r;
}

// acc += q (q affine): madd-2008-s with the exceptional cases resolved exactly.
SPB_HD void xyzz_add_mixed(G1Xyzz& acc, const G1Affine& q) {
  if (affine_is_identity(q)) return;
  if (xyzz_is_identity(acc)) { acc.x = q.x; acc.y = q.y; acc.zz = fp_one<FqParams>(); acc.zzz = fp_one<FqParams>(); return; }
  Fq u2 = fp_mul(q.x, acc.zz);
  Fq s2 = fp_mul(q.y, acc.zzz);
  Fq p = fp_sub(u2, acc.x);
  Fq r = fp_sub(s2, acc.y);
  if (fp_is_zero(p)) {
    if (fp_is_zero(r)) acc = xyzz_dbl_affine(q);
    else acc = xyzz_identity();
    return;
  }
  Fq pp = fp_sqr(p);
  Fq ppp = fp_mul(p, pp);
  Fq qq = fp_mul(acc.x, pp);
  Fq x3 = fp_sub(fp_sub(fp_sqr(r), ppp), fp_dbl(qq));
  Fq y3 = fp_mul_sub_mul(r, fp_sub(qq, x3), acc.y, ppp);
  acc.x = x3;
  acc.y = y3;
  acc.zz = fp_mul(acc.zz, pp);
  acc.zzz = fp_mul(acc.zzz, ppp);
}

// acc += q (both XYZZ): add-2008-s with the exceptional cases resolved exactly.
SPB_HD void xyzz_add(G1Xyzz& acc, const G1Xyzz& q) {
  if (xyzz_is_identity(q)) return;
  if (xyzz_is_identity(acc)) { acc = q; return; }
  Fq u1 = fp_mul(acc.x, q.zz);
  Fq u2 = fp_mul(q.x, acc.zz);
  Fq s1 = fp_mul(acc.y, q.zzz);
  Fq s2 = fp_mul(q.y, acc.zzz);
  Fq p = fp_sub(u2, u1);
  Fq r = fp_sub(s2, s1);
  if (fp_is_zero(p)) {
    if (fp_is_zero(r)) acc = xyzz_dbl(acc);
    else acc = xyzz_identity();
    return;
  }
  Fq pp = fp_sqr(p);
  Fq ppp = fp_mul(p, pp);
  Fq qq = fp_mul(u1, pp);
  Fq x3 = fp_sub(fp_sub(fp_sqr(r), ppp), fp_dbl(qq));
  Fq y3 = fp_mul_sub_mul(r, fp_sub(qq, x3), s1, ppp);
  acc.x = x3;
  acc.y = y3;
  acc.zz = fp_mul(fp_mul(acc.zz, q.zz), pp);
  acc.zzz = fp_mul(fp_mul(acc.zzz, q.zzz), ppp);
}

// XYZZ -> affine (one inversion). Identity -> (0,0), halo2curves' encoding.
SPB_HD G1Affine xyzz_to_affine(const G1Xyzz& p) {
  G1Affine r;
  if (xyzz_is_identity(p)) { r.x = fp_zero<FqParams>(); r.y = fp_zero<FqParams>(); return r; }
  // 1/zzz, then 1/zz = zzz^-2 * zz^2  (since zz^3 = zzz^2)
  Fq izzz = fp_inv(p.zzz);
  Fq izz = fp_mul(fp_sqr(izzz), fp_sqr(p.zz));
  r.x = fp_mul(p.x, izz);
  r.y = fp_mul(p.y, izzz);
  return r;
}

// affine -> Jacobian as halo2curves' `G1::from(G1Affine)`/`to_curve()` does: z = 1, identity -> z = 0.
SPB_HD G1Jac jac_from_affine(const G1Affine& p) {
  G1Jac r;
  if (affine_is_identity(p)) { r.x = fp_zero<FqParams>(); r.y = fp_one<FqParams>(); r.z = fp_zero<FqParams>(); return r; }
  r.x = p.x; r.y = p.y; r.z = fp_one<FqParams>();
  return r;
}
SPB_HD G1Affine jac_to_affine(const G1Jac& p) {
  G1Affine r;
  if (fp_is_zero(p.z)) { r.x = fp_zero<FqParams>(); r.y = fp_zero<FqParams>(); return r; }
  Fq iz = fp_inv(p.z);
  Fq iz2 = fp_sqr(iz);
  r.x = fp_mul(p.x, iz2);
  r.y = fp_mul(p.y, fp_mul(iz2, iz));
  return r;
}
SPB_HD G1Xyzz xyzz_from_jac(const G1Jac& p) {
  if (fp_is_zero(p.z)) return xyzz_identity();
  G1Xyzz r; r.x = p.x; r.y = p.y; r.zz = fp_sqr(p.z); r.zzz = fp_mul(r.zz, p.z);
  return r;
}

// k*P for a small non-negative integer k (double-and-add, MSB first)
SPB_HD G1Xyzz xyzz_mul_u32(const G1Xyzz& p, uint32_t k) {
  G1Xyzz r = xyzz_identity();
  int top = 31;
  while (top >= 0 && !((k >> top) & 1)) top--;
  for (int i = top; i >= 0; i--) {
    r = xyzz_dbl(r);
    if ((k >> i) & 1) xyzz_add(r, p);
  }
  return r;
}

// is (x,y) on the curve (or the identity)?
SPB_HD bool affine_on_curve(const G1Affine& p) {
  if (affine_is_identity(p)) return true;
  Fq three; { constexpr uint32_t v[8] = SPB_FQ_THREE_MONT; for (int i = 0; i < 8; i++) three.l[i] = v[i]; }
  Fq lhs = fp_sqr(p.y);
  Fq rhs = fp_add(fp_mul(fp_sqr(p.x), p.x), three);
  return fp_eq(lhs, rhs);
}

// ---- checks of points read from outside (ParamsKZG::read, SerdeFormat::RawBytes) ----------------------------------------
// The verdict of a point check. The canonical tests come first: the field arithmetic assumes reduced inputs, so the curve
// equation is only evaluated on coordinates already known to be less than p.
enum PointCheck : int { kPointValid = 0, kPointXNotCanonical = 1, kPointYNotCanonical = 2, kPointOffCurve = 3 };

// a G1Affine as stored (raw Montgomery limbs): canonical coordinates and on y^2 = x^3 + 3, or the identity (0, 0)
SPB_HD int affine_check(const G1Affine& p) {
  if (!fp_is_canonical(p.x)) return kPointXNotCanonical;
  if (!fp_is_canonical(p.y)) return kPointYNotCanonical;
  return affine_on_curve(p) ? kPointValid : kPointOffCurve;
}

// BN254 G2 affine over Fq2 = Fq[u]/(u^2 + 1): 128 B as stored in a params file (x.c0, x.c1, y.c0, y.c1), identity (0, 0).
// Only the two points of the params trailer (g2, s_g2) are ever checked, on the host.
struct alignas(16) Fq2 { Fq c0, c1; };
struct alignas(16) G2Affine { Fq2 x, y; };

SPB_HD Fq2 fq2_mul(const Fq2& a, const Fq2& b) {
  Fq2 r;
  r.c0 = fp_mul_sub_mul(a.c0, b.c0, a.c1, b.c1);  // u^2 = -1
  r.c1 = fp_add(fp_mul(a.c0, b.c1), fp_mul(a.c1, b.c0));
  return r;
}

// canonical coordinates and on the twist y^2 = x^3 + b', b' = 3 / (9 + u), or the identity
SPB_HD int g2_affine_check(const G2Affine& p) {
  if (!fp_is_canonical(p.x.c0) || !fp_is_canonical(p.x.c1)) return kPointXNotCanonical;
  if (!fp_is_canonical(p.y.c0) || !fp_is_canonical(p.y.c1)) return kPointYNotCanonical;
  if (fp_is_zero(p.x.c0) && fp_is_zero(p.x.c1) && fp_is_zero(p.y.c0) && fp_is_zero(p.y.c1)) return kPointValid;
  Fq2 b;
  { constexpr uint32_t v0[8] = SPB_FQ2_TWIST_B_C0_MONT, v1[8] = SPB_FQ2_TWIST_B_C1_MONT; for (int i = 0; i < 8; i++) { b.c0.l[i] = v0[i]; b.c1.l[i] = v1[i]; } }
  Fq2 lhs = fq2_mul(p.y, p.y);
  Fq2 rhs = fq2_mul(fq2_mul(p.x, p.x), p.x);
  rhs.c0 = fp_add(rhs.c0, b.c0);
  rhs.c1 = fp_add(rhs.c1, b.c1);
  return fp_eq(lhs.c0, rhs.c0) && fp_eq(lhs.c1, rhs.c1) ? kPointValid : kPointOffCurve;
}

}  // namespace spb
