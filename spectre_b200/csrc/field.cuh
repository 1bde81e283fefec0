// BN254 prime-field arithmetic (Fr scalar field, Fq base field), Montgomery form, R = 2^256.
//
// Replaces halo2curves::bn256::{Fr,Fq} ([UPSTREAM] halo2curves src/bn256/{fr,fq}.rs, reached from the
// reference at lightclient-circuits/src/util/circuit.rs:12). In-memory value of an element is the same
// 32 bytes halo2curves keeps in `Fr(pub(crate) [u64; 4])`: little-endian limbs of a*R mod m. All
// functions take and return fully reduced values in [0, m).
//
// Two code paths, one contract:
//   * device (and -DSPB_EMULATE_PTX host test builds): 8 x u32 limbs, even/odd interleaved CIOS
//     Montgomery product built from fused IMAD.WIDE carry chains (see mont_mul below for the derivation);
//   * host: 4 x u64 limbs with unsigned __int128 (used by the library's host-side glue only: the final
//     window Horner of an MSM, domain constants, affine normalisation).
#pragma once
#include "ptx.cuh"
#include "bn254_constants.h"

namespace spb {

struct alignas(16) Fp256 {
  uint32_t l[8];
};

#define SPB_PARAM_FN(name, init)                                   \
  SPB_HD static constexpr uint32_t name(int i) {                     \
    constexpr uint32_t v[8] = init;                                  \
    return v[i];                                                     \
  }
// Constants are exposed as constexpr functions (not static arrays) so device code can use them as
// immediates without a __constant__ copy.
struct FrParams {
  SPB_PARAM_FN(mod, SPB_FR_MOD)
  SPB_PARAM_FN(r, SPB_FR_R)
  SPB_PARAM_FN(r2, SPB_FR_R2)
  static constexpr uint32_t INV32 = SPB_FR_INV32;
  static constexpr uint64_t INV64 = SPB_FR_INV64;
};
struct FqParams {
  SPB_PARAM_FN(mod, SPB_FQ_MOD)
  SPB_PARAM_FN(r, SPB_FQ_R)
  SPB_PARAM_FN(r2, SPB_FQ_R2)
  static constexpr uint32_t INV32 = SPB_FQ_INV32;
  static constexpr uint64_t INV64 = SPB_FQ_INV64;
};

template <class P>
struct Fp : Fp256 {
  typedef P params;
};
typedef Fp<FrParams> Fr;
typedef Fp<FqParams> Fq;

template <class P> SPB_HD Fp<P> fp_zero() { Fp<P> r; for (int i = 0; i < 8; i++) r.l[i] = 0; return r; }
template <class P> SPB_HD Fp<P> fp_one() { Fp<P> r; for (int i = 0; i < 8; i++) r.l[i] = P::r(i); return r; }
template <class P> SPB_HD bool fp_is_zero(const Fp<P>& a) {
  uint32_t t = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) t |= a.l[i];
  return t == 0;
}
template <class P> SPB_HD bool fp_eq(const Fp<P>& a, const Fp<P>& b) {
  uint32_t t = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) t |= a.l[i] ^ b.l[i];
  return t == 0;
}
// Are the raw limbs less than the modulus? Every other function here assumes they are, so a value read from outside the
// library (a params file) is tested with this before any arithmetic touches it. Compared from the top limb down.
template <class P> SPB_HD bool fp_is_canonical(const Fp<P>& a) {
  uint32_t lt = 0, eq = 1;
#pragma unroll
  for (int i = 7; i >= 0; i--) {
    lt |= eq & (a.l[i] < P::mod(i) ? 1u : 0u);
    eq &= a.l[i] == P::mod(i) ? 1u : 0u;
  }
  return lt != 0;
}

#if defined(SPB_LIMB32_PATH)
// ------------------------------------------------------------------------------------------------
// 32-bit limb path (device).
// ------------------------------------------------------------------------------------------------

// r = a - m if a >= m else a      (a < 2m)
template <class P> SPB_D void fp_final_sub(uint32_t* a) {
  uint32_t t[8];
  t[0] = ptx::sub_cc(a[0], P::mod(0));
#pragma unroll
  for (int i = 1; i < 8; i++) t[i] = ptx::subc_cc(a[i], P::mod(i));
  uint32_t borrow = ptx::subc(0, 0);  // 0xffffffff when a < m
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = borrow ? a[i] : t[i];
}

template <class P> SPB_D Fp<P> fp_add(const Fp<P>& a, const Fp<P>& b) {
  Fp<P> r;
  r.l[0] = ptx::add_cc(a.l[0], b.l[0]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.l[i] = ptx::addc_cc(a.l[i], b.l[i]);
  r.l[7] = ptx::addc(a.l[7], b.l[7]);  // both < 2^254: no carry out
  fp_final_sub<P>(r.l);
  return r;
}

template <class P> SPB_D Fp<P> fp_sub(const Fp<P>& a, const Fp<P>& b) {
  Fp<P> r;
  r.l[0] = ptx::sub_cc(a.l[0], b.l[0]);
#pragma unroll
  for (int i = 1; i < 8; i++) r.l[i] = ptx::subc_cc(a.l[i], b.l[i]);
  uint32_t borrow = ptx::subc(0, 0);  // all-ones when a < b
  r.l[0] = ptx::add_cc(r.l[0], P::mod(0) & borrow);
#pragma unroll
  for (int i = 1; i < 7; i++) r.l[i] = ptx::addc_cc(r.l[i], P::mod(i) & borrow);
  r.l[7] = ptx::addc(r.l[7], P::mod(7) & borrow);
  return r;
}

template <class P> SPB_D Fp<P> fp_neg(const Fp<P>& a) {
  Fp<P> r;
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) nz |= a.l[i];
  uint32_t mask = nz ? 0xffffffffu : 0u;
  r.l[0] = ptx::sub_cc(P::mod(0) & mask, a.l[0]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.l[i] = ptx::subc_cc(P::mod(i) & mask, a.l[i]);
  r.l[7] = ptx::subc(P::mod(7) & mask, a.l[7]);
  return r;
}

// Montgomery product a*b*2^-256 mod m, inputs < m, output < m.
//
// Accumulator T is kept as two 8-limb arrays: X aligned at limb 0 and Y aligned at limb 1
// (T = X + 2^32 * Y). For a fixed multiplier limb b_i the products a_j*b_i with j even tile X without
// overlap and those with j odd tile Y without overlap, so each array takes one unbroken
// mad.lo.cc/madc.hi.cc chain (4 fused IMAD.WIDE). After adding m_i*MOD the low limb X[0] is zero and
// T/2^32 = Y + (X >> 32): Y becomes the new limb-0 array as it stands, X shifted down by two limbs
// becomes the new limb-1 array, and the one limb that falls between them (X[1]) is added into the new
// X[0] with its carry feeding straight into the next odd chain. Bounds: T < a + m < 2^255 at every
// iteration boundary, the running total < 2^288 inside one, so the limb-1 array (top limb = bit 256..287)
// never carries out; carries out of the limb-0 array land on Y[7].
template <class P> SPB_D Fp<P> fp_mul(const Fp<P>& A, const Fp<P>& B) {
  const uint32_t* a = A.l;
  const uint32_t* b = B.l;
  uint32_t ev[8], od[8];
  // i = 0: plain products
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    ptx::mul_wide(ev[j], ev[j + 1], a[j], b[0]);
    ptx::mul_wide(od[j], od[j + 1], a[j + 1], b[0]);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint32_t* X = (i & 1) ? od : ev;
    uint32_t* Y = (i & 1) ? ev : od;
    if (i > 0) {
      uint32_t bi = b[i];
      X[0] = ptx::add_cc(X[0], Y[1]);
      // Y <- (Y >> 64) + a_odd * bi + carry
      ptx::madc_wide_cc(Y[0], Y[1], a[1], bi, Y[2], Y[3]);
      ptx::madc_wide_cc(Y[2], Y[3], a[3], bi, Y[4], Y[5]);
      ptx::madc_wide_cc(Y[4], Y[5], a[5], bi, Y[6], Y[7]);
      ptx::madc_wide(Y[6], Y[7], a[7], bi, 0u, 0u);
      // X += a_even * bi
      ptx::mad_wide_cc(X[0], X[1], a[0], bi, X[0], X[1]);
      ptx::madc_wide_cc(X[2], X[3], a[2], bi, X[2], X[3]);
      ptx::madc_wide_cc(X[4], X[5], a[4], bi, X[4], X[5]);
      ptx::madc_wide_cc(X[6], X[7], a[6], bi, X[6], X[7]);
      Y[7] = ptx::addc(Y[7], 0u);
    }
    uint32_t m = ptx::mul_lo(X[0], P::INV32);
    ptx::mad_wide_cc(Y[0], Y[1], P::mod(1), m, Y[0], Y[1]);
    ptx::madc_wide_cc(Y[2], Y[3], P::mod(3), m, Y[2], Y[3]);
    ptx::madc_wide_cc(Y[4], Y[5], P::mod(5), m, Y[4], Y[5]);
    ptx::madc_wide(Y[6], Y[7], P::mod(7), m, Y[6], Y[7]);
    ptx::mad_wide_cc(X[0], X[1], P::mod(0), m, X[0], X[1]);
    ptx::madc_wide_cc(X[2], X[3], P::mod(2), m, X[2], X[3]);
    ptx::madc_wide_cc(X[4], X[5], P::mod(4), m, X[4], X[5]);
    ptx::madc_wide_cc(X[6], X[7], P::mod(6), m, X[6], X[7]);
    Y[7] = ptx::addc(Y[7], 0u);
  }
  // after i = 7: X = od (X[0] == 0), Y = ev; result = (X >> 32) + Y
  Fp<P> r;
  r.l[0] = ptx::add_cc(od[1], ev[0]);
#pragma unroll
  for (int k = 1; k < 7; k++) r.l[k] = ptx::addc_cc(od[k + 1], ev[k]);
  r.l[7] = ptx::addc(ev[7], 0u);
  fp_final_sub<P>(r.l);
  return r;
}


// ---- separate product and reduction: squaring, and a*b - c*d under one reduction -------------------------------------
// The wide multiply-add (IMAD.WIDE = a fused mad.lo.cc / madc.hi.cc pair) does NOT overlap with the integer adds around it -- their issue times add (an IADD3 costs
// a sizeable fraction of an IMAD.WIDE). So the multiplier above (128 wide + ~60 other) is already at the optimum for a general
// product: a Karatsuba split (48 + 64 wide, ~90 more adds) trades wide multiplies for more adds than it saves. What does pay is removing wide
// multiplies outright:
//   * squaring: 28 cross products + 8 squares + 64 reduction rows = 100 wide instead of 128;
//   * a*b - c*d (the y-coordinate of every XYZZ addition / doubling): two 64-wide products, ONE 64-wide reduction.
// The 16-limb products are accumulated in the same even/odd split as above: array e holds the 64-bit column sums that
// start at even limbs (e[k] = limb k), array o those that start at odd limbs (o[k] = limb k + 1), so every row of partial
// products is an unbroken mad.lo.cc / madc.hi.cc chain on aligned register pairs.
namespace detail {
// the register pair that starts at limb p: in e when p is even, in o when p is odd
#define SPB_LO(p) (((p) & 1) ? o[(p) - 1] : e[(p)])
#define SPB_HI(p) (((p) & 1) ? o[(p)] : e[(p) + 1])
#define SPB_MAD_CC(p, x, y) ptx::mad_wide_cc(SPB_LO(p), SPB_HI(p), x, y, SPB_LO(p), SPB_HI(p))
#define SPB_MADC_CC(p, x, y) ptx::madc_wide_cc(SPB_LO(p), SPB_HI(p), x, y, SPB_LO(p), SPB_HI(p))
#define SPB_MADC_TOP(p, x, y) ptx::madc_wide(SPB_LO(p), SPB_HI(p), x, y, SPB_LO(p), 0u) /* low limb = a carry bit, high limb fresh */
// t[0..15] = e + (o << 32); o[14] = limb 15 is the last one
SPB_D void merge_eo(uint32_t* t, const uint32_t* e, const uint32_t* o) {
  t[0] = e[0];
  t[1] = ptx::add_cc(e[1], o[0]);
#pragma unroll
  for (int k = 2; k < 15; k++) t[k] = ptx::addc_cc(e[k], o[k - 1]);
  t[15] = ptx::addc(e[15], o[14]);
}
// t[0..15] = a[0..7] * b[0..7] (schoolbook, 64 wide multiplies). Row i adds a_j * b_i at limb i + j: the chain over even j
// ends on a pair the previous row initialised and carries out into a fresh limb; the chain over odd j ends on the fresh
// pair above it, whose low limb holds exactly that carry bit of the previous row.
SPB_D void mul8x8(uint32_t* t, const uint32_t* a, const uint32_t* b) {
  uint32_t e[16], o[15];
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    ptx::mul_wide(e[j], e[j + 1], a[j], b[0]);
    ptx::mul_wide(o[j], o[j + 1], a[j + 1], b[0]);
  }
  e[8] = 0u;  // row 0 carries nothing into limb 8
#pragma unroll
  for (int i = 1; i < 8; i++) {
    const uint32_t bi = b[i];
    SPB_MAD_CC(i, a[0], bi);
    SPB_MADC_CC(i + 2, a[2], bi);
    SPB_MADC_CC(i + 4, a[4], bi);
    SPB_MADC_CC(i + 6, a[6], bi);
    SPB_LO(i + 8) = ptx::addc(0u, 0u);
    SPB_MAD_CC(i + 1, a[1], bi);
    SPB_MADC_CC(i + 3, a[3], bi);
    SPB_MADC_CC(i + 5, a[5], bi);
    SPB_MADC_TOP(i + 7, a[7], bi);
  }
  // after row 7: e[15] = limb 15 from the top pair, o[14] = limb 15 carry bit of the even-j chain
  merge_eo(t, e, o);
}
// t[0..15] = a[0..7]^2: the 28 cross products a_i a_j (i < j) once, doubled by a one-bit funnel shift, then the eight
// squares added by wide multiply-adds whose addend is the doubled cross sum (36 wide multiplies).
SPB_D void sqr8(uint32_t* t, const uint32_t* a) {
  uint32_t e[16], o[15];
  e[0] = 0u; e[1] = 0u; e[14] = 0u; e[15] = 0u; o[14] = 0u;
  // row 0: limbs 1..7, all fresh
  ptx::mul_wide(SPB_LO(1), SPB_HI(1), a[0], a[1]);
  ptx::mul_wide(SPB_LO(2), SPB_HI(2), a[0], a[2]);
  ptx::mul_wide(SPB_LO(3), SPB_HI(3), a[0], a[3]);
  ptx::mul_wide(SPB_LO(4), SPB_HI(4), a[0], a[4]);
  ptx::mul_wide(SPB_LO(5), SPB_HI(5), a[0], a[5]);
  ptx::mul_wide(SPB_LO(6), SPB_HI(6), a[0], a[6]);
  ptx::mul_wide(SPB_LO(7), SPB_HI(7), a[0], a[7]);
  // row 1: a1 a2, a1 a4, a1 a6 -> limbs 3, 5, 7 (carry into limb 9) | a1 a3, a1 a5 -> 4, 6, a1 a7 -> 8 (fresh)
  SPB_MAD_CC(3, a[1], a[2]); SPB_MADC_CC(5, a[1], a[4]); SPB_MADC_CC(7, a[1], a[6]); SPB_LO(9) = ptx::addc(0u, 0u);
  SPB_MAD_CC(4, a[1], a[3]); SPB_MADC_CC(6, a[1], a[5]); ptx::madc_wide(SPB_LO(8), SPB_HI(8), a[1], a[7], 0u, 0u);
  // row 2: a2 a3, a2 a5 -> 5, 7, a2 a7 -> 9 (carry bit, fresh) | a2 a4, a2 a6 -> 6, 8 (carry into limb 10)
  SPB_MAD_CC(5, a[2], a[3]); SPB_MADC_CC(7, a[2], a[5]); SPB_MADC_TOP(9, a[2], a[7]);
  SPB_MAD_CC(6, a[2], a[4]); SPB_MADC_CC(8, a[2], a[6]); SPB_LO(10) = ptx::addc(0u, 0u);
  // row 3: a3 a4, a3 a6 -> 7, 9 (carry into limb 11) | a3 a5 -> 8, a3 a7 -> 10 (carry bit, fresh)
  SPB_MAD_CC(7, a[3], a[4]); SPB_MADC_CC(9, a[3], a[6]); SPB_LO(11) = ptx::addc(0u, 0u);
  SPB_MAD_CC(8, a[3], a[5]); SPB_MADC_TOP(10, a[3], a[7]);
  // row 4: a4 a5 -> 9, a4 a7 -> 11 (carry bit, fresh) | a4 a6 -> 10 (carry into limb 12)
  SPB_MAD_CC(9, a[4], a[5]); SPB_MADC_TOP(11, a[4], a[7]);
  SPB_MAD_CC(10, a[4], a[6]); SPB_LO(12) = ptx::addc(0u, 0u);
  // row 5: a5 a6 -> 11 (carry into limb 13) | a5 a7 -> 12 (carry bit, fresh)
  SPB_MAD_CC(11, a[5], a[6]); SPB_LO(13) = ptx::addc(0u, 0u);
  ptx::mad_wide_cc(SPB_LO(12), SPB_HI(12), a[5], a[7], SPB_LO(12), 0u);
  // row 6: a6 a7 -> 13 (carry bit, fresh)
  ptx::mad_wide_cc(SPB_LO(13), SPB_HI(13), a[6], a[7], SPB_LO(13), 0u);
  uint32_t c[16];
  merge_eo(c, e, o);  // cross sum < 2^511: doubling does not overflow
  uint32_t d[16];
  d[0] = 0u;          // c[0] = 0
#pragma unroll
  for (int k = 1; k < 16; k++) d[k] = ptx::shl1_hi(c[k - 1], c[k]);
  ptx::mad_wide_cc(t[0], t[1], a[0], a[0], d[0], d[1]);
#pragma unroll
  for (int i = 1; i < 7; i++) ptx::madc_wide_cc(t[2 * i], t[2 * i + 1], a[i], a[i], d[2 * i], d[2 * i + 1]);
  ptx::madc_wide(t[14], t[15], a[7], a[7], d[14], d[15]);
}
#undef SPB_LO
#undef SPB_HI
#undef SPB_MAD_CC
#undef SPB_MADC_CC
#undef SPB_MADC_TOP
}  // namespace detail

// t (16 limbs, < m * 2^256) -> t * 2^-256 mod m, fully reduced. Only the low half drives the quotient digits, so the
// eight reduction rows run on the low half alone -- the loop of fp_mul with (a, b_i) replaced by (MOD, m_i) and
// no product rows -- and the high half is added at the end: (t_lo + q m) / 2^256 + t_hi < 2m.
template <class P> SPB_D Fp<P> fp_mont_reduce(const uint32_t* t) {
  uint32_t ev[8], od[8];
#pragma unroll
  for (int k = 0; k < 8; k++) ev[k] = t[k];
  {
    uint32_t m = ptx::mul_lo(ev[0], P::INV32);
    ptx::mul_wide(od[0], od[1], P::mod(1), m);
    ptx::mul_wide(od[2], od[3], P::mod(3), m);
    ptx::mul_wide(od[4], od[5], P::mod(5), m);
    ptx::mul_wide(od[6], od[7], P::mod(7), m);
    ptx::mad_wide_cc(ev[0], ev[1], P::mod(0), m, ev[0], ev[1]);
    ptx::madc_wide_cc(ev[2], ev[3], P::mod(2), m, ev[2], ev[3]);
    ptx::madc_wide_cc(ev[4], ev[5], P::mod(4), m, ev[4], ev[5]);
    ptx::madc_wide_cc(ev[6], ev[7], P::mod(6), m, ev[6], ev[7]);
    od[7] = ptx::addc(od[7], 0u);
  }
#pragma unroll
  for (int i = 1; i < 8; i++) {
    uint32_t* X = (i & 1) ? od : ev;
    uint32_t* Y = (i & 1) ? ev : od;
    X[0] = ptx::add_cc(X[0], Y[1]);
    uint32_t m = ptx::mul_lo(X[0], P::INV32);
    ptx::madc_wide_cc(Y[0], Y[1], P::mod(1), m, Y[2], Y[3]);
    ptx::madc_wide_cc(Y[2], Y[3], P::mod(3), m, Y[4], Y[5]);
    ptx::madc_wide_cc(Y[4], Y[5], P::mod(5), m, Y[6], Y[7]);
    ptx::madc_wide(Y[6], Y[7], P::mod(7), m, 0u, 0u);
    ptx::mad_wide_cc(X[0], X[1], P::mod(0), m, X[0], X[1]);
    ptx::madc_wide_cc(X[2], X[3], P::mod(2), m, X[2], X[3]);
    ptx::madc_wide_cc(X[4], X[5], P::mod(4), m, X[4], X[5]);
    ptx::madc_wide_cc(X[6], X[7], P::mod(6), m, X[6], X[7]);
    Y[7] = ptx::addc(Y[7], 0u);
  }
  Fp<P> r;
  r.l[0] = ptx::add_cc(od[1], ev[0]);
#pragma unroll
  for (int k = 1; k < 7; k++) r.l[k] = ptx::addc_cc(od[k + 1], ev[k]);
  r.l[7] = ptx::addc(ev[7], 0u);
  r.l[0] = ptx::add_cc(r.l[0], t[8]);
#pragma unroll
  for (int k = 1; k < 7; k++) r.l[k] = ptx::addc_cc(r.l[k], t[8 + k]);
  r.l[7] = ptx::addc(r.l[7], t[15]);
  fp_final_sub<P>(r.l);
  return r;
}

#if defined(SPB_FP_NO_SOS)  // A/B builds only: everything through the interleaved multiplier
template <class P> SPB_D Fp<P> fp_sqr(const Fp<P>& A) { return fp_mul(A, A); }
template <class P> SPB_D Fp<P> fp_mul_sub_mul(const Fp<P>& A, const Fp<P>& B, const Fp<P>& C, const Fp<P>& D) { return fp_sub(fp_mul(A, B), fp_mul(C, D)); }
#else
template <class P> SPB_D Fp<P> fp_sqr(const Fp<P>& A) {
  uint32_t t[16];
  detail::sqr8(t, A.l);
  return fp_mont_reduce<P>(t);
}
// a*b - c*d with ONE Montgomery reduction (lazy reduction). Both 16-limb products are < m^2 < m * 2^256; their difference
// is brought back into [0, m * 2^256) by adding m * 2^256 when it is negative, which is all fp_mont_reduce needs.
template <class P> SPB_D Fp<P> fp_mul_sub_mul(const Fp<P>& A, const Fp<P>& B, const Fp<P>& C, const Fp<P>& D) {
  uint32_t t[16], u[16];
  detail::mul8x8(t, A.l, B.l);
  detail::mul8x8(u, C.l, D.l);
  t[0] = ptx::sub_cc(t[0], u[0]);
#pragma unroll
  for (int k = 1; k < 16; k++) t[k] = ptx::subc_cc(t[k], u[k]);
  const uint32_t borrow = ptx::subc(0u, 0u);  // all-ones when a*b < c*d
  t[8] = ptx::add_cc(t[8], P::mod(0) & borrow);
#pragma unroll
  for (int k = 1; k < 7; k++) t[8 + k] = ptx::addc_cc(t[8 + k], P::mod(k) & borrow);
  t[15] = ptx::addc(t[15], P::mod(7) & borrow);
  return fp_mont_reduce<P>(t);
}
#endif

#else
// ------------------------------------------------------------------------------------------------
// 64-bit limb path (host glue).
// ------------------------------------------------------------------------------------------------
namespace detail {
inline void load64(uint64_t* d, const uint32_t* s) { for (int i = 0; i < 4; i++) d[i] = ((uint64_t)s[2 * i + 1] << 32) | s[2 * i]; }
inline void store64(uint32_t* d, const uint64_t* s) { for (int i = 0; i < 4; i++) { d[2 * i] = (uint32_t)s[i]; d[2 * i + 1] = (uint32_t)(s[i] >> 32); } }
template <class P> inline void mod64(uint64_t* m) { uint32_t t[8]; for (int i = 0; i < 8; i++) t[i] = P::mod(i); load64(m, t); }
template <class P> inline void cond_sub(uint64_t* t, uint64_t extra) {
  uint64_t m[4], d[4]; mod64<P>(m);
  unsigned __int128 bw = 0;
  for (int i = 0; i < 4; i++) { unsigned __int128 x = (unsigned __int128)t[i] - m[i] - (uint64_t)bw; d[i] = (uint64_t)x; bw = (x >> 64) & 1; }
  if (extra || !bw) for (int i = 0; i < 4; i++) t[i] = d[i];
}
}  // namespace detail

template <class P> inline Fp<P> fp_add(const Fp<P>& a, const Fp<P>& b) {
  uint64_t x[4], y[4]; detail::load64(x, a.l); detail::load64(y, b.l);
  unsigned __int128 c = 0;
  for (int i = 0; i < 4; i++) { c += (unsigned __int128)x[i] + y[i]; x[i] = (uint64_t)c; c >>= 64; }
  detail::cond_sub<P>(x, (uint64_t)c);
  Fp<P> r; detail::store64(r.l, x); return r;
}
template <class P> inline Fp<P> fp_sub(const Fp<P>& a, const Fp<P>& b) {
  uint64_t x[4], y[4], m[4]; detail::load64(x, a.l); detail::load64(y, b.l); detail::mod64<P>(m);
  unsigned __int128 bw = 0;
  for (int i = 0; i < 4; i++) { unsigned __int128 t = (unsigned __int128)x[i] - y[i] - (uint64_t)bw; x[i] = (uint64_t)t; bw = (t >> 64) & 1; }
  if (bw) { unsigned __int128 c = 0; for (int i = 0; i < 4; i++) { c += (unsigned __int128)x[i] + m[i]; x[i] = (uint64_t)c; c >>= 64; } }
  Fp<P> r; detail::store64(r.l, x); return r;
}
template <class P> inline Fp<P> fp_neg(const Fp<P>& a) { return fp_sub(fp_zero<P>(), a); }
template <class P> inline Fp<P> fp_mul(const Fp<P>& a, const Fp<P>& b) {
  uint64_t x[4], y[4], m[4]; detail::load64(x, a.l); detail::load64(y, b.l); detail::mod64<P>(m);
  uint64_t t[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    unsigned __int128 c = 0;
    for (int j = 0; j < 4; j++) { c += (unsigned __int128)x[j] * y[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
    c += t[4]; t[4] = (uint64_t)c; t[5] = (uint64_t)(c >> 64);
    uint64_t q = t[0] * P::INV64;
    c = (unsigned __int128)q * m[0] + t[0]; c >>= 64;
    for (int j = 1; j < 4; j++) { c += (unsigned __int128)q * m[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
    c += t[4]; t[3] = (uint64_t)c; t[4] = t[5] + (uint64_t)(c >> 64);
  }
  detail::cond_sub<P>(t, t[4]);
  Fp<P> r; detail::store64(r.l, t); return r;
}
#endif

// ------------------------------------------------------------------------------------------------
// Shared on both paths.
// ------------------------------------------------------------------------------------------------
#if !defined(SPB_LIMB32_PATH)
template <class P> inline Fp<P> fp_sqr(const Fp<P>& a) { return fp_mul(a, a); }
template <class P> inline Fp<P> fp_mul_sub_mul(const Fp<P>& a, const Fp<P>& b, const Fp<P>& c, const Fp<P>& d) { return fp_sub(fp_mul(a, b), fp_mul(c, d)); }
#endif
template <class P> SPB_HD Fp<P> fp_dbl(const Fp<P>& a) { return fp_add(a, a); }

// Montgomery -> canonical integer (what halo2curves' to_repr() serialises, little-endian).
template <class P> SPB_HD Fp<P> fp_from_mont(const Fp<P>& a) {
  Fp<P> one; for (int i = 0; i < 8; i++) one.l[i] = (i == 0);
  return fp_mul(a, one);
}
template <class P> SPB_HD Fp<P> fp_to_mont(const Fp<P>& a) {
  Fp<P> r2; for (int i = 0; i < 8; i++) r2.l[i] = P::r2(i);
  return fp_mul(a, r2);
}
// a^e for a 256-bit little-endian exponent (square-and-multiply, MSB first)
template <class P> SPB_HD Fp<P> fp_pow(const Fp<P>& a, const uint32_t* e) {
  Fp<P> r = fp_one<P>();
  for (int i = 255; i >= 0; i--) {
    r = fp_sqr(r);
    if ((e[i >> 5] >> (i & 31)) & 1) r = fp_mul(r, a);
  }
  return r;
}
template <class P> SPB_HD Fp<P> fp_pow_u64(const Fp<P>& a, uint64_t e) {
  if (e == 0) return fp_one<P>();
  int top = 63;
  while (!((e >> top) & 1)) top--;
  Fp<P> r = a;
  for (int i = top - 1; i >= 0; i--) {
    r = fp_sqr(r);
    if ((e >> i) & 1) r = fp_mul(r, a);
  }
  return r;
}
// Fermat inversion; inv(0) = 0 (callers that care test for zero first, as halo2's batch_invert does).
template <class P> SPB_HD Fp<P> fp_inv(const Fp<P>& a) {
  uint32_t e[8];
  for (int i = 0; i < 8; i++) e[i] = P::mod(i);
  e[0] -= 2;  // low limb of both moduli is >= 2
  return fp_pow(a, e);
}

}  // namespace spb
