/*
 * halo2_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C restatement of the CPU algorithms that Spectre's prover executes on the create_proof hot
 * path. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this file's shared object; the product library (spectre_b200/csrc) never links or calls it.
 *
 * The arithmetic lives in third-party crates that are NOT vendored in the reference tree (no Cargo.lock,
 * no vendor dir -- SURVEY.md section 8c): halo2_proofs (PSE fork, pulled through halo2-base's `halo2-pse`
 * feature, reference Cargo.toml:44-48), halo2curves-axiom =0.5.2 (Cargo.toml:52), snark-verifier-sdk
 * v0.1.7-git (Cargo.toml:55-67), rand_chacha. Each function below names the upstream routine it
 * restates ([UPSTREAM] path) and the reference call site that reaches it.
 *
 * PINNING. The oracle is pinned against the only numeric artefacts the reference commits for this path,
 * the generated verifier contracts (tests/test_oracle_golden.py, fixtures tests/golden/verifier_kats.json):
 *   - tau*G2 of the seed-0 "unsafe" SRS  == contracts/snark-verifiers/sync_step_verifier.sol:1203-1206
 *     (pins ChaCha20Rng::from_seed([0;32]), Fr::random = from_u512 of the first 64 keystream bytes,
 *      ParamsKZG::setup drawing tau first);
 *   - commit_lagrange(range table 0..2^19) at K=23 == sync_step_verifier.sol:1048-1049 and
 *     commit_lagrange(range table 0..2^23) at K=24 == committee_update_verifier.sol:1061-1062
 *     (pins g_lagrange derivation, omega_n = ROOT_OF_UNITY^(2^(28-k)), Lagrange indexing, MSM, affine
 *      normalisation).
 * The coset (ZETA) convention is not exercised by those artefacts; it is restated from halo2curves'
 * published constant and cross-checked by direct evaluation (tests/test_oracle_domain.py). Proof BYTES
 * are not pinned by the reference at all (proofs are randomised and no proof file is committed).
 *
 * Build: see oracle/Makefile (gcc -O3 -march=x86-64-v3 -pthread -shared).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <pthread.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t l[4]; } fe;            /* Montgomery residue, little-endian limbs        */
typedef struct { fe x, y; } g1a;                 /* halo2curves G1Affine: identity = (0,0)          */
typedef struct { fe x, y, z; } g1j;              /* halo2curves G1 (Jacobian): identity z = 0       */
typedef struct { fe c0, c1; } fe2;               /* Fq2 = Fq[u]/(u^2+1)                              */
typedef struct { fe2 x, y; } g2a;
typedef struct { fe2 x, y, z; } g2j;

typedef struct {
  uint64_t m[4];     /* modulus */
  uint64_t inv;      /* -m^-1 mod 2^64 */
  fe r, r2;          /* 2^256 mod m, 2^512 mod m */
} field_t;

static field_t FR, FQ;
static fe FR_ROOT_OF_UNITY, FR_ZETA, FR_ZETA2, FQ_THREE;
static g1a G1_GEN;
static g2a G2_GEN;
static int g_inited = 0;

/* ------------------------------------------------------------------------------------------------
 * 256-bit helpers and Montgomery arithmetic: [UPSTREAM] halo2curves src/derive/field.rs
 * (field_arithmetic! macro: 4x64 CIOS-style montgomery_reduce, `asm` feature off -- Cargo.toml:44-52).
 * ---------------------------------------------------------------------------------------------- */
static inline int geq(const uint64_t* a, const uint64_t* b) {
  for (int i = 3; i >= 0; i--) { if (a[i] != b[i]) return a[i] > b[i]; }
  return 1;
}
static inline uint64_t sub_into(uint64_t* a, const uint64_t* b) {
  u128 bw = 0;
  for (int i = 0; i < 4; i++) { u128 t = (u128)a[i] - b[i] - (uint64_t)bw; a[i] = (uint64_t)t; bw = (t >> 64) & 1; }
  return (uint64_t)bw;
}
static inline uint64_t add_into(uint64_t* a, const uint64_t* b) {
  u128 c = 0;
  for (int i = 0; i < 4; i++) { c += (u128)a[i] + b[i]; a[i] = (uint64_t)c; c >>= 64; }
  return (uint64_t)c;
}
static inline fe f_add(const field_t* F, fe a, fe b) {
  uint64_t c = add_into(a.l, b.l);
  if (c || geq(a.l, F->m)) sub_into(a.l, F->m);
  return a;
}
static inline fe f_sub(const field_t* F, fe a, fe b) {
  if (sub_into(a.l, b.l)) add_into(a.l, F->m);
  return a;
}
static inline fe f_neg(const field_t* F, fe a) { fe z = {{0, 0, 0, 0}}; return f_sub(F, z, a); }
static inline fe f_dbl(const field_t* F, fe a) { return f_add(F, a, a); }
static inline int f_is_zero(fe a) { return (a.l[0] | a.l[1] | a.l[2] | a.l[3]) == 0; }
static inline int f_eq(fe a, fe b) { return a.l[0] == b.l[0] && a.l[1] == b.l[1] && a.l[2] == b.l[2] && a.l[3] == b.l[3]; }

static inline fe f_mul(const field_t* F, fe a, fe b) {
  /* schoolbook 4x4 product then word-by-word Montgomery reduction, as halo2curves' mul + montgomery_reduce */
  uint64_t t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)a.l[j] * b.l[i] + t[i + j]; t[i + j] = (uint64_t)c; c >>= 64; }
    t[i + 4] = (uint64_t)c;
  }
  uint64_t carry2 = 0;
  for (int i = 0; i < 4; i++) {
    uint64_t k = t[i] * F->inv;
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)k * F->m[j] + t[i + j]; t[i + j] = (uint64_t)c; c >>= 64; }
    u128 s = (u128)t[i + 4] + (uint64_t)c + carry2;
    t[i + 4] = (uint64_t)s; carry2 = (uint64_t)(s >> 64);
  }
  fe r = {{t[4], t[5], t[6], t[7]}};
  if (carry2 || geq(r.l, F->m)) sub_into(r.l, F->m);
  return r;
}
static inline fe f_sqr(const field_t* F, fe a) { return f_mul(F, a, a); }
static fe f_pow(const field_t* F, fe a, const uint64_t e[4]) {
  fe r = F->r;
  for (int i = 255; i >= 0; i--) {
    r = f_sqr(F, r);
    if ((e[i >> 6] >> (i & 63)) & 1) r = f_mul(F, r, a);
  }
  return r;
}
static fe f_inv(const field_t* F, fe a) {  /* Fermat: a^(m-2); invert(0) -> 0 */
  uint64_t e[4] = {F->m[0] - 2, F->m[1], F->m[2], F->m[3]};
  return f_pow(F, a, e);
}
static fe f_from_u64(const field_t* F, uint64_t v) { fe a = {{v, 0, 0, 0}}; return f_mul(F, a, F->r2); }
static fe f_from_raw(const field_t* F, const uint64_t v[4]) { fe a = {{v[0], v[1], v[2], v[3]}}; return f_mul(F, a, F->r2); }
static fe f_to_canonical(const field_t* F, fe a) { fe one = {{1, 0, 0, 0}}; return f_mul(F, a, one); }

static void field_setup(field_t* F, const uint64_t m[4]) {
  memcpy(F->m, m, 32);
  /* inv = -m^-1 mod 2^64 by Newton iteration */
  uint64_t x = 1;
  for (int i = 0; i < 7; i++) x *= 2 - m[0] * x;
  F->inv = (uint64_t)0 - x;
  /* r = 2^256 mod m by 256 modular doublings of 1; r2 by 256 more */
  uint64_t v[4] = {1, 0, 0, 0};
  for (int i = 0; i < 512; i++) {
    uint64_t c = add_into(v, v);
    if (c || geq(v, m)) sub_into(v, m);
    if (i == 255) memcpy(F->r.l, v, 32);
  }
  memcpy(F->r2.l, v, 32);
}

/* ------------------------------------------------------------------------------------------------
 * G1: [UPSTREAM] halo2curves src/derive/curve.rs (new_curve_impl!: Jacobian add / mixed add / double
 * for a = 0 curves), src/bn256/curve.rs (generator (1,2), b = 3).
 * ---------------------------------------------------------------------------------------------- */
static inline int g1a_is_identity(const g1a* p) { return f_is_zero(p->x) && f_is_zero(p->y); }
static inline int g1j_is_identity(const g1j* p) { return f_is_zero(p->z); }
static g1j g1j_identity(void) { g1j r; memset(&r, 0, sizeof r); r.y = FQ.r; return r; }
static g1j g1j_from_affine(const g1a* p) {
  if (g1a_is_identity(p)) return g1j_identity();
  g1j r; r.x = p->x; r.y = p->y; r.z = FQ.r; return r;
}
static g1j g1j_double(const g1j* p) {
  if (g1j_is_identity(p)) return *p;
  /* dbl-2009-l */
  fe a = f_sqr(&FQ, p->x), b = f_sqr(&FQ, p->y), c = f_sqr(&FQ, b);
  fe d = f_sub(&FQ, f_sub(&FQ, f_sqr(&FQ, f_add(&FQ, p->x, b)), a), c); d = f_dbl(&FQ, d);
  fe e = f_add(&FQ, f_dbl(&FQ, a), a), f = f_sqr(&FQ, e);
  g1j r;
  r.z = f_dbl(&FQ, f_mul(&FQ, p->z, p->y));
  r.x = f_sub(&FQ, f, f_dbl(&FQ, d));
  fe c8 = f_dbl(&FQ, f_dbl(&FQ, f_dbl(&FQ, c)));
  r.y = f_sub(&FQ, f_mul(&FQ, e, f_sub(&FQ, d, r.x)), c8);
  return r;
}
static g1j g1j_add(const g1j* p, const g1j* q) {
  if (g1j_is_identity(p)) return *q;
  if (g1j_is_identity(q)) return *p;
  fe z1z1 = f_sqr(&FQ, p->z), z2z2 = f_sqr(&FQ, q->z);
  fe u1 = f_mul(&FQ, p->x, z2z2), u2 = f_mul(&FQ, q->x, z1z1);
  fe s1 = f_mul(&FQ, f_mul(&FQ, p->y, z2z2), q->z), s2 = f_mul(&FQ, f_mul(&FQ, q->y, z1z1), p->z);
  if (f_eq(u1, u2)) { if (f_eq(s1, s2)) return g1j_double(p); return g1j_identity(); }
  fe h = f_sub(&FQ, u2, u1), i = f_sqr(&FQ, f_dbl(&FQ, h)), j = f_mul(&FQ, h, i);
  fe rr = f_dbl(&FQ, f_sub(&FQ, s2, s1)), v = f_mul(&FQ, u1, i);
  g1j r;
  r.x = f_sub(&FQ, f_sub(&FQ, f_sqr(&FQ, rr), j), f_dbl(&FQ, v));
  r.y = f_sub(&FQ, f_mul(&FQ, rr, f_sub(&FQ, v, r.x)), f_dbl(&FQ, f_mul(&FQ, s1, j)));
  r.z = f_mul(&FQ, f_sub(&FQ, f_sub(&FQ, f_sqr(&FQ, f_add(&FQ, p->z, q->z)), z1z1), z2z2), h);
  return r;
}
static g1j g1j_add_mixed(const g1j* p, const g1a* q) {
  if (g1a_is_identity(q)) return *p;
  if (g1j_is_identity(p)) return g1j_from_affine(q);
  fe z1z1 = f_sqr(&FQ, p->z), u2 = f_mul(&FQ, q->x, z1z1), s2 = f_mul(&FQ, f_mul(&FQ, q->y, z1z1), p->z);
  if (f_eq(p->x, u2)) { if (f_eq(p->y, s2)) return g1j_double(p); return g1j_identity(); }
  fe h = f_sub(&FQ, u2, p->x), hh = f_sqr(&FQ, h), i = f_dbl(&FQ, f_dbl(&FQ, hh)), j = f_mul(&FQ, h, i);
  fe rr = f_dbl(&FQ, f_sub(&FQ, s2, p->y)), v = f_mul(&FQ, p->x, i);
  g1j r;
  r.x = f_sub(&FQ, f_sub(&FQ, f_sqr(&FQ, rr), j), f_dbl(&FQ, v));
  r.y = f_sub(&FQ, f_mul(&FQ, rr, f_sub(&FQ, v, r.x)), f_dbl(&FQ, f_mul(&FQ, p->y, j)));
  r.z = f_sub(&FQ, f_sub(&FQ, f_sqr(&FQ, f_add(&FQ, p->z, h)), z1z1), hh);
  return r;
}
static g1a g1j_to_affine(const g1j* p) {
  g1a r; memset(&r, 0, sizeof r);
  if (g1j_is_identity(p)) return r;
  fe zi = f_inv(&FQ, p->z), zi2 = f_sqr(&FQ, zi);
  r.x = f_mul(&FQ, p->x, zi2); r.y = f_mul(&FQ, p->y, f_mul(&FQ, zi2, zi));
  return r;
}
/* [UPSTREAM] halo2curves CurveExt::batch_normalize: Montgomery's trick */
static void g1_batch_normalize(const g1j* p, g1a* out, size_t n) {
  fe* acc = (fe*)malloc(n * sizeof(fe));
  fe run = FQ.r;
  for (size_t i = 0; i < n; i++) { acc[i] = run; if (!g1j_is_identity(&p[i])) run = f_mul(&FQ, run, p[i].z); }
  run = f_inv(&FQ, run);
  for (size_t i = n; i-- > 0;) {
    if (g1j_is_identity(&p[i])) { memset(&out[i], 0, sizeof(g1a)); continue; }
    fe zi = f_mul(&FQ, run, acc[i]);
    run = f_mul(&FQ, run, p[i].z);
    fe zi2 = f_sqr(&FQ, zi);
    out[i].x = f_mul(&FQ, p[i].x, zi2); out[i].y = f_mul(&FQ, p[i].y, f_mul(&FQ, zi2, zi));
  }
  free(acc);
}
static g1j g1_mul_canonical(const g1a* base, const uint64_t e[4]) {  /* double-and-add, MSB first */
  g1j r = g1j_identity();
  for (int i = 255; i >= 0; i--) {
    r = g1j_double(&r);
    if ((e[i >> 6] >> (i & 63)) & 1) r = g1j_add_mixed(&r, base);
  }
  return r;
}

/* ------------------------------------------------------------------------------------------------
 * Fq2 / G2 -- only to reproduce s_g2 = tau*G2 for the SRS known-answer test.
 * [UPSTREAM] halo2curves src/bn256/fq2.rs (u^2 = -1), src/bn256/curve.rs (G2 generator).
 * ---------------------------------------------------------------------------------------------- */
static fe2 f2_add(fe2 a, fe2 b) { fe2 r = {f_add(&FQ, a.c0, b.c0), f_add(&FQ, a.c1, b.c1)}; return r; }
static fe2 f2_sub(fe2 a, fe2 b) { fe2 r = {f_sub(&FQ, a.c0, b.c0), f_sub(&FQ, a.c1, b.c1)}; return r; }
static fe2 f2_dbl(fe2 a) { return f2_add(a, a); }
static fe2 f2_mul(fe2 a, fe2 b) {
  fe t0 = f_mul(&FQ, a.c0, b.c0), t1 = f_mul(&FQ, a.c1, b.c1);
  fe2 r;
  r.c0 = f_sub(&FQ, t0, t1);
  r.c1 = f_sub(&FQ, f_sub(&FQ, f_mul(&FQ, f_add(&FQ, a.c0, a.c1), f_add(&FQ, b.c0, b.c1)), t0), t1);
  return r;
}
static fe2 f2_sqr(fe2 a) { return f2_mul(a, a); }
static int f2_is_zero(fe2 a) { return f_is_zero(a.c0) && f_is_zero(a.c1); }
static int f2_eq(fe2 a, fe2 b) { return f_eq(a.c0, b.c0) && f_eq(a.c1, b.c1); }
static fe2 f2_inv(fe2 a) {
  fe n = f_add(&FQ, f_sqr(&FQ, a.c0), f_sqr(&FQ, a.c1)), ni = f_inv(&FQ, n);
  fe2 r = {f_mul(&FQ, a.c0, ni), f_neg(&FQ, f_mul(&FQ, a.c1, ni))};
  return r;
}
static g2j g2j_double(const g2j* p) {
  if (f2_is_zero(p->z)) return *p;
  fe2 a = f2_sqr(p->x), b = f2_sqr(p->y), c = f2_sqr(b);
  fe2 d = f2_dbl(f2_sub(f2_sub(f2_sqr(f2_add(p->x, b)), a), c));
  fe2 e = f2_add(f2_dbl(a), a), f = f2_sqr(e);
  g2j r;
  r.z = f2_dbl(f2_mul(p->z, p->y));
  r.x = f2_sub(f, f2_dbl(d));
  r.y = f2_sub(f2_mul(e, f2_sub(d, r.x)), f2_dbl(f2_dbl(f2_dbl(c))));
  return r;
}
static g2j g2j_add_mixed(const g2j* p, const g2a* q) {
  if (f2_is_zero(p->z)) { g2j r; r.x = q->x; r.y = q->y; memset(&r.z, 0, sizeof r.z); r.z.c0 = FQ.r; return r; }
  fe2 z1z1 = f2_sqr(p->z), u2 = f2_mul(q->x, z1z1), s2 = f2_mul(f2_mul(q->y, z1z1), p->z);
  if (f2_eq(p->x, u2)) { if (f2_eq(p->y, s2)) return g2j_double(p); g2j r; memset(&r, 0, sizeof r); r.y.c0 = FQ.r; return r; }
  fe2 h = f2_sub(u2, p->x), hh = f2_sqr(h), i = f2_dbl(f2_dbl(hh)), j = f2_mul(h, i);
  fe2 rr = f2_dbl(f2_sub(s2, p->y)), v = f2_mul(p->x, i);
  g2j r;
  r.x = f2_sub(f2_sub(f2_sqr(rr), j), f2_dbl(v));
  r.y = f2_sub(f2_mul(rr, f2_sub(v, r.x)), f2_dbl(f2_mul(p->y, j)));
  r.z = f2_sub(f2_sub(f2_sqr(f2_add(p->z, h)), z1z1), hh);
  return r;
}

/* ------------------------------------------------------------------------------------------------
 * One-time constants.
 * ---------------------------------------------------------------------------------------------- */
static const uint64_t R_MOD[4] = {0x43e1f593f0000001ull, 0x2833e84879b97091ull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
static const uint64_t P_MOD[4] = {0x3c208c16d87cfd47ull, 0x97816a916871ca8dull, 0xb85045b68181585dull, 0x30644e72e131a029ull};

static void shr_u256(uint64_t* v, int k) { for (int s = 0; s < k; s++) { for (int i = 0; i < 4; i++) v[i] = (v[i] >> 1) | (i < 3 ? v[i + 1] << 63 : 0); } }

void orc_init(void) {
  if (g_inited) return;
  field_setup(&FR, R_MOD);
  field_setup(&FQ, P_MOD);
  /* [UPSTREAM] halo2curves src/bn256/fr.rs: MULTIPLICATIVE_GENERATOR = 7, S = 28,
   * ROOT_OF_UNITY = 7^((r-1)/2^28), ZETA = a primitive cube root of unity (the square of 7^((r-1)/3)). */
  uint64_t e[4]; memcpy(e, R_MOD, 32); e[0] -= 1; shr_u256(e, 28);
  fe seven = f_from_u64(&FR, 7);
  FR_ROOT_OF_UNITY = f_pow(&FR, seven, e);
  /* (r-1)/3: r-1 is divisible by 3; divide limb-wise */
  uint64_t q[4]; memcpy(q, R_MOD, 32); q[0] -= 1;
  { u128 rem = 0; for (int i = 3; i >= 0; i--) { u128 cur = (rem << 64) | q[i]; q[i] = (uint64_t)(cur / 3); rem = cur % 3; } }
  fe z = f_pow(&FR, seven, q);
  FR_ZETA = f_sqr(&FR, z);
  FR_ZETA2 = f_sqr(&FR, FR_ZETA);
  FQ_THREE = f_from_u64(&FQ, 3);
  G1_GEN.x = f_from_u64(&FQ, 1); G1_GEN.y = f_from_u64(&FQ, 2);
  /* G2 generator, [UPSTREAM] halo2curves src/bn256/curve.rs G2_GENERATOR_{X,Y}; the same four words are
   * committed by the reference at contracts/snark-verifiers/sync_step_verifier.sol:1197-1200 (as x.c1,x.c0,y.c1,y.c0). */
  static const uint64_t g2x0[4] = {0x46debd5cd992f6edull, 0x674322d4f75edaddull, 0x426a00665e5c4479ull, 0x1800deef121f1e76ull};
  static const uint64_t g2x1[4] = {0x97e485b7aef312c2ull, 0xf1aa493335a9e712ull, 0x7260bfb731fb5d25ull, 0x198e9393920d483aull};
  static const uint64_t g2y0[4] = {0x4ce6cc0166fa7daaull, 0xe3d1e7690c43d37bull, 0x4aab71808dcb408full, 0x12c85ea5db8c6debull};
  static const uint64_t g2y1[4] = {0x55acdadcd122975bull, 0xbc4b313370b38ef3ull, 0xec9e99ad690c3395ull, 0x090689d0585ff075ull};
  G2_GEN.x.c0 = f_from_raw(&FQ, g2x0); G2_GEN.x.c1 = f_from_raw(&FQ, g2x1);
  G2_GEN.y.c0 = f_from_raw(&FQ, g2y0); G2_GEN.y.c1 = f_from_raw(&FQ, g2y1);
  g_inited = 1;
}

/* ------------------------------------------------------------------------------------------------
 * Elementwise exports for the tests.
 * ---------------------------------------------------------------------------------------------- */
void orc_fr_mul(fe* o, const fe* a, const fe* b) { *o = f_mul(&FR, *a, *b); }
void orc_fr_add(fe* o, const fe* a, const fe* b) { *o = f_add(&FR, *a, *b); }
void orc_fr_sub(fe* o, const fe* a, const fe* b) { *o = f_sub(&FR, *a, *b); }
void orc_fr_inv(fe* o, const fe* a) { *o = f_inv(&FR, *a); }
void orc_fq_mul(fe* o, const fe* a, const fe* b) { *o = f_mul(&FQ, *a, *b); }
void orc_fq_add(fe* o, const fe* a, const fe* b) { *o = f_add(&FQ, *a, *b); }
void orc_fq_sub(fe* o, const fe* a, const fe* b) { *o = f_sub(&FQ, *a, *b); }
void orc_fq_inv(fe* o, const fe* a) { *o = f_inv(&FQ, *a); }
/* to_repr(): canonical little-endian bytes. from_repr: canonical -> Montgomery (caller guarantees < m). */
void orc_fr_to_repr(uint8_t out[32], const fe* a) { fe c = f_to_canonical(&FR, *a); memcpy(out, c.l, 32); }
void orc_fr_from_repr(fe* o, const uint8_t in[32]) { uint64_t v[4]; memcpy(v, in, 32); *o = f_from_raw(&FR, v); }
void orc_fq_to_repr(uint8_t out[32], const fe* a) { fe c = f_to_canonical(&FQ, *a); memcpy(out, c.l, 32); }
void orc_fq_from_repr(fe* o, const uint8_t in[32]) { uint64_t v[4]; memcpy(v, in, 32); *o = f_from_raw(&FQ, v); }
void orc_fr_constants(fe* root_of_unity, fe* zeta, fe* one) { *root_of_unity = FR_ROOT_OF_UNITY; *zeta = FR_ZETA; *one = FR.r; }

/* [UPSTREAM] halo2curves field_common!/from_u512: (lo + hi*2^256) mod r with lo, hi the little-endian
 * 256-bit halves = lo*R2*R^-1 + hi*R3*R^-1 in Montgomery arithmetic. Fr::random(rng) feeds it eight
 * consecutive next_u64() draws. */
void orc_fr_from_u512(fe* o, const uint8_t in[64]) {
  uint64_t v[8]; memcpy(v, in, 64);
  fe lo = {{v[0], v[1], v[2], v[3]}}, hi = {{v[4], v[5], v[6], v[7]}};
  fe r3 = f_mul(&FR, FR.r2, FR.r2);
  *o = f_add(&FR, f_mul(&FR, lo, FR.r2), f_mul(&FR, hi, r3));
}

void orc_fr_seq(fe* out, size_t n) { fe v; memset(&v, 0, sizeof v); for (size_t i = 0; i < n; i++) { out[i] = v; v = f_add(&FR, v, FR.r); } }

void orc_g1_add(g1j* o, const g1j* a, const g1j* b) { *o = g1j_add(a, b); }
void orc_g1_add_mixed(g1j* o, const g1j* a, const g1a* b) { *o = g1j_add_mixed(a, b); }
void orc_g1_double(g1j* o, const g1j* a) { *o = g1j_double(a); }
void orc_g1_to_affine(g1a* o, const g1j* a) { *o = g1j_to_affine(a); }
void orc_g1_generator(g1a* o) { *o = G1_GEN; }
/* scalar in Montgomery Fr form, as a halo2 caller would hold it */
void orc_g1_mul(g1j* o, const g1a* base, const fe* scalar) { fe c = f_to_canonical(&FR, *scalar); *o = g1_mul_canonical(base, c.l); }
int orc_g1_on_curve(const g1a* p) {
  if (g1a_is_identity(p)) return 1;
  fe lhs = f_sqr(&FQ, p->y), rhs = f_add(&FQ, f_mul(&FQ, f_sqr(&FQ, p->x), p->x), FQ_THREE);
  return f_eq(lhs, rhs);
}

/* ------------------------------------------------------------------------------------------------
 * Thread helper (stands in for rayon's scope/join in the restated algorithms).
 * ---------------------------------------------------------------------------------------------- */
typedef struct { void (*fn)(void*); void* arg; } task_t;
static void* task_tramp(void* p) { task_t* t = (task_t*)p; t->fn(t->arg); return NULL; }
static void run_tasks(task_t* tasks, int n) {
  if (n == 1) { tasks[0].fn(tasks[0].arg); return; }
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * n);
  for (int i = 1; i < n; i++) pthread_create(&th[i], NULL, task_tramp, &tasks[i]);
  tasks[0].fn(tasks[0].arg);
  for (int i = 1; i < n; i++) pthread_join(th[i], NULL);
  free(th);
}

/* ------------------------------------------------------------------------------------------------
 * best_fft: [UPSTREAM] halo2_proofs/src/arithmetic.rs `best_fft` + `recursive_butterfly_arithmetic`.
 * Reached from the reference through EvaluationDomain inside create_proof/keygen
 * (lightclient-circuits/src/util/circuit.rs:131,158,177,211,263).
 * In-place, natural order in and out, out[i] = sum_j in[j]*omega^(i*j), no 1/n scaling.
 * Shape kept for timing fairness: bit-reversal swap, n/2 twiddles by repeated multiplication, iterative
 * radix-2 when log_n <= floor(log2(threads)), otherwise the recursive split whose two halves are joined
 * in parallel while the combining butterfly loop of each level runs on one thread.
 * ---------------------------------------------------------------------------------------------- */
static inline size_t bitreverse(size_t n, unsigned l) { size_t r = 0; for (unsigned i = 0; i < l; i++) { r = (r << 1) | (n & 1); n >>= 1; } return r; }
static inline void butterfly_pair(fe* a, fe* b, const fe* tw) {
  fe t = tw ? f_mul(&FR, *b, *tw) : *b;
  *b = f_sub(&FR, *a, t);
  *a = f_add(&FR, *a, t);
}
typedef struct { fe* a; size_t n; size_t twiddle_chunk; const fe* tw; int par_depth; } rba_t;
static void rba(void* p) {
  rba_t* s = (rba_t*)p;
  fe* a = s->a; size_t n = s->n;
  if (n == 2) { butterfly_pair(&a[0], &a[1], NULL); return; }
  rba_t l = {a, n / 2, s->twiddle_chunk * 2, s->tw, s->par_depth - 1};
  rba_t r = {a + n / 2, n / 2, s->twiddle_chunk * 2, s->tw, s->par_depth - 1};
  if (s->par_depth > 0) { task_t t[2] = {{rba, &l}, {rba, &r}}; run_tasks(t, 2); }
  else { rba(&l); rba(&r); }
  fe* left = a; fe* right = a + n / 2;
  butterfly_pair(&left[0], &right[0], NULL);                      /* twiddle == 1 special case */
  for (size_t i = 1; i < n / 2; i++) butterfly_pair(&left[i], &right[i], &s->tw[i * s->twiddle_chunk]);
}
void orc_best_fft(fe* a, const fe* omega, uint32_t log_n, int threads) {
  size_t n = (size_t)1 << log_n;
  if (threads < 1) threads = 1;
  int log_threads = 0; while ((2 << log_threads) <= threads) log_threads++;
  for (size_t k = 0; k < n; k++) { size_t rk = bitreverse(k, log_n); if (k < rk) { fe t = a[rk]; a[rk] = a[k]; a[k] = t; } }
  if (n < 2) return;
  fe* tw = (fe*)malloc((n / 2) * sizeof(fe));
  fe w = FR.r;
  for (size_t i = 0; i < n / 2; i++) { tw[i] = w; w = f_mul(&FR, w, *omega); }
  if ((int)log_n <= log_threads) {
    size_t chunk = 2, twiddle_chunk = n / 2;
    for (uint32_t s = 0; s < log_n; s++) {
      for (size_t base = 0; base < n; base += chunk) {
        fe* left = a + base; fe* right = a + base + chunk / 2;
        butterfly_pair(&left[0], &right[0], NULL);
        for (size_t i = 1; i < chunk / 2; i++) butterfly_pair(&left[i], &right[i], &tw[i * twiddle_chunk]);
      }
      chunk *= 2; twiddle_chunk /= 2;
    }
  } else {
    rba_t top = {a, n, 1, tw, log_threads};
    rba(&top);
  }
  free(tw);
}

/* ------------------------------------------------------------------------------------------------
 * best_multiexp / multiexp_serial: [UPSTREAM] halo2_proofs/src/arithmetic.rs.
 * Reached from every ParamsKZG::commit / commit_lagrange inside create_proof and keygen.
 * Shape kept: threads contiguous chunks of floor(n/threads) (so a remainder makes one extra chunk);
 * per chunk c = 1 (<4), 3 (<32), else ceil(ln(len)); segments = 256/c + 1 processed high to low with c
 * doublings each; unsigned c-bit digits read from the canonical little-endian repr through a 64-bit
 * window; 2^c - 1 buckets promoted lazily None -> Affine -> Projective; summation by parts; the
 * per-chunk results are folded in order.
 * ---------------------------------------------------------------------------------------------- */
static inline size_t get_at(size_t segment, size_t c, const uint8_t bytes[32]) {
  size_t skip_bits = segment * c, skip_bytes = skip_bits / 8;
  if (skip_bytes >= 32) return 0;
  uint8_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t i = 0; i < 8 && skip_bytes + i < 32; i++) v[i] = bytes[skip_bytes + i];
  uint64_t tmp; memcpy(&tmp, v, 8);
  tmp >>= skip_bits - skip_bytes * 8;
  tmp %= ((uint64_t)1 << c);
  return (size_t)tmp;
}
typedef struct { uint8_t kind; g1a a; g1j p; } bucket_t;  /* 0 None, 1 Affine, 2 Projective */
static void multiexp_serial(const fe* coeffs, const g1a* bases, size_t n, g1j* acc) {
  uint8_t (*repr)[32] = (uint8_t(*)[32])malloc(n * 32);
  for (size_t i = 0; i < n; i++) { fe c = f_to_canonical(&FR, coeffs[i]); memcpy(repr[i], c.l, 32); }
  size_t c;
  if (n < 4) c = 1; else if (n < 32) c = 3; else c = (size_t)ceil(log((double)(uint32_t)n));
  size_t segments = 256 / c + 1, nb = ((size_t)1 << c) - 1;
  bucket_t* buckets = (bucket_t*)malloc(nb * sizeof(bucket_t));
  for (size_t seg = segments; seg-- > 0;) {
    for (size_t d = 0; d < c; d++) *acc = g1j_double(acc);
    for (size_t b = 0; b < nb; b++) buckets[b].kind = 0;
    for (size_t i = 0; i < n; i++) {
      size_t d = get_at(seg, c, repr[i]);
      if (!d) continue;
      bucket_t* bk = &buckets[d - 1];
      if (bk->kind == 0) { bk->kind = 1; bk->a = bases[i]; }
      else if (bk->kind == 1) { g1j t = g1j_from_affine(&bk->a); bk->p = g1j_add_mixed(&t, &bases[i]); bk->kind = 2; }
      else bk->p = g1j_add_mixed(&bk->p, &bases[i]);
    }
    g1j running = g1j_identity();
    for (size_t b = nb; b-- > 0;) {
      bucket_t* bk = &buckets[b];
      if (bk->kind == 1) running = g1j_add_mixed(&running, &bk->a);
      else if (bk->kind == 2) running = g1j_add(&running, &bk->p);
      *acc = g1j_add(acc, &running);
    }
  }
  free(buckets); free(repr);
}
typedef struct { const fe* c; const g1a* b; size_t n; g1j acc; } mes_t;
static void mes_run(void* p) { mes_t* s = (mes_t*)p; s->acc = g1j_identity(); multiexp_serial(s->c, s->b, s->n, &s->acc); }
void orc_best_multiexp(const fe* coeffs, const g1a* bases, size_t n, int threads, g1j* out) {
  if (threads < 1) threads = 1;
  if (n > (size_t)threads) {
    size_t chunk = n / threads, nchunks = (n + chunk - 1) / chunk;
    mes_t* st = (mes_t*)malloc(nchunks * sizeof(mes_t));
    task_t* tk = (task_t*)malloc(nchunks * sizeof(task_t));
    for (size_t i = 0; i < nchunks; i++) {
      size_t lo = i * chunk, len = (lo + chunk <= n) ? chunk : n - lo;
      st[i].c = coeffs + lo; st[i].b = bases + lo; st[i].n = len;
      tk[i].fn = mes_run; tk[i].arg = &st[i];
    }
    run_tasks(tk, (int)nchunks);
    g1j acc = g1j_identity();
    for (size_t i = 0; i < nchunks; i++) acc = g1j_add(&acc, &st[i].acc);
    *out = acc;
    free(st); free(tk);
  } else {
    g1j acc = g1j_identity();
    multiexp_serial(coeffs, bases, n, &acc);
    *out = acc;
  }
}

/* ------------------------------------------------------------------------------------------------
 * EvaluationDomain: [UPSTREAM] halo2_proofs/src/poly/domain.rs (new, lagrange_to_coeff, coeff_to_extended,
 * extended_to_coeff, divide_by_vanishing_poly, rotate_extended). SURVEY.md Appendix B.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  uint32_t k, extended_k, quotient_poly_degree;
  fe omega, omega_inv, extended_omega, extended_omega_inv, g_coset, g_coset_inv, ifft_divisor, extended_ifft_divisor;
  uint32_t t_len;
  fe* t_evaluations;
} orc_domain;

orc_domain* orc_domain_new(uint32_t j, uint32_t k) {
  orc_domain* d = (orc_domain*)calloc(1, sizeof(orc_domain));
  d->k = k; d->quotient_poly_degree = j - 1;
  uint64_t n = (uint64_t)1 << k;
  uint32_t ek = k; while (((uint64_t)1 << ek) < n * d->quotient_poly_degree) ek++;
  d->extended_k = ek;
  fe w = FR_ROOT_OF_UNITY;
  for (uint32_t i = ek; i < 28; i++) w = f_sqr(&FR, w);
  d->extended_omega = w; d->extended_omega_inv = f_inv(&FR, w);
  for (uint32_t i = k; i < ek; i++) w = f_sqr(&FR, w);
  d->omega = w; d->omega_inv = f_inv(&FR, w);
  d->g_coset = FR_ZETA; d->g_coset_inv = FR_ZETA2;
  d->ifft_divisor = f_inv(&FR, f_from_u64(&FR, n));
  d->extended_ifft_divisor = f_inv(&FR, f_from_u64(&FR, (uint64_t)1 << ek));
  /* t_evaluations[i] = ((zeta * extended_omega^i)^n - 1)^-1 for i < 2^(ek-k) */
  d->t_len = 1u << (ek - k);
  d->t_evaluations = (fe*)malloc(d->t_len * sizeof(fe));
  fe cur = f_pow(&FR, d->g_coset, (uint64_t[4]){n, 0, 0, 0});
  fe step = f_pow(&FR, d->extended_omega, (uint64_t[4]){n, 0, 0, 0});
  for (uint32_t i = 0; i < d->t_len; i++) { d->t_evaluations[i] = f_inv(&FR, f_sub(&FR, cur, FR.r)); cur = f_mul(&FR, cur, step); }
  return d;
}
void orc_domain_free(orc_domain* d) { if (d) { free(d->t_evaluations); free(d); } }
void orc_domain_describe(const orc_domain* d, uint32_t* extended_k, fe* omega, fe* extended_omega, fe* consts6, fe* t_eval /* t_len */) {
  *extended_k = d->extended_k; *omega = d->omega; *extended_omega = d->extended_omega;
  consts6[0] = d->omega_inv; consts6[1] = d->extended_omega_inv; consts6[2] = d->g_coset; consts6[3] = d->g_coset_inv;
  consts6[4] = d->ifft_divisor; consts6[5] = d->extended_ifft_divisor;
  if (t_eval) memcpy(t_eval, d->t_evaluations, d->t_len * sizeof(fe));
}
/* a: n values in place */
void orc_lagrange_to_coeff(const orc_domain* d, fe* a, int threads) {
  size_t n = (size_t)1 << d->k;
  orc_best_fft(a, &d->omega_inv, d->k, threads);
  for (size_t i = 0; i < n; i++) a[i] = f_mul(&FR, a[i], d->ifft_divisor);
}
/* in: n coefficients; out: 2^extended_k evaluations over the zeta-coset */
void orc_coeff_to_extended(const orc_domain* d, const fe* in, fe* out, int threads) {
  size_t n = (size_t)1 << d->k, e = (size_t)1 << d->extended_k;
  for (size_t i = 0; i < n; i++) {
    size_t m = i % 3;
    out[i] = (m == 0) ? in[i] : f_mul(&FR, in[i], m == 1 ? d->g_coset : d->g_coset_inv);
  }
  memset(out + n, 0, (e - n) * sizeof(fe));
  orc_best_fft(out, &d->extended_omega, d->extended_k, threads);
}
/* in: 2^extended_k evaluations (destroyed); out: n*(j-1) coefficients */
void orc_extended_to_coeff(const orc_domain* d, fe* in, fe* out, int threads) {
  size_t e = (size_t)1 << d->extended_k, keep = ((size_t)1 << d->k) * d->quotient_poly_degree;
  orc_best_fft(in, &d->extended_omega_inv, d->extended_k, threads);
  for (size_t i = 0; i < e; i++) {
    fe v = f_mul(&FR, in[i], d->extended_ifft_divisor);
    size_t m = i % 3;
    if (m) v = f_mul(&FR, v, m == 1 ? d->g_coset_inv : d->g_coset);
    in[i] = v;
  }
  memcpy(out, in, keep * sizeof(fe));
}
void orc_divide_by_vanishing_poly(const orc_domain* d, fe* a) {
  size_t e = (size_t)1 << d->extended_k;
  for (size_t i = 0; i < e; i++) a[i] = f_mul(&FR, a[i], d->t_evaluations[i % d->t_len]);
}

/* [UPSTREAM] arithmetic.rs eval_polynomial (Horner), kate_division (synthetic division by X - b),
 * ff::BatchInvert (zero entries stay zero). */
void orc_eval_polynomial(fe* out, const fe* poly, size_t n, const fe* point) {
  fe acc; memset(&acc, 0, sizeof acc);
  for (size_t i = n; i-- > 0;) acc = f_add(&FR, f_mul(&FR, acc, *point), poly[i]);
  *out = acc;
}
void orc_kate_division(fe* q /* n-1 */, const fe* a, size_t n, const fe* b) {
  fe nb = f_neg(&FR, *b), tmp; memset(&tmp, 0, sizeof tmp);
  for (size_t i = n - 1; i-- > 0;) {
    fe lead = f_sub(&FR, a[i + 1], tmp);
    q[i] = lead;
    tmp = f_mul(&FR, lead, nb);
  }
}
void orc_batch_invert(fe* a, size_t n) {
  fe* acc = (fe*)malloc(n * sizeof(fe));
  fe run = FR.r;
  for (size_t i = 0; i < n; i++) { acc[i] = run; if (!f_is_zero(a[i])) run = f_mul(&FR, run, a[i]); }
  run = f_inv(&FR, run);
  for (size_t i = n; i-- > 0;) {
    if (f_is_zero(a[i])) continue;
    fe t = f_mul(&FR, run, acc[i]);
    run = f_mul(&FR, run, a[i]);
    a[i] = t;
  }
  free(acc);
}

/* ------------------------------------------------------------------------------------------------
 * ChaCha20 keystream: [UPSTREAM] rand_chacha ChaCha20Rng (djb variant: 64-bit block counter in words
 * 12-13, 64-bit stream id 0 in words 14-15, 20 rounds, output words in keystream order).
 * halo2-base utils::fs::gen_srs seeds it with [0u8;32] (reference call sites prover/src/cli.rs:48,165,191).
 * ---------------------------------------------------------------------------------------------- */
#define ROTL32(v, n) (((v) << (n)) | ((v) >> (32 - (n))))
#define QR(a, b, c, d) a += b; d ^= a; d = ROTL32(d, 16); c += d; b ^= c; b = ROTL32(b, 12); a += b; d ^= a; d = ROTL32(d, 8); c += d; b ^= c; b = ROTL32(b, 7);
void orc_chacha20_block(const uint8_t key[32], uint64_t counter, uint8_t out[64]) {
  uint32_t s[16], x[16];
  s[0] = 0x61707865; s[1] = 0x3320646e; s[2] = 0x79622d32; s[3] = 0x6b206574;
  memcpy(&s[4], key, 32);
  s[12] = (uint32_t)counter; s[13] = (uint32_t)(counter >> 32); s[14] = 0; s[15] = 0;
  memcpy(x, s, 64);
  for (int i = 0; i < 10; i++) {
    QR(x[0], x[4], x[8], x[12]) QR(x[1], x[5], x[9], x[13]) QR(x[2], x[6], x[10], x[14]) QR(x[3], x[7], x[11], x[15])
    QR(x[0], x[5], x[10], x[15]) QR(x[1], x[6], x[11], x[12]) QR(x[2], x[7], x[8], x[13]) QR(x[3], x[4], x[9], x[14])
  }
  for (int i = 0; i < 16; i++) x[i] += s[i];
  memcpy(out, x, 64);
}
/* Fill `n` Fr elements the way `Fr::random(&mut ChaCha20Rng::from_seed(seed))` called n times would. */
void orc_fr_random_chacha(fe* out, size_t n, const uint8_t seed[32]) {
  for (size_t i = 0; i < n; i++) { uint8_t blk[64]; orc_chacha20_block(seed, i, blk); orc_fr_from_u512(&out[i], blk); }
}
/* the same stream from its `first`-th draw on (draw i = keystream block i) */
void orc_fr_random_chacha_from(fe* out, size_t n, const uint8_t seed[32], uint64_t first) {
  for (size_t i = 0; i < n; i++) { uint8_t blk[64]; orc_chacha20_block(seed, first + i, blk); orc_fr_from_u512(&out[i], blk); }
}

/* ------------------------------------------------------------------------------------------------
 * ParamsKZG::setup with the seed-0 RNG: [UPSTREAM] halo2_proofs/src/poly/kzg/commitment.rs `setup`
 * (s = Fr::random(rng) first; g[i] = s^i * G1; g_lagrange[i] = ((s^n - 1)/n) * omega^i / (s - omega^i) * G1;
 * s_g2 = s * G2) as invoked by halo2-base gen_srs(k). Ranges are generated on demand so the K=23/24
 * known-answer tests need not materialise 2^24 points.
 * ---------------------------------------------------------------------------------------------- */
void orc_srs_tau(fe* tau) { uint8_t seed[32] = {0}; orc_fr_random_chacha(tau, 1, seed); }

/* fixed-base table for G1 generator: 32 windows of 8 bits, affine */
static g1a* g_fb_table = NULL;  /* [32][255] */
static pthread_mutex_t g_fb_lock = PTHREAD_MUTEX_INITIALIZER;
static void fb_table_build(void) {
  pthread_mutex_lock(&g_fb_lock);
  if (!g_fb_table) {
    g1j* t = (g1j*)malloc(32 * 255 * sizeof(g1j));
    g1j base = g1j_from_affine(&G1_GEN);
    for (int w = 0; w < 32; w++) {
      g1j cur = base;
      for (int d = 0; d < 255; d++) { t[w * 255 + d] = cur; cur = g1j_add(&cur, &base); }
      base = cur;  /* 256 * base */
    }
    g1a* a = (g1a*)malloc(32 * 255 * sizeof(g1a));
    g1_batch_normalize(t, a, 32 * 255);
    free(t);
    g_fb_table = a;
  }
  pthread_mutex_unlock(&g_fb_lock);
}
static g1j fb_mul(const fe* scalar_mont) {
  fe c = f_to_canonical(&FR, *scalar_mont);
  const uint8_t* b = (const uint8_t*)c.l;
  g1j acc = g1j_identity();
  for (int w = 0; w < 32; w++) if (b[w]) acc = g1j_add_mixed(&acc, &g_fb_table[w * 255 + b[w] - 1]);
  return acc;
}
typedef struct { const fe* s; g1a* out; size_t n; } fbm_t;
static void fbm_run(void* p) {
  fbm_t* s = (fbm_t*)p;
  g1j* tmp = (g1j*)malloc(s->n * sizeof(g1j));
  for (size_t i = 0; i < s->n; i++) tmp[i] = fb_mul(&s->s[i]);
  g1_batch_normalize(tmp, s->out, s->n);
  free(tmp);
}
/* out[i] = scalars[i] * G1 (affine) */
void orc_g1_fixed_base_mul(const fe* scalars, size_t n, int threads, g1a* out) {
  fb_table_build();
  if (threads < 1) threads = 1;
  if ((size_t)threads > n) threads = (int)(n ? n : 1);
  fbm_t* st = (fbm_t*)malloc(threads * sizeof(fbm_t));
  task_t* tk = (task_t*)malloc(threads * sizeof(task_t));
  size_t per = (n + threads - 1) / threads;
  int used = 0;
  for (int t = 0; t < threads; t++) {
    size_t lo = (size_t)t * per; if (lo >= n) break;
    size_t len = lo + per <= n ? per : n - lo;
    st[used].s = scalars + lo; st[used].out = out + lo; st[used].n = len;
    tk[used].fn = fbm_run; tk[used].arg = &st[used]; used++;
  }
  if (used) run_tasks(tk, used);
  free(st); free(tk);
}
/* scalars of g[start .. start+count): tau^i */
void orc_srs_g_scalars(uint32_t k, size_t start, size_t count, fe* out) {
  (void)k;
  fe tau; orc_srs_tau(&tau);
  fe cur = f_pow(&FR, tau, (uint64_t[4]){start, 0, 0, 0});
  for (size_t i = 0; i < count; i++) { out[i] = cur; cur = f_mul(&FR, cur, tau); }
}
/* scalars of g_lagrange[start .. start+count): L_i(tau) = ((tau^n - 1)/n) * omega^i / (tau - omega^i) */
void orc_srs_g_lagrange_scalars(uint32_t k, size_t start, size_t count, fe* out) {
  fe tau; orc_srs_tau(&tau);
  uint64_t n = (uint64_t)1 << k;
  fe omega = FR_ROOT_OF_UNITY; for (uint32_t i = k; i < 28; i++) omega = f_sqr(&FR, omega);
  fe tn = f_pow(&FR, tau, (uint64_t[4]){n, 0, 0, 0});
  fe coef = f_mul(&FR, f_sub(&FR, tn, FR.r), f_inv(&FR, f_from_u64(&FR, n)));
  fe wi = f_pow(&FR, omega, (uint64_t[4]){start, 0, 0, 0});
  fe* den = (fe*)malloc(count * sizeof(fe));
  fe* num = (fe*)malloc(count * sizeof(fe));
  for (size_t i = 0; i < count; i++) { num[i] = f_mul(&FR, coef, wi); den[i] = f_sub(&FR, tau, wi); wi = f_mul(&FR, wi, omega); }
  orc_batch_invert(den, count);
  for (size_t i = 0; i < count; i++) out[i] = f_mul(&FR, num[i], den[i]);
  free(den); free(num);
}
void orc_srs_g(uint32_t k, size_t start, size_t count, int threads, g1a* out) {
  fe* s = (fe*)malloc(count * sizeof(fe)); orc_srs_g_scalars(k, start, count, s);
  orc_g1_fixed_base_mul(s, count, threads, out); free(s);
}
void orc_srs_g_lagrange(uint32_t k, size_t start, size_t count, int threads, g1a* out) {
  fe* s = (fe*)malloc(count * sizeof(fe)); orc_srs_g_lagrange_scalars(k, start, count, s);
  orc_g1_fixed_base_mul(s, count, threads, out); free(s);
}
/* s_g2 = tau * G2, affine, canonical big-endian-free: returns Montgomery limbs (x.c0, x.c1, y.c0, y.c1) */
void orc_srs_s_g2(fe out[4]) {
  fe tau; orc_srs_tau(&tau);
  fe c = f_to_canonical(&FR, tau);
  g2j r; memset(&r, 0, sizeof r); r.y.c0 = FQ.r;
  for (int i = 255; i >= 0; i--) {
    r = g2j_double(&r);
    if ((c.l[i >> 6] >> (i & 63)) & 1) r = g2j_add_mixed(&r, &G2_GEN);
  }
  fe2 zi = f2_inv(r.z), zi2 = f2_sqr(zi);
  fe2 x = f2_mul(r.x, zi2), y = f2_mul(r.y, f2_mul(zi2, zi));
  out[0] = x.c0; out[1] = x.c1; out[2] = y.c0; out[3] = y.c1;
}

/* Known-tau shortcut (SURVEY.md 8c): commit(p) = p(tau)*G1, commit_lagrange(v) = (sum v_i L_i(tau))*G1.
 * An INDEPENDENT check of any MSM over the seed-0 SRS in O(n) field operations. */
void orc_commit_known_tau(const fe* coeffs, size_t n, g1a* out) {
  fe tau; orc_srs_tau(&tau);
  fe v; orc_eval_polynomial(&v, coeffs, n, &tau);
  fb_table_build();
  g1j p = fb_mul(&v); *out = g1j_to_affine(&p);
}
void orc_commit_lagrange_known_tau(uint32_t k, const fe* evals, size_t n_used, g1a* out) {
  size_t blk = 1 << 16;
  fe* ls = (fe*)malloc(blk * sizeof(fe));
  fe acc; memset(&acc, 0, sizeof acc);
  for (size_t lo = 0; lo < n_used; lo += blk) {
    size_t len = lo + blk <= n_used ? blk : n_used - lo;
    orc_srs_g_lagrange_scalars(k, lo, len, ls);
    for (size_t i = 0; i < len; i++) acc = f_add(&FR, acc, f_mul(&FR, evals[lo + i], ls[i]));
  }
  free(ls);
  fb_table_build();
  g1j p = fb_mul(&acc); *out = g1j_to_affine(&p);
}

/* ------------------------------------------------------------------------------------------------
 * Quotient numerator: [UPSTREAM] halo2_proofs/src/plonk/evaluation.rs -- GraphEvaluator::evaluate,
 * Evaluator::evaluate_h (custom gates, permutation argument, lookup argument), restated from the PSE fork
 * (SURVEY.md 8a row a6). No reference-owned vector pins these (no Rust host, proofs are randomised), so
 * parity for this row is GPU vs this restatement on synthetic constraint systems: "parity unpinned".
 *
 * Program encoding shared with the CUDA side (spectre_b200/csrc/quotient.cu): a calculation is
 *   word0 = op | nparts << 8        op: 0 Add 1 Sub 2 Mul 3 Square 4 Double 5 Negate 6 Horner 7 Store
 *   word1 = target intermediate
 *   then sources, two words each: kind, idx | rot_idx << 16
 *       kind: 0 Constant 1 Intermediate 2 Fixed 3 Advice 4 Instance 5 Challenge 6 Beta 7 Gamma 8 Theta 9 Y 10 PreviousValue
 *   Add/Sub/Mul: a, b. Square/Double/Negate/Store: a. Horner: start, factor, then nparts parts.
 * ---------------------------------------------------------------------------------------------- */
static inline uint64_t rotation_idx(uint64_t idx, int32_t rot, int32_t rot_scale, int64_t isize) {
  int64_t v = ((int64_t)idx + (int64_t)rot * rot_scale) % isize;
  if (v < 0) v += isize;
  return (uint64_t)v;
}
typedef struct {
  const fe* constants; const fe* inter; const uint64_t* rot_idx;
  const fe* const* fixed; const fe* const* advice; const fe* const* instance; const fe* challenges;
  const fe* bgty; fe previous;
} graph_env;
static inline fe graph_src(const graph_env* e, const uint32_t* w) {
  uint32_t kind = w[0], idx = w[1] & 0xffff, rot = w[1] >> 16;
  switch (kind) {
    case 0: return e->constants[idx];
    case 1: return e->inter[idx];
    case 2: return e->fixed[idx][e->rot_idx[rot]];
    case 3: return e->advice[idx][e->rot_idx[rot]];
    case 4: return e->instance[idx][e->rot_idx[rot]];
    case 5: return e->challenges[idx];
    case 6: return e->bgty[0];
    case 7: return e->bgty[1];
    case 8: return e->bgty[2];
    case 9: return e->bgty[3];
    default: return e->previous;
  }
}
void orc_graph_evaluate(const uint32_t* prog, uint32_t ncalc, uint32_t n_inter, const fe* constants, const int32_t* rotations, uint32_t nrot,
                        const fe* const* fixed, const fe* const* advice, const fe* const* instance, const fe* challenges, const fe* bgty,
                        fe* values, uint64_t size, int32_t rot_scale) {
  fe* inter = (fe*)malloc((n_inter ? n_inter : 1) * sizeof(fe));
  uint64_t* ridx = (uint64_t*)malloc((nrot ? nrot : 1) * sizeof(uint64_t));
  for (uint64_t idx = 0; idx < size; idx++) {
    for (uint32_t r = 0; r < nrot; r++) ridx[r] = rotation_idx(idx, rotations[r], rot_scale, (int64_t)size);
    graph_env e = {constants, inter, ridx, fixed, advice, instance, challenges, bgty, values[idx]};
    const uint32_t* w = prog;
    fe last; memset(&last, 0, sizeof last);
    for (uint32_t c = 0; c < ncalc; c++) {
      uint32_t op = w[0] & 0xff, nparts = w[0] >> 8, target = w[1];
      fe r;
      if (op <= 2) {
        fe a = graph_src(&e, w + 2), b = graph_src(&e, w + 4);
        r = op == 0 ? f_add(&FR, a, b) : op == 1 ? f_sub(&FR, a, b) : f_mul(&FR, a, b);
        w += 6;
      } else if (op == 6) {
        fe acc = graph_src(&e, w + 2), factor = graph_src(&e, w + 4);
        for (uint32_t p = 0; p < nparts; p++) acc = f_add(&FR, f_mul(&FR, acc, factor), graph_src(&e, w + 6 + 2 * p));
        r = acc; w += 6 + 2 * nparts;
      } else {
        fe a = graph_src(&e, w + 2);
        r = op == 3 ? f_sqr(&FR, a) : op == 4 ? f_dbl(&FR, a) : op == 5 ? f_neg(&FR, a) : a;
        w += 4;
      }
      inter[target] = r; last = r;
    }
    values[idx] = ncalc ? last : (fe){{0, 0, 0, 0}};
  }
  free(inter); free(ridx);
}

/* Permutation argument part of evaluate_h. sets: n_sets product cosets z_i; columns: n_cols value cosets and sigma
 * cosets in permutation order, chunk_len per set (last set may be short). */
void orc_permutation_constraints(fe* values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len,
                                 const fe* const* z, uint32_t n_cols, const fe* const* col_values, const fe* const* sigma,
                                 const fe* l0, const fe* l_last, const fe* l_active, const fe* beta, const fe* gamma, const fe* y,
                                 const fe* delta, const fe* extended_omega) {
  if (!n_sets) return;
  fe delta_start = f_mul(&FR, *beta, FR_ZETA);
  fe beta_term = FR.r;  /* extended_omega^idx */
  for (uint64_t idx = 0; idx < size; idx++) {
    uint64_t r_next = rotation_idx(idx, 1, rot_scale, (int64_t)size), r_last = rotation_idx(idx, last_rotation, rot_scale, (int64_t)size);
    fe v = values[idx];
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, FR.r, z[0][idx]), l0[idx]));
    fe zl = z[n_sets - 1][idx];
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, f_sqr(&FR, zl), zl), l_last[idx]));
    for (uint32_t s = 1; s < n_sets; s++)
      v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, z[s][idx], z[s - 1][r_last]), l0[idx]));
    fe current_delta = f_mul(&FR, delta_start, beta_term);
    for (uint32_t s = 0; s < n_sets; s++) {
      uint32_t lo = s * chunk_len, hi = lo + chunk_len < n_cols ? lo + chunk_len : n_cols;
      fe left = z[s][r_next], right = z[s][idx];
      for (uint32_t c = lo; c < hi; c++) left = f_mul(&FR, left, f_add(&FR, f_add(&FR, col_values[c][idx], f_mul(&FR, *beta, sigma[c][idx])), *gamma));
      for (uint32_t c = lo; c < hi; c++) { right = f_mul(&FR, right, f_add(&FR, f_add(&FR, col_values[c][idx], current_delta), *gamma)); current_delta = f_mul(&FR, current_delta, *delta); }
      v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, left, right), l_active[idx]));
    }
    values[idx] = v;
    beta_term = f_mul(&FR, beta_term, *extended_omega);
  }
}

/* Lookup argument part of evaluate_h for one lookup; table_value[idx] = (compressed input + beta)(compressed table + gamma)
 * as produced by that lookup's GraphEvaluator. */
void orc_lookup_constraints(fe* values, uint64_t size, int32_t rot_scale, const fe* product, const fe* permuted_input, const fe* permuted_table,
                            const fe* table_value, const fe* l0, const fe* l_last, const fe* l_active, const fe* beta, const fe* gamma, const fe* y) {
  for (uint64_t idx = 0; idx < size; idx++) {
    uint64_t r_next = rotation_idx(idx, 1, rot_scale, (int64_t)size), r_prev = rotation_idx(idx, -1, rot_scale, (int64_t)size);
    fe a_minus_s = f_sub(&FR, permuted_input[idx], permuted_table[idx]);
    fe v = values[idx], zp = product[idx];
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, FR.r, zp), l0[idx]));
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, f_sqr(&FR, zp), zp), l_last[idx]));
    fe lhs = f_mul(&FR, f_mul(&FR, product[r_next], f_add(&FR, permuted_input[idx], *beta)), f_add(&FR, permuted_table[idx], *gamma));
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_sub(&FR, lhs, f_mul(&FR, zp, table_value[idx])), l_active[idx]));
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, a_minus_s, l0[idx]));
    v = f_add(&FR, f_mul(&FR, v, *y), f_mul(&FR, f_mul(&FR, a_minus_s, f_sub(&FR, permuted_input[idx], permuted_input[r_prev])), l_active[idx]));
    values[idx] = v;
  }
}
void orc_fr_delta(fe* out) {  /* Fr::DELTA = MULTIPLICATIVE_GENERATOR^(2^S) = 7^(2^28) */
  *out = f_pow(&FR, f_from_u64(&FR, 7), (uint64_t[4]){1ull << 28, 0, 0, 0});
}

/* G2 generator and s_g2 in the RawBytes layout of ParamsKZG::write (x.c0, x.c1, y.c0, y.c1; Montgomery limbs). */
void orc_srs_g2_raw(fe g2[4], fe s_g2[4]) {
  g2[0] = G2_GEN.x.c0; g2[1] = G2_GEN.x.c1; g2[2] = G2_GEN.y.c0; g2[3] = G2_GEN.y.c1;
  orc_srs_s_g2(s_g2);
}

/* ------------------------------------------------------------------------------------------------
 * permute_expression_pair: [UPSTREAM] halo2_proofs/src/plonk/lookup/prover.rs (stage 4 of create_proof,
 * SURVEY.md 8a row a8). Values are compared as halo2curves' `Ord for Fr` does: by canonical integer.
 * Returns 0, or -1 when an input value does not occur in the table (upstream: Error::ConstraintSystemFailure).
 * Only the first `usable` rows take part; blinding rows are appended by the caller from its RNG.
 * ---------------------------------------------------------------------------------------------- */
static int canon_cmp(const void* pa, const void* pb) {
  const uint64_t* a = (const uint64_t*)pa; const uint64_t* b = (const uint64_t*)pb;
  for (int i = 3; i >= 0; i--) { if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1; }
  return 0;
}
int orc_permute_expression_pair(const fe* input, const fe* table, size_t usable, fe* permuted_input, fe* permuted_table) {
  fe* in = (fe*)malloc((usable ? usable : 1) * sizeof(fe));
  fe* tb = (fe*)malloc((usable ? usable : 1) * sizeof(fe));
  uint8_t* used = (uint8_t*)calloc(usable ? usable : 1, 1);
  size_t* repeated = (size_t*)malloc((usable ? usable : 1) * sizeof(size_t));
  for (size_t i = 0; i < usable; i++) { in[i] = f_to_canonical(&FR, input[i]); tb[i] = f_to_canonical(&FR, table[i]); }
  qsort(in, usable, sizeof(fe), canon_cmp);      /* permuted_input_expression.sort() */
  qsort(tb, usable, sizeof(fe), canon_cmp);      /* the BTreeMap of table values, as a sorted multiset */
  size_t nrep = 0; int rc = 0;
  for (size_t row = 0; row < usable; row++) {
    permuted_input[row] = f_mul(&FR, in[row], FR.r2);
    if (row == 0 || canon_cmp(&in[row], &in[row - 1]) != 0) {
      permuted_table[row] = permuted_input[row];
      /* remove one instance of the value from the leftover multiset: first unused occurrence */
      size_t lo = 0, hi = usable;
      while (lo < hi) { size_t mid = (lo + hi) / 2; if (canon_cmp(&tb[mid], &in[row]) < 0) lo = mid + 1; else hi = mid; }
      if (lo >= usable || canon_cmp(&tb[lo], &in[row]) != 0) { rc = -1; break; }
      used[lo] = 1;   /* distinct input values hit distinct first occurrences */
    } else repeated[nrep++] = row;
  }
  if (rc == 0) {
    /* leftover table elements ascending, each popped onto the LAST remaining repeated row */
    for (size_t i = 0; i < usable; i++) {
      if (used[i]) continue;
      if (!nrep) { rc = -2; break; }
      permuted_table[repeated[--nrep]] = f_mul(&FR, tb[i], FR.r2);
    }
    if (rc == 0 && nrep) rc = -2;
  }
  free(in); free(tb); free(used); free(repeated);
  return rc;
}

/* ------------------------------------------------------------------------------------------------
 * Argument provers: [UPSTREAM] halo2_proofs/src/plonk/permutation/prover.rs (Argument::commit),
 * src/plonk/lookup/prover.rs (Permuted::commit_product) -- SURVEY.md 8a row a8. Restated in the
 * upstream order: denominators over all rows, batch inversion, numerators, running product, blinding
 * tail. "parity unpinned" (no reference-owned vector; GPU vs this restatement).
 * ---------------------------------------------------------------------------------------------- */
static fe fr_omega_k(uint32_t k) { fe w = FR_ROOT_OF_UNITY; for (uint32_t i = k; i < 28; i++) w = f_sqr(&FR, w); return w; }

/* One permutation set: columns values[c], permuted columns sigma[c] (Lagrange basis, n = 2^k rows). deltaomega starts at
 * delta^first_col; z[0] = *last_z; the last n_blinds rows are overwritten with blinds; *last_z <- z[n - n_blinds - 1]. */
void orc_permutation_product(uint32_t k, const fe* const* values, const fe* const* sigma, uint32_t n_cols, uint32_t first_col,
                             const fe* beta, const fe* gamma, const fe* blinds, uint32_t n_blinds, fe* last_z, fe* z) {
  size_t n = (size_t)1 << k;
  fe* modified = (fe*)malloc(n * sizeof(fe));
  for (size_t i = 0; i < n; i++) modified[i] = FR.r;
  for (uint32_t c = 0; c < n_cols; c++)
    for (size_t i = 0; i < n; i++) modified[i] = f_mul(&FR, modified[i], f_add(&FR, f_add(&FR, f_mul(&FR, *beta, sigma[c][i]), *gamma), values[c][i]));
  orc_batch_invert(modified, n);
  fe delta; orc_fr_delta(&delta);
  fe omega = fr_omega_k(k);
  fe deltaomega = FR.r;
  for (uint32_t c = 0; c < first_col; c++) deltaomega = f_mul(&FR, deltaomega, delta);
  for (uint32_t c = 0; c < n_cols; c++) {
    fe beta_term = deltaomega;   /* delta^j * omega^i */
    for (size_t i = 0; i < n; i++) {
      modified[i] = f_mul(&FR, modified[i], f_add(&FR, f_add(&FR, f_mul(&FR, beta_term, *beta), *gamma), values[c][i]));
      beta_term = f_mul(&FR, beta_term, omega);
    }
    deltaomega = f_mul(&FR, deltaomega, delta);
  }
  z[0] = *last_z;
  for (size_t row = 1; row < n; row++) z[row] = f_mul(&FR, z[row - 1], modified[row - 1]);
  for (uint32_t b = 0; b < n_blinds; b++) z[n - n_blinds + b] = blinds[b];
  *last_z = z[n - n_blinds - 1];
  free(modified);
}

void orc_lookup_product(size_t n, const fe* compressed_input, const fe* compressed_table, const fe* permuted_input, const fe* permuted_table,
                        const fe* beta, const fe* gamma, const fe* blinds, uint32_t n_blinds, fe* z) {
  fe* prod = (fe*)malloc(n * sizeof(fe));
  for (size_t i = 0; i < n; i++) prod[i] = f_mul(&FR, f_add(&FR, permuted_input[i], *beta), f_add(&FR, permuted_table[i], *gamma));
  orc_batch_invert(prod, n);
  for (size_t i = 0; i < n; i++)
    prod[i] = f_mul(&FR, prod[i], f_mul(&FR, f_add(&FR, compressed_input[i], *beta), f_add(&FR, compressed_table[i], *gamma)));
  /* z = once(1).chain(prod).scan(1, *).take(n - blinding_factors).chain(blinds) */
  fe state = FR.r;
  z[0] = state;
  for (size_t i = 1; i < n - n_blinds; i++) { state = f_mul(&FR, state, prod[i - 1]); z[i] = state; }
  for (uint32_t b = 0; b < n_blinds; b++) z[n - n_blinds + b] = blinds[b];
  free(prod);
}

/* ------------------------------------------------------------------------------------------------
 * SHPLONK prover: [UPSTREAM] halo2_proofs/src/poly/kzg/multiopen/shplonk/prover.rs
 * (ProverSHPLONK::create_proof, quotient_contribution, linearisation_contribution; SURVEY.md 8a row a9)
 * and arithmetic.rs lagrange_interpolate / evaluate_vanishing_polynomial. Polynomials are whole
 * coefficient vectors handled one after the other, as upstream does. "parity unpinned".
 * The rotation sets come from construct_intermediate_sets (restated in Python next to the transcript).
 * ---------------------------------------------------------------------------------------------- */
typedef struct { const fe* points; uint32_t n_points; const fe* const* polys; uint32_t n_polys; const fe* evals; } orc_rotation_set;

static void lagrange_interpolate(const fe* points, const fe* evals, uint32_t m, fe* out /* m */) {
  if (m == 1) { out[0] = evals[0]; return; }
  fe denoms[8][8];
  for (uint32_t j = 0; j < m; j++) { uint32_t t = 0; for (uint32_t k2 = 0; k2 < m; k2++) if (k2 != j) denoms[j][t++] = f_inv(&FR, f_sub(&FR, points[j], points[k2])); }
  for (uint32_t i = 0; i < m; i++) memset(&out[i], 0, sizeof(fe));
  for (uint32_t j = 0; j < m; j++) {
    fe tmp[9], product[9]; uint32_t tlen = 1; tmp[0] = FR.r;
    uint32_t t = 0;
    for (uint32_t k2 = 0; k2 < m; k2++) {
      if (k2 == j) continue;
      fe denom = denoms[j][t++];
      /* product = tmp * (X - x_k) * denom */
      for (uint32_t a = 0; a <= tlen; a++) memset(&product[a], 0, sizeof(fe));
      fe c0 = f_mul(&FR, f_neg(&FR, denom), points[k2]);
      for (uint32_t a = 0; a < tlen; a++) {
        product[a] = f_add(&FR, product[a], f_mul(&FR, tmp[a], c0));
        product[a + 1] = f_add(&FR, product[a + 1], f_mul(&FR, tmp[a], denom));
      }
      tlen++;
      for (uint32_t a = 0; a < tlen; a++) tmp[a] = product[a];
    }
    for (uint32_t a = 0; a < m; a++) out[a] = f_add(&FR, out[a], f_mul(&FR, tmp[a], evals[j]));
  }
}
static fe evaluate_vanishing_polynomial(const fe* roots, uint32_t m, fe z) {
  fe acc = FR.r;
  for (uint32_t i = 0; i < m; i++) acc = f_mul(&FR, acc, f_sub(&FR, z, roots[i]));
  return acc;
}
/* poly <- poly / prod (X - root): successive kate divisions; returns the new length */
static size_t div_by_vanishing(fe* poly, size_t len, const fe* roots, uint32_t m, fe* scratch) {
  for (uint32_t i = 0; i < m; i++) { orc_kate_division(scratch, poly, len, &roots[i]); len--; memcpy(poly, scratch, len * sizeof(fe)); }
  return len;
}
static int fe_same(const fe* a, const fe* b) { return memcmp(a, b, sizeof(fe)) == 0; }

/* h_x (n coefficients) = sum over sets, weighted by powers(v), of [ sum over commitments, weighted by powers(y), of (P - R) ] / Z_set
 * (upstream: `.zip(powers(*y)).map(|(q, p)| q * p).reduce(+)`, ascending powers starting at 1) */
void orc_shplonk_quotient(size_t n, const orc_rotation_set* sets, uint32_t n_sets, const fe* y, const fe* v, fe* h_x) {
  fe* n_x = (fe*)malloc(n * sizeof(fe)); fe* scratch = (fe*)malloc(n * sizeof(fe));
  memset(h_x, 0, n * sizeof(fe));
  fe power_of_v = FR.r;
  for (uint32_t s = 0; s < n_sets; s++) {
    const orc_rotation_set* rs = &sets[s];
    memset(n_x, 0, n * sizeof(fe));
    fe power_of_y = FR.r;
    for (uint32_t j = 0; j < rs->n_polys; j++) {
      fe r[8]; lagrange_interpolate(rs->points, rs->evals + (size_t)j * rs->n_points, rs->n_points, r);
      for (size_t i = 0; i < n; i++) {          /* acc + (poly - low_degree_equivalent) * power_of_y */
        fe q = rs->polys[j][i];
        if (i < rs->n_points) q = f_sub(&FR, q, r[i]);
        n_x[i] = f_add(&FR, n_x[i], f_mul(&FR, q, power_of_y));
      }
      power_of_y = f_mul(&FR, power_of_y, *y);
    }
    size_t len = div_by_vanishing(n_x, n, rs->points, rs->n_points, scratch);
    for (size_t i = len; i < n; i++) memset(&n_x[i], 0, sizeof(fe));   /* poly.resize(n, 0) */
    for (size_t i = 0; i < n; i++) h_x[i] = f_add(&FR, h_x[i], f_mul(&FR, n_x[i], power_of_v));
    power_of_v = f_mul(&FR, power_of_v, *v);
  }
  free(n_x); free(scratch);
}
/* final (n - 1 coefficients): ((sum_i v^i [ z_i * sum_j y^j (P_ij - R_ij(u)) ]) - zt_eval * h_x) / (X - u) / z_0 */
int orc_shplonk_linearisation(size_t n, const orc_rotation_set* sets, uint32_t n_sets, const fe* y, const fe* v, const fe* u, const fe* h_x, fe* out) {
  fe super[64]; uint32_t n_super = 0;
  for (uint32_t s = 0; s < n_sets; s++) for (uint32_t p = 0; p < sets[s].n_points; p++) {
    int seen = 0;
    for (uint32_t t = 0; t < n_super; t++) if (fe_same(&super[t], &sets[s].points[p])) seen = 1;
    if (!seen) { if (n_super == 64) return -1; super[n_super++] = sets[s].points[p]; }
  }
  fe* l_x = (fe*)calloc(n, sizeof(fe)); fe* inner = (fe*)malloc(n * sizeof(fe));
  fe z_0_diff; memset(&z_0_diff, 0, sizeof z_0_diff);
  fe power_of_v = FR.r;
  for (uint32_t s = 0; s < n_sets; s++) {
    const orc_rotation_set* rs = &sets[s];
    fe diffs[64]; uint32_t nd = 0;
    for (uint32_t t = 0; t < n_super; t++) { int in_set = 0; for (uint32_t p = 0; p < rs->n_points; p++) if (fe_same(&super[t], &rs->points[p])) in_set = 1; if (!in_set) diffs[nd++] = super[t]; }
    fe z_i = evaluate_vanishing_polynomial(diffs, nd, *u);
    if (s == 0) z_0_diff = z_i;
    memset(inner, 0, n * sizeof(fe));
    fe power_of_y = FR.r;
    for (uint32_t j = 0; j < rs->n_polys; j++) {
      fe r[8]; lagrange_interpolate(rs->points, rs->evals + (size_t)j * rs->n_points, rs->n_points, r);
      fe r_eval; orc_eval_polynomial(&r_eval, r, rs->n_points, u);
      for (size_t i = 0; i < n; i++) {
        fe q = rs->polys[j][i];
        if (i == 0) q = f_sub(&FR, q, r_eval);
        inner[i] = f_add(&FR, inner[i], f_mul(&FR, q, power_of_y));
      }
      power_of_y = f_mul(&FR, power_of_y, *y);
    }
    for (size_t i = 0; i < n; i++) l_x[i] = f_add(&FR, l_x[i], f_mul(&FR, f_mul(&FR, inner[i], z_i), power_of_v));
    power_of_v = f_mul(&FR, power_of_v, *v);
  }
  fe zt_eval = evaluate_vanishing_polynomial(super, n_super, *u);
  for (size_t i = 0; i < n; i++) l_x[i] = f_sub(&FR, l_x[i], f_mul(&FR, h_x[i], zt_eval));
  fe must_be_zero; orc_eval_polynomial(&must_be_zero, l_x, n, u);
  int rc = f_is_zero(must_be_zero) ? 0 : -2;      /* upstream debug_assert */
  orc_kate_division(out, l_x, n, u);
  fe z_0_diff_inv = f_inv(&FR, z_0_diff);
  for (size_t i = 0; i + 1 < n; i++) out[i] = f_mul(&FR, out[i], z_0_diff_inv);
  free(l_x); free(inner);
  return rc;
}

/* plain vector helpers for the proof driver's CPU binding (tests/plonk_oracle_engine.py) */
void orc_vec_scale(fe* a, const fe* alpha, size_t n) { for (size_t i = 0; i < n; i++) a[i] = f_mul(&FR, a[i], *alpha); }
/* out[i] = sum_p y^p polys[p][i]: vanishing::evaluate's fold of the h pieces with x^n (rev().fold(acc * xn + piece)) */
void orc_vec_fold(const fe* const* polys, size_t count, const fe* y, fe* out, size_t n) {
  for (size_t i = 0; i < n; i++) {
    fe acc; memset(&acc, 0, sizeof acc);
    for (size_t p = count; p-- > 0;) acc = f_add(&FR, f_mul(&FR, acc, *y), polys[p][i]);
    out[i] = acc;
  }
}
/* compute_inner_product(a, b) = sum_i a_i * b_i ([UPSTREAM] halo2_proofs/src/arithmetic.rs, SURVEY.md 8a row a10). Used by
 * bench.py's parity flags: for bases h_i * G1 with known h_i, MSM(s, bases) = compute_inner_product(s, h) * G1. */
void orc_compute_inner_product(fe* out, const fe* a, const fe* b, size_t n) {
  fe acc; memset(&acc, 0, sizeof acc);
  for (size_t i = 0; i < n; i++) acc = f_add(&FR, acc, f_mul(&FR, a[i], b[i]));
  *out = acc;
}
