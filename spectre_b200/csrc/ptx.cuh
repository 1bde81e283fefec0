// Carry-chain primitives for 256-bit modular arithmetic on sm_90a.
//
// On the device every function is exactly one (or one fused pair of) PTX instruction(s) that reads or
// writes the implicit carry flag CC.CF. ptxas fuses a `mad.lo.cc` / `madc.hi.cc` pair on an adjacent
// register pair into a single IMAD.WIDE.U32(.X) -- that is what makes the even/odd Montgomery
// multiplier in field.cuh cost ~128 wide multiply-adds instead of ~256 narrow ones.
//
// With -DSPB_EMULATE_PTX (host compilers only) the same functions are emulated with an explicit
// thread-local carry so the *device* limb algorithms can be unit-tested on a machine with no GPU
// (tests/test_hostemu.py). The product never ships that mode.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define SPB_HD __host__ __device__ __forceinline__
#define SPB_D __device__ __forceinline__
#else
#define SPB_HD inline
#define SPB_D inline
#endif

#if defined(__CUDA_ARCH__) || defined(SPB_EMULATE_PTX)
#define SPB_LIMB32_PATH 1
#endif

namespace spb {
namespace ptx {

#if defined(__CUDA_ARCH__)

SPB_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
SPB_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
// (hi:lo) << 1, upper word: one SHF.L.W on the ALU pipe (the doubling step of a squaring)
SPB_D uint32_t shl1_hi(uint32_t lo, uint32_t hi) { uint32_t r; asm("shf.l.clamp.b32 %0, %1, %2, 1;" : "=r"(r) : "r"(lo), "r"(hi)); return r; }

// (lo,hi) = a*b
SPB_D void mul_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {
  asm("{ .reg .u64 t; mul.wide.u32 t, %2, %3; mov.b64 {%0, %1}, t; }" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
// (lo,hi) = (clo,chi) + a*b, carry-out set, no carry-in
SPB_D void mad_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
               : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}
// (lo,hi) = (clo,chi) + a*b + carry-in, carry-out set
SPB_D void madc_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
               : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}
// same, last link of a chain (carry-out proven zero by the caller, not recorded)
SPB_D void madc_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, %5;"
               : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}

#elif defined(SPB_EMULATE_PTX)

static thread_local uint32_t g_cf = 0;
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + g_cf; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + g_cf; }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; g_cf = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - g_cf; g_cf = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - g_cf; }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t shl1_hi(uint32_t lo, uint32_t hi) { return (hi << 1) | (lo >> 31); }
inline void mul_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a * b; lo = (uint32_t)t; hi = (uint32_t)(t >> 32); }
inline void wide_acc_(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi, uint32_t cin, bool set) {
  unsigned __int128 t = (unsigned __int128)a * b + (((uint64_t)chi << 32) | clo) + cin;
  lo = (uint32_t)t; hi = (uint32_t)(t >> 32);
  if (set) g_cf = (uint32_t)(t >> 64);
}
inline void mad_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) { wide_acc_(lo, hi, a, b, clo, chi, 0, true); }
inline void madc_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) { wide_acc_(lo, hi, a, b, clo, chi, g_cf, true); }
inline void madc_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) { wide_acc_(lo, hi, a, b, clo, chi, g_cf, false); }

#endif

}  // namespace ptx
}  // namespace spb
