// Carry-chain primitives for 256-bit modular arithmetic on sm_90a.
//
// On the device every function is exactly one (or one fused pair of) PTX instruction(s) that reads or
// writes the implicit carry flag CC.CF. ptxas fuses a `mad.lo.cc` / `madc.hi.cc` pair on an adjacent
// register pair into a single IMAD.WIDE.U32(.X) -- that is what makes the even/odd Montgomery
// multiplier in field.cuh cost ~128 wide multiply-adds instead of ~256 narrow ones.
//
// With -DSPB_EMULATE_PTX (host compilers only) the same functions are emulated with an explicit
// thread-local carry so the *device* limb algorithms can be unit-tested on a machine with no GPU
// (tests/test_hostemu.py). The product never ships that mode. Adding -DSPB_EMULATE_PTX_TRACE records, per call site, the
// carries the emulated instructions read and drop (tests/test_hostemu_carry_coverage.py). Neither build compiles the asm
// below: only the device tests (tests/test_gpu_arith.py) run it.
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

#if defined(SPB_EMULATE_PTX_TRACE)
// Carry trace (CPU tests only, tests/test_hostemu_carry_coverage.py). Every instruction that reads CF records, at its call
// site, whether it saw CF = 0 or CF = 1; one that also drops its carry / borrow out (addc, subc, the last link of
// madc_wide) records the value of that carry out. The call site is the caller's, through defaulted __builtin_LINE() /
// __builtin_FILE() arguments, so the limbs of one unrolled loop share a line; the instance (the number of traced
// instructions since the last trace_mark(), which a caller issues before each element) tells them apart.
enum : uint32_t { kTraceCfIn0 = 1, kTraceCfIn1 = 2, kTraceDrop0 = 4, kTraceDrop1 = 8 };
struct TraceSite { const char* file; int line; int seq; const char* op; uint32_t seen; };
static const int kTraceCap = 8192;      // open addressing; a full table drops new sites
static const int kTraceSeqMax = 1023;   // the instances of a long element past this share one index
static TraceSite g_trace[kTraceCap];
static int g_trace_seq = 0;
inline void trace_mark() { g_trace_seq = 0; }
inline void trace_(const char* file, int line, const char* op, bool drops, uint64_t carry_out) {
  const int seq = g_trace_seq;
  const uint32_t bits = (g_cf ? kTraceCfIn1 : kTraceCfIn0) | (drops ? (carry_out ? kTraceDrop1 : kTraceDrop0) : 0u);
  if (g_trace_seq < kTraceSeqMax) g_trace_seq++;
  for (int k = 0, h = (line * 7 + seq * 131) & (kTraceCap - 1); k < kTraceCap; k++, h = (h + 1) & (kTraceCap - 1)) {
    TraceSite& s = g_trace[h];
    if (!s.file) { s = TraceSite{file, line, seq, op, bits}; return; }
    if (s.line == line && s.seq == seq && s.op == op && s.file == file) { s.seen |= bits; return; }
  }
}
#define SPB_SITE , int line_ = __builtin_LINE(), const char* file_ = __builtin_FILE()
#define SPB_TRACE(op, drops, carry_out) trace_(file_, line_, op, drops, carry_out)
#else
#define SPB_SITE
#define SPB_TRACE(op, drops, carry_out) ((void)0)
#endif

inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b SPB_SITE) { SPB_TRACE("addc_cc", false, 0); uint64_t t = (uint64_t)a + b + g_cf; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b SPB_SITE) { SPB_TRACE("addc", true, ((uint64_t)a + b + g_cf) >> 32); return a + b + g_cf; }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; g_cf = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b SPB_SITE) { SPB_TRACE("subc_cc", false, 0); uint64_t t = (uint64_t)a - b - g_cf; g_cf = (uint32_t)(t >> 63); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b SPB_SITE) { SPB_TRACE("subc", true, ((uint64_t)a - b - g_cf) >> 63); return a - b - g_cf; }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t shl1_hi(uint32_t lo, uint32_t hi) { return (hi << 1) | (lo >> 31); }
inline void mul_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a * b; lo = (uint32_t)t; hi = (uint32_t)(t >> 32); }
inline unsigned __int128 wide_acc_(uint32_t a, uint32_t b, uint32_t clo, uint32_t chi, uint32_t cin) {
  return (unsigned __int128)a * b + (((uint64_t)chi << 32) | clo) + cin;
}
inline void mad_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  unsigned __int128 t = wide_acc_(a, b, clo, chi, 0);
  lo = (uint32_t)t; hi = (uint32_t)(t >> 32); g_cf = (uint32_t)(t >> 64);
}
inline void madc_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi SPB_SITE) {
  SPB_TRACE("madc_wide_cc", false, 0);
  unsigned __int128 t = wide_acc_(a, b, clo, chi, g_cf);
  lo = (uint32_t)t; hi = (uint32_t)(t >> 32); g_cf = (uint32_t)(t >> 64);
}
inline void madc_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi SPB_SITE) {
  unsigned __int128 t = wide_acc_(a, b, clo, chi, g_cf);
  SPB_TRACE("madc_wide", true, (uint64_t)(t >> 64));
  lo = (uint32_t)t; hi = (uint32_t)(t >> 32);
}
#undef SPB_SITE
#undef SPB_TRACE

#endif

}  // namespace ptx
}  // namespace spb
