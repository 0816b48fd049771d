// blance_b200/csrc/pass_common.cuh — helpers shared by the two assign-pass kernels
// (assign_pass.cuh: all warps in lock step; assign_pass_seq.cuh: sequencer warp + on-demand CTA).
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <cstdio>

#include "blance_b200.h"
#include "device_types.cuh"
#include "sticky_rank.cuh"

namespace blance_dev {

#define BL_QTAB 64
#define BL_REC_HDR 8        // record = row[SLP] | meta, w_p, top, partition | stick (2 words), 2 spare
#define BL_REC_MAX (BL_SLP_MAX + BL_REC_HDR)

struct Best { uint32_t hi, lo, pos; };

// Explicit .shared::cta accesses with 32-bit addresses for the hot loop (the generic-pointer
// path makes the compiler rebuild the shared window base from SR_CgaCtaId inside the loop).
__device__ __forceinline__ int4 lds128(uint32_t a) {
  int4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ double lds64f(uint32_t a) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ int32_t lds32(uint32_t a) {
  int32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" :: "r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t a, int32_t x) {
  asm volatile("st.shared.b32 [%0], %1;" :: "r"(a), "r"(x) : "memory");
}


// order-preserving map double -> uint64 (total order == numeric order for non-NaN)
__device__ __forceinline__ unsigned long long score_key(double r) {
  const long long b = __double_as_longlong(r);
  return (unsigned long long)(b ^ ((b >> 63) | (long long)0x8000000000000000ull));
}

// lexicographic min of (hi, lo, pos) over the warp; non-participants pass all-ones
__device__ __forceinline__ Best warp_argmin(Best v) {
  const unsigned full = 0xFFFFFFFFu;
  const uint32_t mhi = __reduce_min_sync(full, v.hi);
  const uint32_t lo2 = (v.hi == mhi) ? v.lo : 0xFFFFFFFFu;
  const uint32_t mlo = __reduce_min_sync(full, lo2);
  const uint32_t p2 = (lo2 == mlo && v.hi == mhi) ? v.pos : 0xFFFFFFFFu;
  const uint32_t mpos = __reduce_min_sync(full, p2);
  return Best{mhi, mlo, mpos};
}


// a / b, correctly rounded, for an integer-valued divisor 1 <= b < 2^31, from y = RN(1/b):
//   q0 = RN(a*y);  e = a - b*q0 (exact in one FMA);  q1 = RN(q0 + e*y)  ==  RN(a/b).
// Why one correction is enough here: q0 = (a/b)(1+e1)(1+e2) with |e1|,|e2| <= 2^-53, so the residual
// a - b*q0 has at most ~32 significant bits (b has <= 31, the cancellation removes the rest) and the FMA
// returns it exactly; then q0 + e*y = a/b + (a/b - q0)*e1, i.e. a/b perturbed by at most |a/b| * 2^-105,
// while a/b (b an integer < 2^31, a a double) is never closer than |a/b| * 2^-84 to a rounding boundary
// and never exactly on one (that would need a 54-bit significand in a).  tests/test_division.py checks
// the sequence against true division on 4e7 adversarial operands.  b == 1 (y == 1) returns a unchanged.
__device__ __forceinline__ double div_exact(double a, double b, double y) {
  const double q = __dmul_rn(a, y);
  const double e = __fma_rn(-b, q, a);
  return __fma_rn(e, y, q);
}

// rare path: n2n count beyond the j/P table
__device__ __noinline__ double q_over_p_slow(int32_t q, double Pd, double Py);


__device__ __noinline__ double q_over_p_slow(int32_t q, double Pd, double Py) { return div_exact((double)q, Pd, Py); }

// atomic add without a return value.  atomicAdd() with an unused result compiles to ATOMG ... RZ here, not RED: the
// warp then holds a scoreboard for the L2 round trip and stalls on it at its next branch.  red.* is the same relaxed, device-scope atomic and nothing waits for it.
__device__ __forceinline__ void red_add(int32_t* p, int32_t v) {
  asm volatile("red.relaxed.gpu.global.add.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// named barriers (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory"); }

}  // namespace blance_dev
