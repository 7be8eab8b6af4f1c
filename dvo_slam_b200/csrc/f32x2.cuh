// f32x2.cuh -- fp32 pairs {lo, hi} kept in one 64-bit register pair.  sm_90 has no packed fp32
// arithmetic, so every pair operation is two scalar IEEE fp32 instructions with the rounding mode
// spelled out (ptxas keeps the halves in adjacent registers: packing and unpacking cost nothing).
// Every operation here is a single correctly rounded fp32 op per lane: results are bit-identical
// to the scalar __fmaf_rn / __fmul_rn / __fadd_rn sequence the oracle's MIRROR mode restates.
#pragma once
#include <cuda_runtime.h>

namespace dvo_b200 {

typedef unsigned long long f2;  // {lo, hi} fp32 pair in an aligned 64-bit register pair

__device__ __forceinline__ f2 pk(float lo, float hi) {
  f2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ float lo(f2 v) { return __uint_as_float((unsigned)v); }
__device__ __forceinline__ float hi(f2 v) { return __uint_as_float((unsigned)(v >> 32)); }
__device__ __forceinline__ f2 bc(float s) { return pk(s, s); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) {
  return pk(__fmaf_rn(lo(a), lo(b), lo(c)), __fmaf_rn(hi(a), hi(b), hi(c)));
}
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return pk(__fmul_rn(lo(a), lo(b)), __fmul_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return pk(__fadd_rn(lo(a), lo(b)), __fadd_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return pk(__fsub_rn(lo(a), lo(b)), __fsub_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 add2_rz(f2 a, f2 b) { return pk(__fadd_rz(lo(a), lo(b)), __fadd_rz(hi(a), hi(b))); }
__device__ __forceinline__ f2 ldg_f2(const float2* p) {
  float2 v = __ldg(p);
  return pk(v.x, v.y);
}

// Correctly rounded reciprocal for normal-range arguments: MUFU.RCP (<= 1 ulp) + one Newton step in
// FMA.  Verified bit-identical to __frcp_rn for every float with 1e-30 <= |x| <= 1e30
// (scripts/micro/rcp_check.cu); arguments outside that range only occur for points that the bounds
// test rejects.
__device__ __forceinline__ float rcp_rn(float x) {
  float y0;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y0) : "f"(x));
  float e = __fmaf_rn(-x, y0, 1.0f);
  return __fmaf_rn(y0, e, y0);
}
__device__ __forceinline__ float rcp_fast(float x) {
  float y0;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y0) : "f"(x));
  return y0;
}

}  // namespace dvo_b200
