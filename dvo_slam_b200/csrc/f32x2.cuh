// f32x2.cuh -- fp32 pairs {lo, hi}.  sm_90 has no packed fp32 arithmetic, so a pair is a plain two-float struct
// (ptxas places its halves in any two registers) and every pair operation is two scalar IEEE fp32 instructions
// with the rounding mode spelled out.  The pair helpers stay because the kernel is written as the operation
// sequence the oracle's MIRROR mode restates, two channels at a time: every helper is one correctly rounded fp32
// op per lane, bit-identical to the scalar __fmaf_rn / __fmul_rn / __fadd_rn sequence MIRROR spells out.
#pragma once
#include <cuda_runtime.h>

namespace dvo_b200 {

struct f2 {  // {lo, hi} fp32 pair
  float x, y;
};

__device__ __forceinline__ f2 pk(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ float lo(f2 v) { return v.x; }
__device__ __forceinline__ float hi(f2 v) { return v.y; }
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
