// f32x2.cuh - pairs of fp32 values carried in one 64-bit register pair (.x in the low register, .y in the high one):
// the front-end FFT and mel sums and conv1 are written over such pairs.  sm_90 has no packed fp32 instructions, so every
// pair operation is two scalar IEEE fp32 operations: each lane result is the correctly rounded fp32 result of the same
// scalar operation, exactly as a kernel written with fmaf directly.
#pragma once
#include <cuda_runtime.h>

namespace nisqa {

typedef unsigned long long f2;      // two floats: .x in the low register, .y in the high one

__device__ __forceinline__ f2 pk(float lo, float hi) {
  f2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ f2 pk(float2 v) { return pk(v.x, v.y); }
__device__ __forceinline__ f2 bc(float a) { return pk(a, a); }
__device__ __forceinline__ float2 upk(f2 v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) {
  const float2 x = upk(a), y = upk(b), z = upk(c);
  return pk(fmaf(x.x, y.x, z.x), fmaf(x.y, y.y, z.y));
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) {
  const float2 x = upk(a), y = upk(b);
  return pk(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}

// c ? a : b as a register select.  Written as `c ? x[i] : x[j]` on two array elements, the compiler may turn the choice
// into a load from a computed address, which keeps the whole array in local memory.
__device__ __forceinline__ f2 sel(bool c, f2 a, f2 b) {
  f2 r;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\tselp.b64 %0, %1, %2, p;\n\t}" : "=l"(r) : "l"(a), "l"(b), "r"((int)c));
  return r;
}
__device__ __forceinline__ float sel(bool c, float a, float b) {
  float r;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\tselp.f32 %0, %1, %2, p;\n\t}" : "=f"(r) : "f"(a), "f"(b), "r"((int)c));
  return r;
}

}  // namespace nisqa
