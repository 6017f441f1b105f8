// Pair arithmetic on float2: two independent IEEE round-to-nearest operations.  The kernels keep their data in row pairs
// (one 8- or 16-byte load brings both rows); sm_90 has no packed FP32 instruction, so each pair is two scalar
// instructions.  __fmaf_rn / __fadd_rn / __fmul_rn are never contracted or reassociated by the compiler, so a pair
// rounds exactly as the packed form would.
#pragma once
#include <cuda_runtime.h>

namespace pdsb {

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

}  // namespace pdsb
