// pair_math.cuh -- element-wise fp32 arithmetic on float2 pairs.  sm_90 has no packed fp32 pipe, so each pair is two scalar IEEE
// operations; __fadd_rn / __fmul_rn are never contracted into an fma, so every lane is rounded exactly like the scalar instruction.
#pragma once
#include <cuda_runtime.h>

__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
