// dbw_viz_math.cuh -- the per-pixel arithmetic of the resolving hard render (resolve_hard_viz_kernel, dbw_render.cu), in the
// order of operations of the torch code it replaces:
//
//   frame = avg_pool2d(samples, 4)            sum of the 4 x 4 samples row by row from a float zero, then / 16
//   rgb   = rec * alpha + (1 - alpha) * bkg   each product and sum rounded on its own (no FMA contraction)
//   u8    = (rgb * 255).clamp(0, 255).to(uint8), which truncates
//
// Division by 16 is exact as a multiplication by 1/16 (both are the correctly rounded x / 16).  The header also compiles as
// plain C++ (tests/host_math/dbw_viz_host.cpp, built with -ffp-contract=off).
#pragma once

#ifdef __CUDA_ARCH__
#define DBW_VIZ_ADD(a, b) __fadd_rn((a), (b))
#define DBW_VIZ_SUB(a, b) __fsub_rn((a), (b))
#define DBW_VIZ_MUL(a, b) __fmul_rn((a), (b))
#define DBW_VIZ_TRUNC_U8(x) ((unsigned char)__float2uint_rz(x))
#else
#define DBW_VIZ_ADD(a, b) ((a) + (b))
#define DBW_VIZ_SUB(a, b) ((a) - (b))
#define DBW_VIZ_MUL(a, b) ((a) * (b))
#define DBW_VIZ_TRUNC_U8(x) ((unsigned char)(unsigned)(x))
#endif

// one step of the box filter's running sum (samples taken row by row, left to right), and its mean
__device__ __forceinline__ float dbw_viz_box_add(float acc, float x) { return DBW_VIZ_ADD(acc, x); }
__device__ __forceinline__ float dbw_viz_box_mean(float sum) { return DBW_VIZ_MUL(sum, 0.0625f); }

__device__ __forceinline__ float dbw_viz_composite(float rec, float alpha, float bkg) {
  return DBW_VIZ_ADD(DBW_VIZ_MUL(rec, alpha), DBW_VIZ_MUL(DBW_VIZ_SUB(1.f, alpha), bkg));
}

__device__ __forceinline__ unsigned char dbw_viz_u8(float x) {
  return DBW_VIZ_TRUNC_U8(fminf(fmaxf(DBW_VIZ_MUL(x, 255.f), 0.f), 255.f));
}
