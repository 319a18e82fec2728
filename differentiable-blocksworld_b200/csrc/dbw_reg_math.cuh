// dbw_reg_math.cuh -- per-element math of the regulariser kernels (dbw_reg.cu): the as_sdf=2 superquadric implicit of the
// overlap term with its analytic gradient, the per-difference norms of the total-variation term with their derivatives, and
// the square root of the parsimony term (src/model/dbw.py:373-405, src/utils/superquadric.py:17-38, src/model/loss.py:45).
// Plain C++ apart from the __device__ markers: tests/host_math compiles it for the CPU and checks it against torch autograd.
//
// torch's conventions are kept at every boundary, because they decide the gradients there:
//  - safe_pow(t, e) = t.clamp(1e-6).pow(e): clamp passes the gradient where t >= 1e-6 (bound included), none below it;
//  - points.clamp(-5, 5): the gradient passes where -5 <= x <= 5;
//  - pow(b, e) with both differentiable: d/db = e b^(e-1), d/de = b^e log(b);
//  - l1: d|d|/dd = sign(d), sign(0) = 0;
//  - the overlap excess clamp(min=0) passes the gradient where the excess is >= 0.
// Divisions that torch rounds correctly use __fdiv_rn: the library is built with -prec-div=false.
#pragma once
#include <math.h>

#define DBW_REG_SQRT_EPS 1e-6f           // geometry.SQRT_EPS
#define DBW_REG_POINT_CLAMP 5.f          // superquadric_implicit's points.clamp(-5, 5)
#define DBW_REG_OVERLAP_N_BLOCKS 1.95f   // losses.OVERLAP_N_BLOCKS
#define DBW_REG_OVERLAP_TEMPERATURE 0.005f

enum { DBW_REG_TV_L2 = 0, DBW_REG_TV_L1 = 1, DBW_REG_TV_L2SQ = 2 };

__device__ __forceinline__ float reg_sigmoid(float x) { return __fdiv_rn(1.f, 1.f + expf(-x)); }

// superquadric exponents eps = sigmoid(sq_eps) * 1.8 + 0.1 (dbw.py:638)
__device__ __forceinline__ float reg_sq_eps(float logit) { return reg_sigmoid(logit) * 1.8f + 0.1f; }

// sdf of geometry.superquadric_implicit at the block-frame point l:
//   p = clamp(l, -5, 5);  res = safe_pow(safe_pow(px^2, 1/e2) + safe_pow(pz^2, 1/e2), e2/e1) + safe_pow(py^2, 1/e1)
//   sdf = safe_pow(res, e1/2) - 1
__device__ __forceinline__ float sq_implicit(const float* l, float e1, float e2) {
  const float ie1 = __fdiv_rn(1.f, e1), ie2 = __fdiv_rn(1.f, e2), r21 = __fdiv_rn(e2, e1), h = e1 * 0.5f;
  const float px = fminf(fmaxf(l[0], -DBW_REG_POINT_CLAMP), DBW_REG_POINT_CLAMP);
  const float py = fminf(fmaxf(l[1], -DBW_REG_POINT_CLAMP), DBW_REG_POINT_CLAMP);
  const float pz = fminf(fmaxf(l[2], -DBW_REG_POINT_CLAMP), DBW_REG_POINT_CLAMP);
  const float x = powf(fmaxf(px * px, DBW_REG_SQRT_EPS), ie2);
  const float y = powf(fmaxf(py * py, DBW_REG_SQRT_EPS), ie1);
  const float z = powf(fmaxf(pz * pz, DBW_REG_SQRT_EPS), ie2);
  const float res = powf(fmaxf(x + z, DBW_REG_SQRT_EPS), r21) + y;
  return powf(fmaxf(res, DBW_REG_SQRT_EPS), h) - 1.f;
}

// the same sdf, and g * its gradient with respect to l (gl[3]), e1 (*ge1) and e2 (*ge2); returns the sdf
__device__ __forceinline__ float sq_implicit_backward(const float* l, float e1, float e2, float g, float* gl, float* ge1, float* ge2) {
  const float ie1 = __fdiv_rn(1.f, e1), ie2 = __fdiv_rn(1.f, e2), r21 = __fdiv_rn(e2, e1), h = e1 * 0.5f;
  float p[3], q2[3], qc[3], b[3];
  for (int k = 0; k < 3; ++k) {
    p[k] = fminf(fmaxf(l[k], -DBW_REG_POINT_CLAMP), DBW_REG_POINT_CLAMP);
    q2[k] = p[k] * p[k];
    qc[k] = fmaxf(q2[k], DBW_REG_SQRT_EPS);
    b[k] = powf(qc[k], k == 1 ? ie1 : ie2);                 // x, y, z
  }
  const float s = b[0] + b[2], sc = fmaxf(s, DBW_REG_SQRT_EPS), w = powf(sc, r21);
  const float res = w + b[1], rc = fmaxf(res, DBW_REG_SQRT_EPS), o = powf(rc, h);
  // sdf = o - 1,  o = rc^h
  const float g_rc = g * (h * powf(rc, h - 1.f));
  const float g_h = g * (o * logf(rc));
  const float g_res = res >= DBW_REG_SQRT_EPS ? g_rc : 0.f;
  // res = w + y,  w = sc^r21
  const float g_sc = g_res * (r21 * powf(sc, r21 - 1.f));
  const float g_r21 = g_res * (w * logf(sc));
  const float g_s = s >= DBW_REG_SQRT_EPS ? g_sc : 0.f;
  float g_ie1 = 0.f, g_ie2 = 0.f;
  for (int k = 0; k < 3; ++k) {
    const float gb = k == 1 ? g_res : g_s, e = k == 1 ? ie1 : ie2;
    const float g_qc = gb * (e * powf(qc[k], e - 1.f));
    const float g_e = gb * (b[k] * logf(qc[k]));
    if (k == 1) g_ie1 += g_e; else g_ie2 += g_e;
    const float g_q2 = q2[k] >= DBW_REG_SQRT_EPS ? g_qc : 0.f;
    const float g_p = g_q2 * 2.f * p[k];
    gl[k] = (l[k] >= -DBW_REG_POINT_CLAMP && l[k] <= DBW_REG_POINT_CLAMP) ? g_p : 0.f;
  }
  // ie = 1/e, r21 = e2/e1, h = e1/2
  *ge1 = -__fdiv_rn(g_ie1, e1 * e1) - __fdiv_rn(g_r21 * e2, e1 * e1) + g_h * 0.5f;
  *ge2 = -__fdiv_rn(g_ie2, e2 * e2) + __fdiv_rn(g_r21, e1);
  return o - 1.f;
}

// TV norm of one colour difference d (losses.TV_NORMS): l2 = safe_pow(|d|^2, 0.5), l1 = |d|_1, l2sq = |d|^2
__device__ __forceinline__ float tv_norm(int type, float dx, float dy, float dz) {
  if (type == DBW_REG_TV_L1) return fabsf(dx) + fabsf(dy) + fabsf(dz);
  const float s = dx * dx + dy * dy + dz * dz;
  return type == DBW_REG_TV_L2 ? sqrtf(fmaxf(s, DBW_REG_SQRT_EPS)) : s;
}

// g * d tv_norm / d d
__device__ __forceinline__ void tv_norm_backward(int type, float dx, float dy, float dz, float g, float* gd) {
  if (type == DBW_REG_TV_L1) {
    gd[0] = dx > 0.f ? g : (dx < 0.f ? -g : 0.f);
    gd[1] = dy > 0.f ? g : (dy < 0.f ? -g : 0.f);
    gd[2] = dz > 0.f ? g : (dz < 0.f ? -g : 0.f);
    return;
  }
  float gs = g;
  if (type == DBW_REG_TV_L2) {
    const float s = dx * dx + dy * dy + dz * dz;
    gs = s >= DBW_REG_SQRT_EPS ? g * (0.5f * __fdiv_rn(1.f, sqrtf(s))) : 0.f;
  }
  gd[0] = gs * 2.f * dx; gd[1] = gs * 2.f * dy; gd[2] = gs * 2.f * dz;
}

// parsimony: safe_pow(alpha, 0.5) and its derivative
__device__ __forceinline__ float parsimony_value(float a) { return sqrtf(fmaxf(a, DBW_REG_SQRT_EPS)); }
__device__ __forceinline__ float parsimony_grad(float a) {
  return a >= DBW_REG_SQRT_EPS ? 0.5f * __fdiv_rn(1.f, sqrtf(a)) : 0.f;
}
