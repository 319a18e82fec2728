// Host build of the regulariser math (differentiable-blocksworld_b200/csrc/dbw_reg_math.cuh), for
// tests/test_regularisers_host.py: the superquadric implicit with its gradient and the TV norms with their derivatives, the
// very functions dbw_reg.cu inlines, driven element by element.  Test infrastructure only.
#include <cmath>

#define __device__
#define __forceinline__ inline
static inline float __fdiv_rn(float a, float b) { return a / b; }

#include "../../differentiable-blocksworld_b200/csrc/dbw_reg_math.cuh"

extern "C" {

// n points (n, 3) against per-point exponents e (n, 2): sdf (n), and with upstream g (n): gl (n, 3), ge (n, 2)
void hr_sq_implicit(int n, const float* pts, const float* e, const float* g, float* sdf, float* sdf_bwd, float* gl, float* ge) {
  for (int i = 0; i < n; ++i) {
    sdf[i] = sq_implicit(pts + 3 * i, e[2 * i], e[2 * i + 1]);
    sdf_bwd[i] = sq_implicit_backward(pts + 3 * i, e[2 * i], e[2 * i + 1], g[i], gl + 3 * i, ge + 2 * i, ge + 2 * i + 1);
  }
}

// n differences (n, 3): norm (n) and g * d norm / d d (n, 3)
void hr_tv_norm(int type, int n, const float* d, const float* g, float* out, float* gd) {
  for (int i = 0; i < n; ++i) {
    out[i] = tv_norm(type, d[3 * i], d[3 * i + 1], d[3 * i + 2]);
    tv_norm_backward(type, d[3 * i], d[3 * i + 1], d[3 * i + 2], g[i], gd + 3 * i);
  }
}

// n opacities: safe_pow(a, 0.5) and its derivative
void hr_parsimony(int n, const float* a, float* out, float* grad) {
  for (int i = 0; i < n; ++i) { out[i] = parsimony_value(a[i]); grad[i] = parsimony_grad(a[i]); }
}

}  // extern "C"
