// dbw_optim_math.cuh -- the per-element Adam update of adam_step_kernel (dbw_optim.cu): torch.optim.Adam's single-tensor
// path with amsgrad=False, maximize=False, in its order of operations.
//
//   g  = grad + weight_decay * p                  (only when weight_decay != 0)
//   m  = m + (1 - beta1) (g - m)
//   v  = beta2 v + (1 - beta2) g g
//   p  = p - (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
//
// The hyper-parameters arrive in double and every per-step scalar is formed in double before it is rounded to the float
// the element arithmetic uses, as torch forms them in Python: 1 - (float)0.999 is 1.3e-5 away from (float)(1 - 0.999), and
// that error would sit in every second moment.  The header also compiles as plain C++ (tests/host_math/dbw_optim_host.cpp).
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDA_ARCH__
#define DBW_OPTIM_DIV(a, b) __fdiv_rn((a), (b))          // the library is built with -prec-div=false
#else
#define DBW_OPTIM_DIV(a, b) ((a) / (b))
#endif

// What one step of one parameter tensor needs besides its elements.
struct DbwAdamCoef {
  float w1, beta2, w2, eps, weight_decay;     // 1 - beta1, beta2, 1 - beta2
  float step_size, bc2_sqrt;                  // lr / (1 - beta1^t), sqrt(1 - beta2^t)
};

// t: the step being taken (the counter after its increment), t >= 1.
__device__ __forceinline__ DbwAdamCoef dbw_adam_coef(double beta1, double beta2, double eps, double weight_decay, float lr, int64_t t) {
  DbwAdamCoef c;
  c.w1 = (float)(1.0 - beta1);
  c.beta2 = (float)beta2;
  c.w2 = (float)(1.0 - beta2);
  c.eps = (float)eps;
  c.weight_decay = (float)weight_decay;
  c.step_size = (float)((double)lr / (1.0 - pow(beta1, (double)t)));
  c.bc2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)t));
  return c;
}

__device__ __forceinline__ void dbw_adam_update(const DbwAdamCoef& c, float g, float& p, float& m, float& v) {
  if (c.weight_decay != 0.f) g = fmaf(c.weight_decay, p, g);
  m = fmaf(c.w1, g - m, m);
  v = fmaf(c.w2 * g, g, v * c.beta2);
  const float denom = DBW_OPTIM_DIV(sqrtf(v), c.bc2_sqrt) + c.eps;
  p = fmaf(-c.step_size, DBW_OPTIM_DIV(m, denom), p);
}
