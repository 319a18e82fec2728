// Host build of the Adam update (differentiable-blocksworld_b200/csrc/dbw_optim_math.cuh), for tests/test_optim.py: the very
// functions adam_step_kernel inlines, driven per tensor the way the kernel drives them.  Test infrastructure only.
#include <cmath>
#include <cstdint>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_optim_math.cuh"

extern "C" {

// one step of one tensor of n elements; t is the step being taken (the counter after its increment)
void ho_adam_step(int64_t n, float* p, const float* g, float* m, float* v, double beta1, double beta2, double eps,
                  double weight_decay, float lr, int64_t t) {
  const DbwAdamCoef c = dbw_adam_coef(beta1, beta2, eps, weight_decay, lr, t);
  for (int64_t i = 0; i < n; ++i) dbw_adam_update(c, g[i], p[i], m[i], v[i]);
}

}  // extern "C"
