// Host build of the RANSAC math (differentiable-blocksworld_b200/csrc/dbw_ransac_math.cuh) for tests/test_baselines_host.py:
// the per-hypothesis solve, the inlier predicate over a cloud and the choice of a hypothesis, each as the kernels of
// csrc/dbw_ransac.cu run them.  Test infrastructure only.
#include <stdint.h>

#define __host__
#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_ransac_math.cuh"

extern "C" {

void hm_solve(const float* points, int n_hyp, int n_sample, const int64_t* idx, float* params) {
  for (int h = 0; h < n_hyp; ++h) ransac_solve(points, idx + (int64_t)h * n_sample, n_sample, params + 3 * h);
}

// counts[h] over the n points, and the inlier flags of hypothesis `flag_h` (if inlier is not NULL)
void hm_count(int64_t n, const float* points, int n_hyp, const float* params, float thresh, int64_t* counts, int flag_h,
              unsigned char* inlier) {
  for (int h = 0; h < n_hyp; ++h) {
    int64_t c = 0;
    for (int64_t i = 0; i < n; ++i) {
      const bool in = ransac_is_inlier(params[3 * h], params[3 * h + 1], params[3 * h + 2], points[3 * i], points[3 * i + 1],
                                       points[3 * i + 2], thresh);
      c += in;
      if (inlier && h == flag_h) inlier[i] = in;
    }
    counts[h] = c;
  }
}

int hm_select(const int64_t* counts, int n_hyp, int batch, int64_t* best_n, int* n_improvements) {
  return ransac_select(counts, n_hyp, batch, best_n, n_improvements);
}

}  // extern "C"
