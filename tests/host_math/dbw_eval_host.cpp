// Host build of the per-triangle sampling math of the DTU chamfer evaluation (differentiable-blocksworld_b200/csrc/
// dbw_eval_math.cuh), for tests/test_dtu_eval_host.py: the very functions the sampling kernels inline, driven per
// (triangle, row, j) the way dbw_eval.cu drives them.  Test infrastructure only; built with -ffp-contract=off so that the
// explicitly rounded intrinsics (__dmul_rn, ...) are plain IEEE operations, as on the device.
#include <cmath>
#include <cstdint>

#define __device__
#define __forceinline__ inline
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
using std::floor;

#include "../../differentiable-blocksworld_b200/csrc/dbw_eval_math.cuh"

extern "C" {

// tv (F,3,3) triangle vertices -> rec (F,12) records, rows (F), and the samples in the reference's order (at most cap
// written to out (cap,3)); returns the number of samples
int64_t he_sample(const double* tv, int64_t F, double* rec, int64_t* rows, double* out, int64_t cap) {
  int64_t s = 0;
  for (int64_t f = 0; f < F; ++f) {
    double* r = rec + DBW_EVAL_TRI_STRIDE * f;
    rows[f] = ev_tri_setup(tv + 9 * f, tv + 9 * f + 3, tv + 9 * f + 6, r);
    for (int64_t i = 0; i < rows[f]; ++i) {
      const int64_t cnt = ev_row_count(r, i);
      for (int64_t j = 0; j < cnt; ++j, ++s)
        if (s < cap) ev_sample(r, i, j, out + 3 * s);
    }
  }
  return s;
}

}  // extern "C"
