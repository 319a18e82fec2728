// dbw_ransac_math.cuh -- per-hypothesis math of the RANSAC ground filter (dbw_ransac.cu): the least-squares plane through a
// hypothesis's sample points, the inlier predicate, and the reference's rule for choosing a hypothesis (src/utils/ransac.py,
// LSLinearRegressor.fit / predict and Ransac.fit).
// Plain C++ apart from the __host__ __device__ markers: tests/host_math compiles it for the CPU, with -ffp-contract=off, and
// checks it against the float64 oracle (oracle/baselines.py), which restates the same operations in the same order.
//
// The solve is (X^T X)^-1 X^T z with X = [1, x, y], in float64: the sums of X^T X and X^T z over the sample in sample order,
// the inverse as adjugate / determinant (X^T X is symmetric, so six cofactors), then the products.  The reference computes
// ((X^T X)^-1 X^T) z in float32; the two agree to float32 rounding times the conditioning of X^T X.  A determinant of exactly
// 0 (repeated or collinear points whose float64 sums cancel exactly) gives NaN parameters; a near-singular one gives huge
// parameters.  Either way the hypothesis then counts no inlier, or almost none.
#pragma once

#include <stdint.h>

#ifdef __CUDA_ARCH__
#define DBW_RS_FADD(a, b) __fadd_rn((a), (b))
#define DBW_RS_FSUB(a, b) __fsub_rn((a), (b))
#define DBW_RS_FMUL(a, b) __fmul_rn((a), (b))
#define DBW_RS_DADD(a, b) __dadd_rn((a), (b))
#define DBW_RS_DSUB(a, b) __dsub_rn((a), (b))
#define DBW_RS_DMUL(a, b) __dmul_rn((a), (b))
#define DBW_RS_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define DBW_RS_FADD(a, b) ((a) + (b))
#define DBW_RS_FSUB(a, b) ((a) - (b))
#define DBW_RS_FMUL(a, b) ((a) * (b))
#define DBW_RS_DADD(a, b) ((a) + (b))
#define DBW_RS_DSUB(a, b) ((a) - (b))
#define DBW_RS_DMUL(a, b) ((a) * (b))
#define DBW_RS_DDIV(a, b) ((a) / (b))
#endif

// (a, b, c) of z = a + b x + c y fitted to the n points points[idx[k]] (x y z rows) in float64, rounded once to float32
__host__ __device__ __forceinline__ void ransac_solve(const float* points, const int64_t* idx, int n, float* abc) {
  double s1 = 0.0, sx = 0.0, sy = 0.0, sxx = 0.0, sxy = 0.0, syy = 0.0, sz = 0.0, sxz = 0.0, syz = 0.0;
  for (int k = 0; k < n; ++k) {
    const float* p = points + 3 * idx[k];
    const double x = p[0], y = p[1], z = p[2];
    s1 = DBW_RS_DADD(s1, 1.0);
    sx = DBW_RS_DADD(sx, x);
    sy = DBW_RS_DADD(sy, y);
    sxx = DBW_RS_DADD(sxx, DBW_RS_DMUL(x, x));
    sxy = DBW_RS_DADD(sxy, DBW_RS_DMUL(x, y));
    syy = DBW_RS_DADD(syy, DBW_RS_DMUL(y, y));
    sz = DBW_RS_DADD(sz, z);
    sxz = DBW_RS_DADD(sxz, DBW_RS_DMUL(x, z));
    syz = DBW_RS_DADD(syz, DBW_RS_DMUL(y, z));
  }
  // cofactors of [[s1, sx, sy], [sx, sxx, sxy], [sy, sxy, syy]]
  const double c00 = DBW_RS_DSUB(DBW_RS_DMUL(sxx, syy), DBW_RS_DMUL(sxy, sxy));
  const double c01 = DBW_RS_DSUB(DBW_RS_DMUL(sxy, sy), DBW_RS_DMUL(sx, syy));
  const double c02 = DBW_RS_DSUB(DBW_RS_DMUL(sx, sxy), DBW_RS_DMUL(sxx, sy));
  const double c11 = DBW_RS_DSUB(DBW_RS_DMUL(s1, syy), DBW_RS_DMUL(sy, sy));
  const double c12 = DBW_RS_DSUB(DBW_RS_DMUL(sx, sy), DBW_RS_DMUL(s1, sxy));
  const double c22 = DBW_RS_DSUB(DBW_RS_DMUL(s1, sxx), DBW_RS_DMUL(sx, sx));
  const double det = DBW_RS_DADD(DBW_RS_DADD(DBW_RS_DMUL(s1, c00), DBW_RS_DMUL(sx, c01)), DBW_RS_DMUL(sy, c02));
  if (det == 0.0) {
    const float nan = __builtin_nanf("");
    abc[0] = nan; abc[1] = nan; abc[2] = nan;
    return;
  }
  const double a = DBW_RS_DADD(DBW_RS_DADD(DBW_RS_DMUL(c00, sz), DBW_RS_DMUL(c01, sxz)), DBW_RS_DMUL(c02, syz));
  const double b = DBW_RS_DADD(DBW_RS_DADD(DBW_RS_DMUL(c01, sz), DBW_RS_DMUL(c11, sxz)), DBW_RS_DMUL(c12, syz));
  const double c = DBW_RS_DADD(DBW_RS_DADD(DBW_RS_DMUL(c02, sz), DBW_RS_DMUL(c12, sxz)), DBW_RS_DMUL(c22, syz));
  abc[0] = (float)DBW_RS_DDIV(a, det);
  abc[1] = (float)DBW_RS_DDIV(b, det);
  abc[2] = (float)DBW_RS_DDIV(c, det);
}

// the reference's predicate (y - X @ params).pow(2) < thresh in float32: r = z - ((a + b x) + c y), then r r < thresh, each
// operation rounded on its own.  NaN anywhere is no inlier.
__host__ __device__ __forceinline__ bool ransac_is_inlier(float a, float b, float c, float x, float y, float z, float thresh) {
  const float r = DBW_RS_FSUB(z, DBW_RS_FADD(DBW_RS_FADD(a, DBW_RS_FMUL(b, x)), DBW_RS_FMUL(c, y)));
  return DBW_RS_FMUL(r, r) < thresh;
}

// Ransac.fit's choice over rounds of `batch` hypotheses: a round's best is its first maximum (torch.argmax), and replaces the
// running best (0 to start with) only when strictly greater.  Returns the last best's index (best_models[-1]) or -1, with its
// count and the number of replacements.
__host__ __device__ __forceinline__ int ransac_select(const int64_t* counts, int n_hyp, int batch, int64_t* best_n,
                                                      int* n_improvements) {
  int best = -1, improvements = 0;
  int64_t best_count = 0;
  for (int r0 = 0; r0 + batch <= n_hyp; r0 += batch) {
    int arg = r0;
    for (int h = r0 + 1; h < r0 + batch; ++h)
      if (counts[h] > counts[arg]) arg = h;
    if (counts[arg] > best_count) {
      best_count = counts[arg];
      best = arg;
      ++improvements;
    }
  }
  *best_n = best_count;
  *n_improvements = improvements;
  return best;
}
