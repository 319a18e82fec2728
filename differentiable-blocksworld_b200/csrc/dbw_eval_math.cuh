// dbw_eval_math.cuh -- per-triangle and per-pair fp64 math of the DTU chamfer evaluation (dbw_eval.cu).
//
// The reference's evaluate_mesh (src/utils/dtu_eval.py, after DTUeval-python) samples every triangle on a regular
// (i, j) lattice and measures point distances, all in numpy fp64.  Everything here is written with non-contracting
// intrinsics in numpy's operation order, so that the samples are bit-identical to numpy's and the distances are those
// of sqrt((dx^2 + dy^2) + dz^2):
//   v1 = t1 - t0, v2 = t2 - t0;  l = sqrt((x^2 + y^2) + z^2);  area2 = |cross(v1, v2)| (same norm)
//   thr = 0.2 * sqrt((l1 * l2) / area2);  n = floor(l / thr)
//   c0 = (i + 0.5) / max(n1, 1e-7), c1 = (j + 0.5) / max(n2, 1e-7);  inside: c0 + c1 < 1;  q = (v1 * c0 + v2 * c1) + t0
// The header also compiles as plain C++ (tests/host_math/dbw_eval_host.cpp, checked bit for bit against numpy).
#pragma once
#include <stdint.h>

#define DBW_EVAL_DENSITY 0.2
// per-triangle record: t0 (3), v1 (3), v2 (3), n1, n2, unused
#define DBW_EVAL_TRI_STRIDE 12

__device__ __forceinline__ double ev_norm3(double x, double y, double z) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

__device__ __forceinline__ double ev_dist2(const double* a, const double* b) {
  const double dx = __dadd_rn(a[0], -b[0]), dy = __dadd_rn(a[1], -b[1]), dz = __dadd_rn(a[2], -b[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Fills the record of triangle (t0, t1, t2) and returns its number of sample rows: n1 + 1 when it has any sample (the
// last row, i = n1, is always empty but costs nothing), 0 for zero-area triangles (dropped by the reference) and for
// n1 == 0 or n2 == 0 (c0 or c1 = 0.5 / 1e-7 then exceeds 1 everywhere).
__device__ __forceinline__ int64_t ev_tri_setup(const double* t0, const double* t1, const double* t2, double* rec) {
  double v1[3], v2[3];
  for (int a = 0; a < 3; ++a) { v1[a] = __dadd_rn(t1[a], -t0[a]); v2[a] = __dadd_rn(t2[a], -t0[a]); }
  const double l1 = ev_norm3(v1[0], v1[1], v1[2]), l2 = ev_norm3(v2[0], v2[1], v2[2]);
  const double cx = __dadd_rn(__dmul_rn(v1[1], v2[2]), -__dmul_rn(v1[2], v2[1]));
  const double cy = __dadd_rn(__dmul_rn(v1[2], v2[0]), -__dmul_rn(v1[0], v2[2]));
  const double cz = __dadd_rn(__dmul_rn(v1[0], v2[1]), -__dmul_rn(v1[1], v2[0]));
  const double area2 = ev_norm3(cx, cy, cz);
  double n1 = 0., n2 = 0.;
  if (area2 > 0.) {
    const double thr = __dmul_rn(DBW_EVAL_DENSITY, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
    n1 = floor(__ddiv_rn(l1, thr));
    n2 = floor(__ddiv_rn(l2, thr));
  }
  for (int a = 0; a < 3; ++a) { rec[a] = t0[a]; rec[3 + a] = v1[a]; rec[6 + a] = v2[a]; }
  rec[9] = n1; rec[10] = n2; rec[11] = 0.;
  return (n1 >= 1. && n2 >= 1.) ? (int64_t)n1 + 1 : 0;     // false for NaN as well
}

__device__ __forceinline__ double ev_c(int64_t i, double n) {
  return __ddiv_rn(__dadd_rn((double)i, 0.5), n > 1e-7 ? n : 1e-7);
}

// Samples in row i of a triangle: the j in [0, n2] with c0 + c1 < 1.  c1 grows with j and rounding is monotone, so the
// inside test is true on a prefix of the row and a binary search with the same fp64 operations finds its length exactly.
__device__ __forceinline__ int64_t ev_row_count(const double* rec, int64_t i) {
  const double c0 = ev_c(i, rec[9]);
  int64_t lo = 0, hi = (int64_t)rec[10] + 1;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (__dadd_rn(c0, ev_c(mid, rec[10])) < 1.) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ void ev_sample(const double* rec, int64_t i, int64_t j, double* q) {
  const double c0 = ev_c(i, rec[9]), c1 = ev_c(j, rec[10]);
  for (int a = 0; a < 3; ++a)
    q[a] = __dadd_rn(__dadd_rn(__dmul_rn(rec[3 + a], c0), __dmul_rn(rec[6 + a], c1)), rec[a]);
}
