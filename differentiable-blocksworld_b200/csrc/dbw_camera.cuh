// dbw_camera.cuh -- backward of the camera projection (SURVEY.md Appendix A1), shared by project_verts_backward_kernel (the
// vertex gradient) and camera_grad_kernel (the gradient of the camera poses) in dbw_render.cu, and by the per-view projection
// backward of dbw_camera_project_backward (camera_project_*_backward_kernel).
//
// Row-vector convention X_view = X_world @ R + T, then x_ndc = (fx x + px z) / d, y_ndc = (fy y + py z) / d, z_ndc = z with
// d = sign(z) max(|z|, eps) (sign(0) = +1).  Where |z| < eps the denominator is the constant +-eps: no gradient reaches z
// through it.  The header also compiles as plain C++ (tests/host_math/dbw_camera_host.cpp).
#pragma once

// d loss / d X_view of one (view, vertex), from d loss / d (x_ndc, y_ndc, z_ndc) = (gx, gy, gz).  r (3,3) and t (3) are the
// view's R and T.
__device__ __forceinline__ void dbw_project_backward(float X, float Y, float Z, const float* r, const float* t, float fx, float fy,
                                                     float px, float py, float eps, float gx, float gy, float gz, float& gxv,
                                                     float& gyv, float& gzv) {
  const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
  const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
  const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
  const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
  const bool clamped = fabsf(zv) < eps;
  const float den = sgn * fmaxf(fabsf(zv), eps);
  const float nx = fx * xv + px * zv, ny = fy * yv + py * zv;
  gxv = gx * fx / den; gyv = gy * fy / den;
  gzv = gz + (gx * px + gy * py) / den;
  if (!clamped) gzv -= (gx * nx + gy * ny) / (den * den);
}

// One (view, vertex)'s share of the intrinsics gradient gK = (g_fx, g_fy, g_px, g_py), from d loss / d (x_ndc, y_ndc) = (gx, gy):
// g_fx += gx x_view / d, g_fy += gy y_view / d, g_px += gx z_view / d, g_py += gy z_view / d.  Inside the clamp d is the constant
// +-eps, as in dbw_project_backward.
__device__ __forceinline__ void dbw_intrinsics_accumulate(float X, float Y, float Z, const float* r, const float* t, float eps,
                                                          float gx, float gy, float* gK) {
  const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
  const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
  const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
  const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
  const float den = sgn * fmaxf(fabsf(zv), eps);
  gK[0] += gx * xv / den; gK[1] += gy * yv / den;
  gK[2] += gx * zv / den; gK[3] += gy * zv / den;
}

// One vertex's share of the pose gradient: g_T[j] += g_view[j], g_R[i][j] += X_world[i] g_view[j] (R row-major).
__device__ __forceinline__ void dbw_camera_accumulate(float X, float Y, float Z, float gxv, float gyv, float gzv, float* gR, float* gT) {
  gT[0] += gxv; gT[1] += gyv; gT[2] += gzv;
  gR[0] += X * gxv; gR[1] += X * gyv; gR[2] += X * gzv;
  gR[3] += Y * gxv; gR[4] += Y * gyv; gR[5] += Y * gzv;
  gR[6] += Z * gxv; gR[7] += Z * gyv; gR[8] += Z * gzv;
}
