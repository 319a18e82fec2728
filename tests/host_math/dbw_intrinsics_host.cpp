// Host build of the per-view projection (dbw_camera_project / dbw_camera_project_backward, csrc/dbw_render.cu) for
// tests/test_intrinsics_host.py: camera_project_kernel's arithmetic, and the functions of csrc/dbw_camera.cuh that
// camera_project_verts_backward_kernel and camera_project_camera_backward_kernel inline, driven per (view, vertex) the way the
// kernels drive them.  Test infrastructure only.
#include <cmath>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_camera.cuh"

extern "C" {

// verts (V,3), R (B,3,3), T (B,3), intr (B,4) -> ndc (B,V,3)
void hi_project(int B, int V, const float* verts, const float* R, const float* T, const float* intr, float eps, float* out) {
  for (int b = 0; b < B; ++b) {
    const float* r = R + b * 9; const float* t = T + b * 3;
    const float fx = intr[b * 4], fy = intr[b * 4 + 1], px = intr[b * 4 + 2], py = intr[b * 4 + 3];
    for (int v = 0; v < V; ++v) {
      const float X = verts[v * 3], Y = verts[v * 3 + 1], Z = verts[v * 3 + 2];
      const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
      const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
      const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
      const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
      const float den = sgn * fmaxf(fabsf(zv), eps);
      float* o = out + ((size_t)b * V + v) * 3;
      o[0] = (fx * xv + px * zv) / den;
      o[1] = (fy * yv + py * zv) / den;
      o[2] = zv;
    }
  }
}

// g_ndc (B,V,3) -> g_verts (V,3), g_R (B,3,3), g_T (B,3), g_intr (B,4), all accumulated
void hi_project_backward(int B, int V, const float* verts, const float* R, const float* T, const float* intr, float eps,
                         const float* g_ndc, float* g_verts, float* g_R, float* g_T, float* g_intr) {
  for (int b = 0; b < B; ++b) {
    const float* r = R + b * 9; const float* t = T + b * 3; const float* k = intr + b * 4;
    for (int v = 0; v < V; ++v) {
      const float X = verts[v * 3], Y = verts[v * 3 + 1], Z = verts[v * 3 + 2];
      const float* g = g_ndc + ((size_t)b * V + v) * 3;
      float gxv, gyv, gzv;
      dbw_project_backward(X, Y, Z, r, t, k[0], k[1], k[2], k[3], eps, g[0], g[1], g[2], gxv, gyv, gzv);
      g_verts[v * 3] += r[0] * gxv + r[1] * gyv + r[2] * gzv;
      g_verts[v * 3 + 1] += r[3] * gxv + r[4] * gyv + r[5] * gzv;
      g_verts[v * 3 + 2] += r[6] * gxv + r[7] * gyv + r[8] * gzv;
      dbw_camera_accumulate(X, Y, Z, gxv, gyv, gzv, g_R + b * 9, g_T + b * 3);
      dbw_intrinsics_accumulate(X, Y, Z, r, t, eps, g[0], g[1], g_intr + b * 4);
    }
  }
}

}  // extern "C"
