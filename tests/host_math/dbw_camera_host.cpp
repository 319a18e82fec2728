// Host build of the camera-projection backward (differentiable-blocksworld_b200/csrc/dbw_camera.cuh), for
// tests/test_camera_grad_host.py: the very functions project_verts_backward_kernel and camera_grad_kernel inline, driven per
// (view, vertex) the way the kernels drive them.  Test infrastructure only.
#include <cmath>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_camera.cuh"

extern "C" {

// verts (V,3), R (B,3,3), T (B,3), g_ndc (B,V,3) -> g_verts (V,3), g_R (B,3,3), g_T (B,3), all accumulated
void hc_project_backward(int B, int V, const float* verts, const float* R, const float* T, float fx, float fy, float px, float py,
                         float eps, const float* g_ndc, float* g_verts, float* g_R, float* g_T) {
  for (int b = 0; b < B; ++b) {
    const float* r = R + b * 9; const float* t = T + b * 3;
    for (int v = 0; v < V; ++v) {
      const float X = verts[v * 3], Y = verts[v * 3 + 1], Z = verts[v * 3 + 2];
      const float* g = g_ndc + ((size_t)b * V + v) * 3;
      float gxv, gyv, gzv;
      dbw_project_backward(X, Y, Z, r, t, fx, fy, px, py, eps, g[0], g[1], g[2], gxv, gyv, gzv);
      g_verts[v * 3] += r[0] * gxv + r[1] * gyv + r[2] * gzv;
      g_verts[v * 3 + 1] += r[3] * gxv + r[4] * gyv + r[5] * gzv;
      g_verts[v * 3 + 2] += r[6] * gxv + r[7] * gyv + r[8] * gzv;
      dbw_camera_accumulate(X, Y, Z, gxv, gyv, gzv, g_R + b * 9, g_T + b * 3);
    }
  }
}

}  // extern "C"
