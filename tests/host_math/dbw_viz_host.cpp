// Host build of the resolving hard render's per-pixel arithmetic (csrc/dbw_viz_math.cuh, inlined by resolve_hard_viz_kernel in
// csrc/dbw_render.cu) for tests/test_viz_views_host.py, driven per pixel the way the kernel drives it.  Test infrastructure only.
#include <cmath>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_viz_math.cuh"

extern "C" {

// samples (n,4,4) row-major -> out (n): the box filter of one channel of n frame pixels
void hv_box(int n, const float* samples, float* out) {
  for (int i = 0; i < n; ++i) {
    float acc = 0.f;
    for (int k = 0; k < 16; ++k) acc = dbw_viz_box_add(acc, samples[i * 16 + k]);
    out[i] = dbw_viz_box_mean(acc);
  }
}

void hv_composite(int n, const float* rec, const float* alpha, const float* bkg, float* out) {
  for (int i = 0; i < n; ++i) out[i] = dbw_viz_composite(rec[i], alpha[i], bkg[i]);
}

void hv_u8(int n, const float* x, unsigned char* out) {
  for (int i = 0; i < n; ++i) out[i] = dbw_viz_u8(x[i]);
}

}
