// Host build of the image-score math (differentiable-blocksworld_b200/csrc/dbw_metrics_math.cuh) for
// tests/test_image_scores_host.py: the SSIM map of one image pair, row pass then column pass as image_scores_tile_kernel
// (csrc/dbw_metrics.cu) drives them, from the very functions the kernel inlines.  Test infrastructure only.
#include <vector>

#define __host__
#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_metrics_math.cuh"

extern "C" {

// x, y (C,H,W), window (11) -> map (C,H-10,W-10)
void hm_ssim_map(int C, int H, int W, const float* x, const float* y, const float* w, float* map) {
  const int Ho = H - DBW_SSIM_HALO, Wo = W - DBW_SSIM_HALO;
  std::vector<SsimMoments> rows((size_t)H * Wo);
  for (int c = 0; c < C; ++c) {
    const float* X = x + (size_t)c * H * W;
    const float* Y = y + (size_t)c * H * W;
    for (int r = 0; r < H; ++r)
      for (int q = 0; q < Wo; ++q) rows[(size_t)r * Wo + q] = ssim_taps_line(w, X + (size_t)r * W + q, Y + (size_t)r * W + q, 1);
    for (int r = 0; r < Ho; ++r)
      for (int q = 0; q < Wo; ++q)
        map[((size_t)c * Ho + r) * Wo + q] = ssim_pixel(ssim_taps_moments(w, &rows[(size_t)r * Wo + q], Wo));
  }
}

}  // extern "C"
