// dbw_metrics.cu -- sm_90a image scores of the evaluation: per view, the summed squared error and the mean SSIM of the
// reference's SSIMLoss(padding=False) (see include/dbw_render.h, "Image scores"; the per-pixel math is dbw_metrics_math.cuh).
//
// Two launches.  image_scores_tile_kernel: one CTA per (32 x 32 tile of the valid SSIM map, view).  For each channel it stages
// the tile and its 10-pixel halo of both images in shared memory (each value read from HBM once per tile), runs the
// horizontal 11-tap pass over every staged row into the five moments, then the vertical pass and the SSIM formula per output
// pixel.  The squared error is summed over the pixels the tile owns: its 32 x 32 top-left block, and up to the image's edge
// for the last tile of a row or column, so every pixel is counted once.  Each CTA writes its two sums as doubles;
// image_scores_finish_kernel, one CTA per view, adds a view's tiles in a fixed order.  No float atomics: two calls give the
// same bits.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_metrics_math.cuh"

constexpr int MS_THREADS = 256;
constexpr int MS_WARPS = MS_THREADS / 32;
constexpr int MS_TW = 32, MS_TH = 32;                        // output pixels of one tile
constexpr int MS_IW = MS_TW + DBW_SSIM_HALO, MS_IH = MS_TH + DBW_SSIM_HALO;   // staged input pixels

struct SsimWindow { float w[DBW_SSIM_TAPS]; };

struct ScoresPlan {
  int n_views, H, W, tiles_x, n_tiles;
};

static bool make_plan(int32_t n_views, int32_t height, int32_t width, ScoresPlan* P) {
  if (n_views < 1 || n_views > 65535 || height < DBW_SSIM_TAPS || width < DBW_SSIM_TAPS) return false;
  P->n_views = n_views; P->H = height; P->W = width;
  P->tiles_x = (width - DBW_SSIM_HALO + MS_TW - 1) / MS_TW;
  P->n_tiles = P->tiles_x * ((height - DBW_SSIM_HALO + MS_TH - 1) / MS_TH);
  return true;
}

__device__ __forceinline__ double cta_sum_double(double v, double* red) {   // fixed-order CTA sum, result in thread 0
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < MS_WARPS; ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(MS_THREADS)
image_scores_tile_kernel(ScoresPlan P, const float* __restrict__ imgs, const float* __restrict__ rec, SsimWindow win,
                         double* __restrict__ partials) {
  __shared__ float sx[MS_IH][MS_IW], sy[MS_IH][MS_IW];
  __shared__ SsimMoments sh[MS_IH][MS_TW];
  __shared__ double red[2][MS_WARPS];
  const int b = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const int Ho = P.H - DBW_SSIM_HALO, Wo = P.W - DBW_SSIM_HALO;
  const int ty0 = (tile / P.tiles_x) * MS_TH, tx0 = (tile % P.tiles_x) * MS_TW;
  const int rows = min(MS_IH, P.H - ty0), cols = min(MS_IW, P.W - tx0);
  // the last tile of a column (row) owns the image's bottom (right) rows (columns) for the squared error
  const int own_r = ty0 + MS_TH >= Ho ? rows : MS_TH, own_c = tx0 + MS_TW >= Wo ? cols : MS_TW;
  float se = 0.f, ss = 0.f;
  for (int c = 0; c < 3; ++c) {
    const size_t plane = ((size_t)b * 3 + c) * P.H * P.W;
    const float* X = imgs + plane;
    const float* Y = rec + plane;
    // the previous channel's horizontal pass, the last reader of sx / sy, ended at a barrier
    for (int i = tid; i < MS_IH * MS_IW; i += MS_THREADS) {
      const int r = i / MS_IW, q = i % MS_IW;
      float a = 0.f, d = 0.f;
      if (r < rows && q < cols) {
        const size_t o = (size_t)(ty0 + r) * P.W + tx0 + q;
        a = X[o]; d = Y[o];
        if (r < own_r && q < own_c) { const float e = a - d; se += e * e; }
      }
      sx[r][q] = a; sy[r][q] = d;
    }
    __syncthreads();
    for (int i = tid; i < rows * MS_TW; i += MS_THREADS) {
      const int r = i / MS_TW, q = i % MS_TW;
      sh[r][q] = ssim_taps_line(win.w, &sx[r][q], &sy[r][q], 1);
    }
    __syncthreads();
    for (int i = tid; i < MS_TH * MS_TW; i += MS_THREADS) {
      const int r = i / MS_TW, q = i % MS_TW;
      if (ty0 + r < Ho && tx0 + q < Wo) ss += ssim_pixel(ssim_taps_moments(win.w, &sh[r][q], MS_TW));
    }
  }
  const double se_cta = cta_sum_double((double)se, red[0]);
  const double ss_cta = cta_sum_double((double)ss, red[1]);
  if (tid == 0) {
    double* out = partials + 2 * ((size_t)b * P.n_tiles + tile);
    out[0] = se_cta; out[1] = ss_cta;
  }
}

__global__ void __launch_bounds__(MS_THREADS)
image_scores_finish_kernel(ScoresPlan P, const double* __restrict__ partials, float* se_sum, float* ssim_mean) {
  __shared__ double red[2][MS_THREADS];
  const int b = blockIdx.x, tid = threadIdx.x;
  double se = 0.0, ss = 0.0;
  for (int t = tid; t < P.n_tiles; t += MS_THREADS) {
    const double* in = partials + 2 * ((size_t)b * P.n_tiles + t);
    se += in[0]; ss += in[1];
  }
  red[0][tid] = se; red[1][tid] = ss;
  __syncthreads();
  for (int h = MS_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h) { red[0][tid] += red[0][tid + h]; red[1][tid] += red[1][tid + h]; }
    __syncthreads();
  }
  if (tid == 0) {
    se_sum[b] = (float)red[0][0];
    ssim_mean[b] = (float)(red[1][0] / (3.0 * (P.H - DBW_SSIM_HALO) * (P.W - DBW_SSIM_HALO)));
  }
}

extern "C" size_t dbw_image_scores_workspace_bytes(int32_t n_views, int32_t height, int32_t width) {
  ScoresPlan P;
  if (!make_plan(n_views, height, width, &P)) return 0;
  return (size_t)P.n_views * P.n_tiles * 2 * sizeof(double);
}

extern "C" int dbw_image_scores(int32_t n_views, int32_t height, int32_t width, const float* imgs, const float* rec,
                                const float* window, float* se_sum, float* ssim_mean, void* workspace, size_t workspace_bytes,
                                void* stream) {
  ScoresPlan P;
  if (!make_plan(n_views, height, width, &P))
    return dbw_fail_("dbw_image_scores: needs 1 <= n_views <= 65535 and height, width >= 11 (the SSIM window)", cudaSuccess);
  if (!imgs || !rec || !window || !se_sum || !ssim_mean) return dbw_fail_("dbw_image_scores: null argument", cudaSuccess);
  if (!workspace || workspace_bytes < dbw_image_scores_workspace_bytes(n_views, height, width))
    return dbw_fail_("dbw_image_scores: workspace too small", cudaSuccess);
  SsimWindow win;
  for (int k = 0; k < DBW_SSIM_TAPS; ++k) win.w[k] = window[k];
  cudaStream_t s = (cudaStream_t)stream;
  double* partials = (double*)workspace;
  image_scores_tile_kernel<<<dim3(P.n_tiles, P.n_views), MS_THREADS, 0, s>>>(P, imgs, rec, win, partials);
  dbw_count_launch_();
  image_scores_finish_kernel<<<P.n_views, MS_THREADS, 0, s>>>(P, partials, se_sum, ssim_mean);
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("image_scores_tile_kernel", e);
}
