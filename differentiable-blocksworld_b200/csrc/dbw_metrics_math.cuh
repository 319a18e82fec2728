// dbw_metrics_math.cuh -- per-pixel math of the image-score kernel (dbw_metrics.cu): the 11-tap Gaussian window sums of the
// five SSIM moments and the SSIM formula of the reference's evaluation (SSIMLoss(padding=False), src/model/loss.py:119-156).
// Plain C++ apart from the __host__ __device__ markers: tests/host_math compiles it for the CPU and checks it against the
// float64 oracle (oracle/image_scores.py), built with -ffp-contract=off.
//
// The 11x11 window is the outer product of the 1-D window w, so it is applied as two 1-D passes: ssim_taps_line along a
// row of the two images, ssim_taps_moments down a column of those row sums.  The formula keeps the reference's order of
// operations (mu1_sq = mu1 * mu1, sigma1_sq = E[x^2] - mu1_sq, ...) with each product and sum rounded on its own
// (no FMA contraction), so an identical pair gives exactly 1.
#pragma once

#define DBW_SSIM_TAPS 11
#define DBW_SSIM_HALO (DBW_SSIM_TAPS - 1)
#define DBW_SSIM_C1 1e-4f                // 0.01 ** 2
#define DBW_SSIM_C2 9e-4f                // 0.03 ** 2

#ifdef __CUDA_ARCH__
#define DBW_SSIM_ADD(a, b) __fadd_rn((a), (b))
#define DBW_SSIM_SUB(a, b) __fsub_rn((a), (b))
#define DBW_SSIM_MUL(a, b) __fmul_rn((a), (b))
#define DBW_SSIM_DIV(a, b) __fdiv_rn((a), (b))
#else
#define DBW_SSIM_ADD(a, b) ((a) + (b))
#define DBW_SSIM_SUB(a, b) ((a) - (b))
#define DBW_SSIM_MUL(a, b) ((a) * (b))
#define DBW_SSIM_DIV(a, b) ((a) / (b))
#endif

struct SsimMoments { float mx, my, xx, yy, xy; };   // window sums of x, y, x*x, y*y, x*y

// sum_k w[k] * (x, y, x x, y y, x y)[k * stride], k = 0..10 in order
__host__ __device__ __forceinline__ SsimMoments ssim_taps_line(const float* w, const float* x, const float* y, int stride) {
  SsimMoments m = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < DBW_SSIM_TAPS; ++k) {
    const float a = x[k * stride], b = y[k * stride];
    m.mx += w[k] * a;
    m.my += w[k] * b;
    m.xx += w[k] * (a * a);
    m.yy += w[k] * (b * b);
    m.xy += w[k] * (a * b);
  }
  return m;
}

// sum_k w[k] * m[k * stride], k = 0..10 in order
__host__ __device__ __forceinline__ SsimMoments ssim_taps_moments(const float* w, const SsimMoments* m, int stride) {
  SsimMoments s = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < DBW_SSIM_TAPS; ++k) {
    const SsimMoments& v = m[k * stride];
    s.mx += w[k] * v.mx;
    s.my += w[k] * v.my;
    s.xx += w[k] * v.xx;
    s.yy += w[k] * v.yy;
    s.xy += w[k] * v.xy;
  }
  return s;
}

// ((2 mu1 mu2 + C1)(2 sigma12 + C2)) / ((mu1^2 + mu2^2 + C1)(sigma1^2 + sigma2^2 + C2)) from the window sums
__host__ __device__ __forceinline__ float ssim_pixel(const SsimMoments& m) {
  const float mu1_sq = DBW_SSIM_MUL(m.mx, m.mx), mu2_sq = DBW_SSIM_MUL(m.my, m.my), mu1_mu2 = DBW_SSIM_MUL(m.mx, m.my);
  const float s11 = DBW_SSIM_SUB(m.xx, mu1_sq), s22 = DBW_SSIM_SUB(m.yy, mu2_sq), s12 = DBW_SSIM_SUB(m.xy, mu1_mu2);
  const float num = DBW_SSIM_MUL(DBW_SSIM_ADD(DBW_SSIM_MUL(2.f, mu1_mu2), DBW_SSIM_C1), DBW_SSIM_ADD(DBW_SSIM_MUL(2.f, s12), DBW_SSIM_C2));
  const float den = DBW_SSIM_MUL(DBW_SSIM_ADD(DBW_SSIM_ADD(mu1_sq, mu2_sq), DBW_SSIM_C1), DBW_SSIM_ADD(DBW_SSIM_ADD(s11, s22), DBW_SSIM_C2));
  return DBW_SSIM_DIV(num, den);
}
