// dbw_data_math.cuh -- per-element math of the training-view kernels (dbw_data.cu): Pillow's bilinear resampler on uint8 RGB,
// ToTensor's uint8 -> float division, and the keyed permutation behind the ground-truth point subsample.
// Plain C++ apart from the __host__ __device__ markers: tests/host_math compiles it for the CPU, with -ffp-contract=off.
//
// The resampler is Pillow's convolution resampler (libImaging/Resample.c, Image.resize(size, Image.BILINEAR), what
// torchvision's Resize runs on a PIL image).  Per output column (row) the filter covers the input range
// [center - support, center + support), support = 1 x max(in / out, 1); its triangle weights are normalised in double and
// stored as 22-bit fixed point, rounded away from zero.  Each output channel is (2^21 + sum pixel * coefficient) >> 22,
// clipped to [0, 255].  The horizontal pass writes a uint8 intermediate covering only the input rows the vertical pass
// reads, then the vertical pass runs; a pass whose size does not change is skipped.  Image.resize runs a tall image's vertical
// pass first (resample_vertical_first), with the full-width intermediate.
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDA_ARCH__
#define DBW_DATA_DIV(a, b) __fdiv_rn((a), (b))
#else
#define DBW_DATA_DIV(a, b) ((a) / (b))
#endif

constexpr int RESAMPLE_PRECISION_BITS = 32 - 8 - 2;

// coefficients per output pixel along one axis: Pillow's ksize
inline int resample_ksize(int in_size, int out_size) {
  double filterscale = (double)(float)in_size / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  return (int)ceil(1.0 * filterscale) * 2 + 1;
}

// Image.resize's branch for tall images (height > 100 x width, shrinking in height): the image is resized to (in_w, out_h)
// first, then to (out_w, out_h), so the vertical pass runs before the horizontal one
inline bool resample_vertical_first(int in_h, int in_w, int out_h) { return in_h > 100ll * in_w && out_h < in_h; }

// Pillow's bilinear_filter at tap x of an output pixel centred at `center`
inline double resample_weight(int x, int xmin, double center, double ss) {
  double t = (x + xmin - center + 0.5) * ss;
  if (t < 0.0) t = -t;
  return t < 1.0 ? 1.0 - t : 0.0;
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for box (0, in_size) with the bilinear filter (support 1), in its order
// of double operations.  bounds[2 o] is the first input index of output o, bounds[2 o + 1] the number of taps;
// kk[o * ksize + t] the fixed-point coefficient of tap t (0 past the taps).  Returns ksize.
inline int resample_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk) {
  const double scale = (double)((float)in_size - 0.f) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 1.0 * filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = 0.f + (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    // the weights are computed twice, identically: once for their sum, once to normalise and store
    for (int x = 0; x < xmax; ++x) ww += resample_weight(x, xmin, center, ss);
    for (int x = 0; x < ksize; ++x) {
      double v = 0.0;
      if (x < xmax) {
        v = resample_weight(x, xmin, center, ss);
        if (ww != 0.0) v /= ww;
      }
      kk[xx * ksize + x] = v < 0 ? (int32_t)(-0.5 + v * (1 << RESAMPLE_PRECISION_BITS))
                                 : (int32_t)(0.5 + v * (1 << RESAMPLE_PRECISION_BITS));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
  return ksize;
}

__host__ __device__ __forceinline__ unsigned char resample_clip8(int32_t acc) {
  const int32_t v = acc >> RESAMPLE_PRECISION_BITS;
  return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// one output pixel of a pass: `taps` input pixels from `src`, `stride` bytes apart, weighted by `k`
__host__ __device__ __forceinline__ void resample_pixel(const unsigned char* src, long long stride, int taps, const int32_t* k,
                                                        unsigned char* out) {
  int32_t s0 = 1 << (RESAMPLE_PRECISION_BITS - 1), s1 = s0, s2 = s0;
  for (int t = 0; t < taps; ++t) {
    const unsigned char* p = src + t * stride;
    const int32_t c = k[t];
    s0 += (int32_t)p[0] * c;
    s1 += (int32_t)p[1] * c;
    s2 += (int32_t)p[2] * c;
  }
  out[0] = resample_clip8(s0);
  out[1] = resample_clip8(s1);
  out[2] = resample_clip8(s2);
}

// ToTensor's x / 255 in float32, correctly rounded (not a multiply by the reciprocal)
__host__ __device__ __forceinline__ float u8_to_unit(unsigned char x) { return DBW_DATA_DIV((float)x, 255.f); }

// ------------------------------------------------------------------ keyed permutation of [0, P)
// A balanced Feistel network on 2 h bits (the least h >= 1 with 4^h >= P) is a bijection of [0, 4^h); cycle-walking (apply it
// again until the value falls below P) restricts it to a bijection of [0, P).  4^h < 4 P, so a walk takes under 4 rounds
// of the network on average.
constexpr int PERM_ROUNDS = 6;

__host__ __device__ __forceinline__ uint64_t perm_mix64(uint64_t z) {       // splitmix64's finaliser
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// the key of view `view` in step `step` of a stream seeded with `seed`
__host__ __device__ __forceinline__ uint64_t perm_key(uint64_t seed, uint64_t step, uint64_t view) {
  return perm_mix64(perm_mix64(perm_mix64(seed) ^ step) ^ view);
}

__host__ __device__ __forceinline__ int perm_half_bits(uint64_t P) {
  int h = 1;
  while (h < 32 && (1ull << (2 * h)) < P) ++h;
  return h;
}

__host__ __device__ __forceinline__ uint64_t perm_feistel(uint64_t x, int h, uint64_t key) {
  const uint64_t mask = (1ull << h) - 1;
  uint64_t l = x >> h, r = x & mask;
  for (int i = 0; i < PERM_ROUNDS; ++i) {
    const uint64_t f = perm_mix64(key + (uint64_t)i * 0x9e3779b97f4a7c15ull + r) & mask;
    const uint64_t t = l ^ f;
    l = r;
    r = t;
  }
  return (l << h) | r;
}

// entry j of the keyed permutation of [0, P), 0 <= j < P
__host__ __device__ __forceinline__ uint64_t perm_index(uint64_t j, uint64_t P, int h, uint64_t key) {
  uint64_t x = j;
  do {
    x = perm_feistel(x, h, key);
  } while (x >= P);
  return x;
}
