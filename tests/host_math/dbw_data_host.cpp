// Host build of the training-view math (differentiable-blocksworld_b200/csrc/dbw_data_math.cuh) for
// tests/test_device_data_host.py: the whole resize run as dbw_resample_u8 (csrc/dbw_data.cu) runs it -- the coefficient
// builder, then the per-pixel body of each pass Pillow would run -- and the keyed permutation.  Test infrastructure only.
#include <stdint.h>
#include <string.h>

#include <vector>

#define __host__
#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_data_math.cuh"

extern "C" {

// src (in_h, in_w, 3), dst (out_h, out_w, 3), host memory
void hm_resample(int in_h, int in_w, const unsigned char* src, int out_h, int out_w, unsigned char* dst) {
  const int kh_size = resample_ksize(in_w, out_w), kv_size = resample_ksize(in_h, out_h);
  std::vector<int32_t> bh(2 * out_w), kh((size_t)out_w * kh_size), bv(2 * out_h), kv((size_t)out_h * kv_size);
  resample_coeffs(in_w, out_w, bh.data(), kh.data());
  resample_coeffs(in_h, out_h, bv.data(), kv.data());
  const bool horizontal = out_w != in_w, vertical = out_h != in_h;
  if (!horizontal && !vertical) {
    memcpy(dst, src, (size_t)in_h * in_w * 3);
    return;
  }
  std::vector<unsigned char> tmp;
  if (horizontal && vertical && resample_vertical_first(in_h, in_w, out_h)) {
    tmp.resize((size_t)out_h * in_w * 3);
    for (int r = 0; r < out_h; ++r)
      for (int c = 0; c < in_w; ++c)
        resample_pixel(src + ((size_t)bv[2 * r] * in_w + c) * 3, 3ll * in_w, bv[2 * r + 1], &kv[(size_t)r * kv_size],
                       &tmp[((size_t)r * in_w + c) * 3]);
    for (int r = 0; r < out_h; ++r)
      for (int c = 0; c < out_w; ++c)
        resample_pixel(&tmp[((size_t)r * in_w + bh[2 * c]) * 3], 3, bh[2 * c + 1], &kh[(size_t)c * kh_size],
                       dst + ((size_t)r * out_w + c) * 3);
    return;
  }
  const unsigned char* cur = src;
  if (horizontal) {
    const int row0 = bv[0], rows = bv[2 * out_h - 2] + bv[2 * out_h - 1] - row0;
    for (int i = 0; i < out_h; ++i) bv[2 * i] -= row0;
    tmp.resize((size_t)rows * out_w * 3);
    unsigned char* out = vertical ? tmp.data() : dst;
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < out_w; ++c)
        resample_pixel(src + ((size_t)(r + row0) * in_w + bh[2 * c]) * 3, 3, bh[2 * c + 1], &kh[(size_t)c * kh_size],
                       out + ((size_t)r * out_w + c) * 3);
    cur = out;
  }
  if (vertical)
    for (int r = 0; r < out_h; ++r)
      for (int c = 0; c < out_w; ++c)
        resample_pixel(cur + ((size_t)bv[2 * r] * out_w + c) * 3, 3ll * out_w, bv[2 * r + 1], &kv[(size_t)r * kv_size],
                       dst + ((size_t)r * out_w + c) * 3);
}

void hm_u8_to_unit(int n, const unsigned char* x, float* out) {
  for (int i = 0; i < n; ++i) out[i] = u8_to_unit(x[i]);
}

// entries [0, n) of the permutation of [0, P) keyed by (seed, step, view)
void hm_permutation(uint64_t P, uint64_t seed, uint64_t step, uint64_t view, int64_t n, int64_t* out) {
  const int h = perm_half_bits(P);
  const uint64_t key = perm_key(seed, step, view);
  for (int64_t j = 0; j < n; ++j) out[j] = (int64_t)perm_index((uint64_t)j, P, h, key);
}

}  // extern "C"
