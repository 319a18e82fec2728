// dbw_lpips_hash.cuh -- the counter-based hash behind the LPIPS lin-layer dropout mask (dbw_lpips.cu).  Shared with the
// host build in tests/host_math/dbw_lpips_host.cpp and restated in numpy by oracle/lpips.py.
//
// fmix(h) is MurmurHash3's 32-bit finaliser.  For a call's seed s, tap k (0..4), image b, channel c and pixel (y, x) of
// the tap:
//   h_img = fmix(fmix(s + 0x9e3779b9 * (k + 1)) ^ b)
//   h     = fmix(fmix(h_img ^ c) ^ ((y << 16) | x))
// and the element is kept (then scaled by 2) when h < 2^31.  All arithmetic is uint32, wrapping.
#pragma once
#include <stdint.h>

__device__ __forceinline__ uint32_t dbw_lpips_fmix(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

__device__ __forceinline__ uint32_t dbw_lpips_hash_image(uint32_t seed, uint32_t tap, uint32_t image) {
  return dbw_lpips_fmix(dbw_lpips_fmix(seed + 0x9e3779b9u * (tap + 1u)) ^ image);
}

__device__ __forceinline__ bool dbw_lpips_keep(uint32_t h_img, uint32_t channel, uint32_t yx) {
  return dbw_lpips_fmix(dbw_lpips_fmix(h_img ^ channel) ^ yx) < 0x80000000u;
}
