// dbw_lpips_cache.cuh -- the lookup math of the LPIPS target cache (dbw_lpips.cu, dbw_lpips_forward_cached): an image's
// fingerprint, the search of the cached entries and the route of a batch.  Shared with the host build in
// tests/host_math/dbw_lpips_host.cpp and restated in numpy by tests/test_lpips_cache_host.py.
//
// fmix64(k) is MurmurHash3's 64-bit finaliser.  The fingerprint of an image of n floats (NCHW, n = 3 H W) with bit
// patterns u_i is
//   fp = sum_{i < n} fmix64((i << 32) | u_i)   (mod 2^64)
// an integer sum, so any reduction order gives the same bits.  A fingerprint only selects candidates: a hit is confirmed
// by comparing the whole image bit for bit.
#pragma once
#include <stdint.h>

__device__ __forceinline__ uint64_t dbw_lpips_fmix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

__device__ __forceinline__ uint64_t dbw_lpips_fp_term(uint64_t i, uint32_t bits) { return dbw_lpips_fmix64((i << 32) | bits); }

// the first cached entry e (in index order) with cache_fp[e] == fp and same_image(e), or -1.  On the device every thread of
// the CTA runs the loop with the same values, so same_image may synchronise the CTA.
template <class SameImage>
__device__ __forceinline__ int dbw_lpips_find(uint64_t fp, const uint64_t* cache_fp, int64_t N, SameImage same_image) {
  for (int64_t e = 0; e < N; ++e)
    if (cache_fp[e] == fp && same_image(e)) return (int)e;
  return -1;
}

// route (B, 2) int32, in place.  On entry route[b][1] is image b's hit (a cache entry, or -1 for a miss).  On exit
// route[b][0] is the hit, or -(s + 1) for the image's miss slot s (misses numbered in b order); route[s][1] is the image b
// of slot s for s < n_miss and -1 beyond.  Returns n_miss.  In place is safe: slot s is written only once image s's hit has
// been read (s <= b).
__device__ __forceinline__ int dbw_lpips_route(int32_t* route, int64_t B) {
  int n_miss = 0;
  for (int64_t b = 0; b < B; ++b) {
    const int32_t hit = route[2 * b + 1];
    if (hit >= 0) {
      route[2 * b] = hit;
    } else {
      route[2 * b] = -(n_miss + 1);
      route[2 * n_miss + 1] = (int32_t)b;
      ++n_miss;
    }
  }
  for (int64_t s = n_miss; s < B; ++s) route[2 * s + 1] = -1;
  return n_miss;
}
