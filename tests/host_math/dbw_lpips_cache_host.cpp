// Host build of the LPIPS target-cache lookup math (differentiable-blocksworld_b200/csrc/dbw_lpips_cache.cuh), for
// tests/test_lpips_cache_host.py: the very functions lpips_fingerprint_kernel, lpips_lookup_kernel and lpips_route_kernel
// inline.  Test infrastructure only.
#include <cstdint>
#include <cstring>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_lpips_cache.cuh"

extern "C" {

// fp[b] = the fingerprint of image b of x (B images of n floats)
void hc_fingerprint(const float* x, int64_t n, int64_t B, uint64_t* fp) {
  for (int64_t b = 0; b < B; ++b) {
    const uint32_t* u = reinterpret_cast<const uint32_t*>(x) + b * n;
    uint64_t s = 0;
    for (int64_t i = 0; i < n; ++i) s += dbw_lpips_fp_term((uint64_t)i, u[i]);
    fp[b] = s;
  }
}

// the lookup of B query images (fingerprints q_fp, n floats each) in a cache of N (fingerprints c_fp), then the route
// (B, 2); returns n_miss.  The fingerprints are arguments, so a test can force collisions.
int hc_lookup(const uint64_t* q_fp, const float* q_img, int64_t B, const uint64_t* c_fp, const float* c_img, int64_t N, int64_t n,
              int32_t* route) {
  for (int64_t b = 0; b < B; ++b) {
    auto same_image = [&](int64_t e) { return std::memcmp(q_img + b * n, c_img + e * n, (size_t)n * 4) == 0; };
    route[2 * b + 1] = dbw_lpips_find(q_fp[b], c_fp, N, same_image);
  }
  return dbw_lpips_route(route, B);
}

}  // extern "C"
