// Host build of the LPIPS dropout hash (differentiable-blocksworld_b200/csrc/dbw_lpips_hash.cuh), for
// tests/test_lpips_host.py: the very functions the head kernels inline.  Test infrastructure only.
#include <cstdint>

#define __device__
#define __forceinline__ inline

#include "../../differentiable-blocksworld_b200/csrc/dbw_lpips_hash.cuh"

extern "C" {

// out (B,C,H,W) uint8: 1 where the element of tap `tap` is kept, driven per element as the head kernels drive the hash
void hl_mask(uint32_t seed, uint32_t tap, int B, int C, int H, int W, uint8_t* out) {
  for (int b = 0; b < B; ++b) {
    const uint32_t h = dbw_lpips_hash_image(seed, tap, (uint32_t)b);
    for (int c = 0; c < C; ++c)
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
          *out++ = dbw_lpips_keep(h, (uint32_t)c, ((uint32_t)y << 16) | (uint32_t)x) ? 1 : 0;
  }
}

}  // extern "C"
