// Host build of the per-pixel fragment list of raster_forward_kernel (differentiable-blocksworld_b200/csrc/dbw_fraglist.cuh)
// TOGETHER WITH the step that orders a tile's listed slots before they are offered: the candidates of one pixel arrive in an
// arbitrary list order (the order in which the kernel's warps won their atomics), are put into frag_order_key order the way
// the kernel does it (frag_order_rank per entry, or a scan over frag_order_slot), and are offered to fraglist_offer.  Test
// infrastructure only (tests/test_fraglist_order_host.py compares the list with the oracle's queue); built like
// dbw_math_host.cpp, with -ffp-contract=off.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#define __device__
#define __forceinline__ inline
#define __restrict__
struct float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.f / a; }
static inline float __fdividef(float a, float b) { return a / b; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline float4 __ldg(const float4* p) { return *p; }

#include "../../differentiable-blocksworld_b200/csrc/dbw_fraglist.cuh"

extern "C" {

int hm_order_key(int slot, int F) { return frag_order_key(slot, F); }
int hm_order_slot(int i, int F) { return frag_order_slot(i, F); }

// n candidates of one pixel of a view with F faces, listed in the given order (slot[i], pz[i], signed squared distance sd[i],
// neighbour slot nb[i] or -1).  mode 0: offered in list order (no ordering step); 1: the list sorted the way the fast path of
// raster_forward_kernel sorts it (every entry moves to its frag_order_rank); 2: found by a scan over frag_order_slot(i, F),
// i = 0 .. 2F-1, the order of the chunked path and of coarse_bin_kernel.  Writes the K kept slots and distances (-1 / 0
// past the end) and returns the entry count, or -1 if the ordering step lost or duplicated an entry.
int hm_list(int K, int F, int n, int mode, const float* pz, const int* slot, const float* sd, const int* nb, int* out_slot,
            float* out_sd) {
  std::vector<int> order(n);
  if (mode == 0) {
    for (int j = 0; j < n; ++j) order[j] = j;
  } else if (mode == 1) {
    std::vector<int> seen(n, 0);
    for (int j = 0; j < n; ++j) {
      const int r = frag_order_rank(slot, n, j, F);
      if (r < 0 || r >= n || seen[r]++) return -1;
      order[r] = j;
    }
  } else {
    int m = 0;
    for (int i = 0; i < 2 * F; ++i) {
      const int s = frag_order_slot(i, F);
      for (int j = 0; j < n; ++j)
        if (slot[j] == s) { if (m == n) return -1; order[m++] = j; }
    }
    if (m != n) return -1;
  }
  const int stride = 5, col = 2;               // this pixel's column inside a wider [K][stride] array, as on the device
  std::vector<float4> A((size_t)K * stride, make_float4(-7.f, -7.f, -7.f, -7.f));
  std::vector<float> V((size_t)K * stride, -7.f);
  int cnt = 0;
  for (int q = 0; q < n; ++q) {
    const int j = order[q];
    cnt = fraglist_offer(A.data() + col, V.data() + col, stride, cnt, K, pz[j], slot[j], 0, sd[j], fabsf(sd[j]), nb[j], 0.f, 0.f);
  }
  for (int k = 0; k < K; ++k) {
    const float4 e = A[(size_t)k * stride + col];
    out_slot[k] = k < cnt ? (__float_as_int(e.y) & DBW_FRAG_SLOT_MASK) : -1;
    out_sd[k] = k < cnt ? e.z : 0.f;
  }
  return cnt;
}

}  // extern "C"
