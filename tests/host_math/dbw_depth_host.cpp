// Host build of the per-fragment depth and its derivative (differentiable-blocksworld_b200/csrc/dbw_depth_math.cuh), for
// tests/test_depth_host.py: the forward pz of bary_from_edges and depth_frag_backward, driven per (pixel, triangle) as
// depth_backward_kernel drives them.  Test infrastructure only.
#include <cmath>
#include <cstring>

#define __device__
#define __forceinline__ inline
#define __restrict__
struct float4 { float x, y, z, w; };
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fdividef(float a, float b) { return a / b; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float4 __ldg(const float4* p) { return *p; }

#include "../../differentiable-blocksworld_b200/csrc/dbw_depth_math.cuh"

extern "C" {

// tri (9) = x, y, z of v0, v1, v2 (NDC xy, view z); p (2); out: pz, inside; g_pz -> gv9 (9)
void hd_depth(const float* tri, const float* p, int persp, int clipb, float g_pz, float* pz, int* inside, float* gv9) {
  TriGeom t;
  t.v0 = {tri[0], tri[1]}; t.v1 = {tri[3], tri[4]}; t.v2 = {tri[6], tri[7]};
  t.z0 = tri[2]; t.z1 = tri[5]; t.z2 = tri[8];
  t.face = 0; t.neighbor = -1; t.flags = 0;
  const float area = edge_nc(t.v2, t.v0, t.v1);
  t.inv_area = 1.f / __fadd_rn(area, DBW_KEPS);
  t.il01 = t.il02 = t.il12 = 1.f;
  const f2 q = {p[0], p[1]};
  const Bary b = eval_bary(q, t, persp != 0, clipb != 0);
  *pz = b.pz;
  *inside = b.inside ? 1 : 0;
  float g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  depth_frag_backward(q, t, b, persp != 0, clipb != 0, g_pz, g);
  std::memcpy(gv9, g, sizeof(g));
}

}  // extern "C"
