// Host build of the tap -> cell mapping of cell maps (tap_to_cells in differentiable-blocksworld_b200/csrc/dbw_math.cuh), for
// tests/test_cell_maps_host.py: the bilinear taps of one (u, v) on a logical atlas, as texel indices and as cell indices.
// Test infrastructure only; built with -ffp-contract=off like dbw_math_host.cpp.
#include <cmath>
#include <cstdint>
#include <cstring>

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
static inline float4 __ldg(const float4* p) { return *p; }

#include "../../differentiable-blocksworld_b200/csrc/dbw_math.cuh"

extern "C" {

// n samples (u, v) of a map with table entry (off, H, W, cells): texel[4 n] = the four taps' texel indices in the atlas
// (first texel off_atlas), cell[4 n] = the same taps as cell indices (first cell off_cells, cells = DBW_MAP_CELLS(f, p_left)),
// w[4 n] = the tap weights.  -1: absent tap.
void hc_taps(const float* uv, int n, int off_atlas, int off_cells, int H, int W, int cells, int* texel, int* cell, float* w) {
  for (int i = 0; i < n; ++i) {
    TexTap t = tex_tap(uv[2 * i], uv[2 * i + 1], off_atlas, H, W);
    texel[4 * i] = t.i00; texel[4 * i + 1] = t.i01; texel[4 * i + 2] = t.i10; texel[4 * i + 3] = t.i11;
    w[4 * i] = t.w00; w[4 * i + 1] = t.w01; w[4 * i + 2] = t.w10; w[4 * i + 3] = t.w11;
    TexTap c = tex_tap(uv[2 * i], uv[2 * i + 1], off_cells, H, W);
    tap_to_cells(c, off_cells, H, cells);
    cell[4 * i] = c.i00; cell[4 * i + 1] = c.i01; cell[4 * i + 2] = c.i10; cell[4 * i + 3] = c.i11;
  }
}

}  // extern "C"
