// dbw_export_math.cuh -- per-texel math of the texture-atlas kernel (dbw_export.cu): which map texel an atlas texel copies,
// and the reference's uint8 quantisation of it (save_obj, src/utils/mesh.py:392-393: (texture_map * 255.0).astype(np.uint8)).
// Plain C++ apart from the __host__ __device__ markers: tests/host_math compiles it for the CPU, with -ffp-contract=off.
//
// The atlas is cut into cells, one per map, that tile it exactly (export.atlas_layout): a cell holds its map's rectangle,
// the rectangle's 1-texel gutter (copies of its edge texels) and, right of and below the gutter, zeros up to the cell's
// extent.  Each cell gets a contiguous range of CTAs; a thread writes one texel of its CTA's cell.
#pragma once

#include <stddef.h>

#ifdef __CUDA_ARCH__
#define DBW_EXPORT_MUL(a, b) __fmul_rn((a), (b))
#else
#define DBW_EXPORT_MUL(a, b) ((a) * (b))
#endif

struct AtlasCell {
  const float* map;       // (h, w, 3)
  int h, w;
  int x0, y0;             // atlas column / row of the map's texel (0, 0); the cell starts at (x0 - 1, y0 - 1)
  int cell_w, cell_h;     // >= w + 2, h + 2
  int cta_begin;          // first CTA of the cell; ascending over the table, 0 for the first cell
  int reserved;
};

// (uint8)(x * 255.f): the float32 product rounded once (no FMA contraction), then converted toward zero.  Products outside
// [0, 255] (x outside [0, 1], where numpy's float -> uint8 cast is undefined) saturate, and NaN gives 0.
__host__ __device__ __forceinline__ unsigned char atlas_quantise(float x) {
  const float y = DBW_EXPORT_MUL(x, 255.f);
  if (!(y > 0.f)) return 0;
  if (y >= 255.f) return 255;
  return (unsigned char)(unsigned int)y;
}

// the map texel (row-major index into the (h, w) map) that texel (r, c) of a cell copies, relative to the cell's origin:
// the rectangle sits at (1, 1), its gutter replicates the nearest edge texel; -1 for the cell's zero texels
__host__ __device__ __forceinline__ int atlas_source_texel(int r, int c, int h, int w) {
  if (r > h + 1 || c > w + 1) return -1;
  const int y = r < 1 ? 0 : (r > h ? h - 1 : r - 1);
  const int x = c < 1 ? 0 : (c > w ? w - 1 : c - 1);
  return y * w + x;
}

// the cell CTA `cta` works on: the last j with cells[j].cta_begin <= cta
__host__ __device__ __forceinline__ int atlas_cell_of(const AtlasCell* cells, int n_cells, int cta) {
  int lo = 0, hi = n_cells - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cells[mid].cta_begin <= cta) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// thread `t` of CTA `cta` (cta_texels texels per CTA) writes its texel of the (., atlas_w, 3) uint8 atlas
__host__ __device__ __forceinline__ void atlas_write_texel(const AtlasCell* cells, int n_cells, int atlas_w, int cta, int t,
                                                           int cta_texels, unsigned char* atlas) {
  const AtlasCell& J = cells[atlas_cell_of(cells, n_cells, cta)];
  const long long i = (long long)(cta - J.cta_begin) * cta_texels + t;
  if (i >= (long long)J.cell_w * J.cell_h) return;
  const int r = (int)(i / J.cell_w), c = (int)(i % J.cell_w);
  unsigned char* o = atlas + 3 * ((size_t)(J.y0 - 1 + r) * atlas_w + (size_t)(J.x0 - 1 + c));
  const int s = atlas_source_texel(r, c, J.h, J.w);
  if (s < 0) {
    o[0] = 0; o[1] = 0; o[2] = 0;
    return;
  }
  const float* m = J.map + 3 * (size_t)s;
  o[0] = atlas_quantise(m[0]);
  o[1] = atlas_quantise(m[1]);
  o[2] = atlas_quantise(m[2]);
}
