// Host build of the texture-atlas math (differentiable-blocksworld_b200/csrc/dbw_export_math.cuh) for
// tests/test_obj_export_host.py: the uint8 quantisation, and the whole atlas composed by running the kernel's per-thread
// body for every (CTA, thread), with the cell table built as dbw_texture_atlas_u8 (csrc/dbw_export.cu) builds it.
// Test infrastructure only.
#include <stdint.h>

#include <vector>

#define __host__
#define __device__
#define __forceinline__ inline

#include "../../include/dbw_render.h"
#include "../../differentiable-blocksworld_b200/csrc/dbw_export_math.cuh"

extern "C" {

void hm_quantise(int64_t n, const float* x, unsigned char* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = atlas_quantise(x[i]);
}

int hm_source_texel(int r, int c, int h, int w) { return atlas_source_texel(r, c, h, w); }

// jobs' maps are HOST pointers here; returns the number of CTAs the launch would have
int hm_atlas(const DbwAtlasJob* jobs, int n_jobs, int atlas_w, int cta_texels, unsigned char* atlas) {
  std::vector<AtlasCell> cells((size_t)n_jobs);
  int ctas = 0;
  for (int j = 0; j < n_jobs; ++j) {
    const DbwAtlasJob& J = jobs[j];
    cells[j] = AtlasCell{J.map, J.h, J.w, J.x0, J.y0, J.cell_w, J.cell_h, ctas, 0};
    ctas += (int)(((int64_t)J.cell_w * J.cell_h + cta_texels - 1) / cta_texels);
  }
  for (int cta = 0; cta < ctas; ++cta)
    for (int t = 0; t < cta_texels; ++t) atlas_write_texel(cells.data(), n_jobs, atlas_w, cta, t, cta_texels, atlas);
  return ctas;
}

}  // extern "C"
