// dbw_export.cu -- sm_90a texture atlas of the OBJ export: every map of a scene quantised to uint8 and composed into one
// (atlas_h, atlas_w, 3) image in one launch (see include/dbw_render.h, "Texture atlas"; the per-texel math is
// dbw_export_math.cuh).
//
// The caller's cells tile the atlas exactly, so every atlas texel is written once: map texels, gutter copies of the edge
// texels, and zeros.  Each cell gets ceil(cell_w cell_h / 256) CTAs; a CTA finds its cell by a binary search over the cells'
// first CTAs, and each of its threads writes one texel.  The cell table reaches the device through the workspace, copied
// from the caller's host table on the stream.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_export_math.cuh"

constexpr int ATLAS_THREADS = 256;

__global__ void __launch_bounds__(ATLAS_THREADS)
texture_atlas_u8_kernel(const AtlasCell* __restrict__ cells, int n_cells, int atlas_w, unsigned char* __restrict__ atlas) {
  atlas_write_texel(cells, n_cells, atlas_w, blockIdx.x, threadIdx.x, ATLAS_THREADS, atlas);
}

extern "C" size_t dbw_texture_atlas_workspace_bytes(int32_t n_jobs) {
  return n_jobs < 1 ? 0 : (size_t)n_jobs * sizeof(AtlasCell);
}

extern "C" int dbw_texture_atlas_u8(const DbwAtlasJob* jobs, int32_t n_jobs, int32_t atlas_h, int32_t atlas_w, uint8_t* atlas,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  if (!jobs || !atlas || n_jobs < 1) return dbw_fail_("dbw_texture_atlas_u8: null argument or no job", cudaSuccess);
  if (atlas_h < 1 || atlas_w < 1 || (int64_t)atlas_h * atlas_w > INT32_MAX)
    return dbw_fail_("dbw_texture_atlas_u8: atlas size must be positive and below 2^31 texels", cudaSuccess);
  if (!workspace || workspace_bytes < dbw_texture_atlas_workspace_bytes(n_jobs))
    return dbw_fail_("dbw_texture_atlas_u8: workspace too small", cudaSuccess);
  std::vector<AtlasCell> cells((size_t)n_jobs);
  int64_t covered = 0, ctas = 0;
  for (int j = 0; j < n_jobs; ++j) {
    const DbwAtlasJob& J = jobs[j];
    if (!J.map || J.h < 1 || J.w < 1) return dbw_fail_("dbw_texture_atlas_u8: a job has no map or an empty map", cudaSuccess);
    if (J.x0 < 1 || J.y0 < 1 || J.cell_w < J.w + 2 || J.cell_h < J.h + 2 || (int64_t)J.x0 - 1 + J.cell_w > atlas_w ||
        (int64_t)J.y0 - 1 + J.cell_h > atlas_h)
      return dbw_fail_("dbw_texture_atlas_u8: a job's cell does not hold its map and gutter inside the atlas", cudaSuccess);
    for (int k = 0; k < j; ++k) {
      const DbwAtlasJob& K = jobs[k];
      if (J.x0 < K.x0 + K.cell_w && K.x0 < J.x0 + J.cell_w && J.y0 < K.y0 + K.cell_h && K.y0 < J.y0 + J.cell_h)
        return dbw_fail_("dbw_texture_atlas_u8: two jobs' cells overlap", cudaSuccess);
    }
    const int64_t area = (int64_t)J.cell_w * J.cell_h;
    cells[j] = AtlasCell{J.map, J.h, J.w, J.x0, J.y0, J.cell_w, J.cell_h, (int)ctas, 0};
    covered += area;
    ctas += (area + ATLAS_THREADS - 1) / ATLAS_THREADS;
  }
  if (covered != (int64_t)atlas_h * atlas_w)
    return dbw_fail_("dbw_texture_atlas_u8: the jobs' cells do not tile the atlas", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  // pageable source: the call returns once `cells` has been staged, so the vector may go out of scope
  cudaError_t e = cudaMemcpyAsync(workspace, cells.data(), cells.size() * sizeof(AtlasCell), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return dbw_fail_("dbw_texture_atlas_u8: job table copy", e);
  texture_atlas_u8_kernel<<<(unsigned)ctas, ATLAS_THREADS, 0, s>>>((const AtlasCell*)workspace, n_jobs, atlas_w, atlas);
  dbw_count_launch_();
  e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("texture_atlas_u8_kernel", e);
}
