// dbw_ransac.cu -- sm_90a RANSAC ground filter of the baseline preprocessing (see include/dbw_render.h, "RANSAC ground
// filter"; the per-hypothesis math is dbw_ransac_math.cuh).
//
// The cloud is cut into tiles of RS_TILE points, one CTA each.  Counting reads each point once into registers and tests
// every hypothesis, held in shared memory, against it: per hypothesis a warp sums its lanes' inliers and adds them to the
// CTA's shared counter (integer adds, so the order does not matter).  The CTA writes its counts as partials[h][tile]; the
// last CTA to finish (a ticket in the workspace) sums every tile's partials per hypothesis.  Nothing of size n_hyp x n_points
// exists.  The filter is a three-pass order-preserving compaction over the same tiles: kept counts per tile, one CTA's
// exclusive scan of them, then each tile scans its threads' counts and writes its kept points at their offsets.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_ransac_math.cuh"

constexpr int RS_THREADS = 256;
constexpr int RS_PTS = 4;                          // points per thread, held in registers
constexpr int RS_TILE = RS_THREADS * RS_PTS;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_SCAN_THREADS = 1024;
constexpr size_t RS_TICKET_BYTES = 256;

static int64_t rs_tiles(int64_t n_points) { return (n_points + RS_TILE - 1) / RS_TILE; }

// the k-th point of thread t in a tile: consecutive points per thread, so that thread order then k is input order
__device__ __forceinline__ int64_t rs_point(int64_t tile, int t, int k) { return tile * RS_TILE + (int64_t)t * RS_PTS + k; }

__device__ __forceinline__ void rs_load(const float* __restrict__ points, int64_t n, int64_t tile, int t, float* x, float* y,
                                        float* z) {
#pragma unroll
  for (int k = 0; k < RS_PTS; ++k) {
    const int64_t i = rs_point(tile, t, k);
    if (i < n) {
      x[k] = points[3 * i]; y[k] = points[3 * i + 1]; z[k] = points[3 * i + 2];
    } else {
      x[k] = y[k] = z[k] = __int_as_float(0x7fc00000);        // NaN: no inlier, and never written by the filter
    }
  }
}

__global__ void ransac_fit_kernel(const float* __restrict__ points, int n_hyp, int n_sample, const int64_t* __restrict__ idx,
                                  float* __restrict__ params) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < n_hyp) ransac_solve(points, idx + (int64_t)h * n_sample, n_sample, params + 3 * h);
}

__global__ void __launch_bounds__(RS_THREADS)
ransac_count_kernel(const float* __restrict__ points, int64_t n, int n_hyp, const float* __restrict__ params, float thresh,
                    int* __restrict__ partials, unsigned int* __restrict__ ticket, int64_t* __restrict__ counts) {
  extern __shared__ float s_params[];                          // (n_hyp, 3), then n_hyp int counters
  int* s_count = (int*)(s_params + 3 * n_hyp);
  __shared__ bool s_last;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t tiles = gridDim.x;
  for (int j = t; j < 3 * n_hyp; j += RS_THREADS) s_params[j] = params[j];
  for (int h = t; h < n_hyp; h += RS_THREADS) s_count[h] = 0;
  float x[RS_PTS], y[RS_PTS], z[RS_PTS];
  rs_load(points, n, blockIdx.x, t, x, y, z);
  __syncthreads();
  for (int h = 0; h < n_hyp; ++h) {
    const float a = s_params[3 * h], b = s_params[3 * h + 1], c = s_params[3 * h + 2];
    unsigned int m = 0;
#pragma unroll
    for (int k = 0; k < RS_PTS; ++k) m += ransac_is_inlier(a, b, c, x[k], y[k], z[k], thresh) ? 1u : 0u;
    m = __reduce_add_sync(0xffffffffu, m);
    if (lane == 0 && m) atomicAdd(&s_count[h], (int)m);
  }
  __syncthreads();
  for (int h = t; h < n_hyp; h += RS_THREADS) partials[(int64_t)h * tiles + blockIdx.x] = s_count[h];
  __threadfence();
  __syncthreads();
  if (t == 0) s_last = atomicAdd(ticket, 1u) == (unsigned int)(tiles - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int h = warp; h < n_hyp; h += RS_WARPS) {                // one warp per hypothesis, lanes over the tiles
    long long s = 0;
    for (int64_t b = lane; b < tiles; b += 32) s += __ldcg(partials + (int64_t)h * tiles + b);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) counts[h] = s;
  }
}

__global__ void ransac_select_kernel(int n_hyp, int batch, const int64_t* __restrict__ counts, const float* __restrict__ params,
                                     DbwRansacResult* __restrict__ result) {
  DbwRansacResult r;
  int improvements = 0;
  int64_t best_n = 0;
  const int best = ransac_select(counts, n_hyp, batch, &best_n, &improvements);
  const float nan = __int_as_float(0x7fc00000);
  for (int j = 0; j < 3; ++j) r.params[j] = best < 0 ? nan : params[3 * best + j];
  r.hypothesis = best;
  r.n_inliers = best_n;
  r.n_improvements = improvements;
  r.reserved = 0;
  *result = r;
}

// the tile's kept flags (bit k of the return value: point k of thread t is kept)
__device__ __forceinline__ unsigned int rs_kept_bits(const float* __restrict__ points, int64_t n, int64_t tile, int t,
                                                     const DbwRansacResult* __restrict__ result, float thresh) {
  float x[RS_PTS], y[RS_PTS], z[RS_PTS];
  rs_load(points, n, tile, t, x, y, z);
  const bool none = result->hypothesis < 0;
  const float a = result->params[0], b = result->params[1], c = result->params[2];
  unsigned int bits = 0;
#pragma unroll
  for (int k = 0; k < RS_PTS; ++k)
    if (rs_point(tile, t, k) < n && (none || !ransac_is_inlier(a, b, c, x[k], y[k], z[k], thresh))) bits |= 1u << k;
  return bits;
}

__global__ void __launch_bounds__(RS_THREADS)
ransac_filter_count_kernel(const float* __restrict__ points, int64_t n, const DbwRansacResult* __restrict__ result, float thresh,
                           int64_t* __restrict__ tile_kept) {
  __shared__ int s_warp[RS_WARPS];
  const int t = threadIdx.x;
  const int m = __reduce_add_sync(0xffffffffu, (unsigned int)__popc(rs_kept_bits(points, n, blockIdx.x, t, result, thresh)));
  if ((t & 31) == 0) s_warp[t >> 5] = m;
  __syncthreads();
  if (t == 0) {
    int64_t s = 0;
    for (int w = 0; w < RS_WARPS; ++w) s += s_warp[w];
    tile_kept[blockIdx.x] = s;
  }
}

// exclusive scan of the tiles' kept counts in one CTA, chunk by chunk; the total goes to *n_kept
__global__ void __launch_bounds__(RS_SCAN_THREADS)
ransac_scan_kernel(const int64_t* __restrict__ tile_kept, int64_t tiles, int64_t* __restrict__ tile_offset,
                   int64_t* __restrict__ n_kept) {
  __shared__ long long s_warp[RS_SCAN_THREADS / 32];
  __shared__ long long s_carry;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t == 0) s_carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < tiles; base += RS_SCAN_THREADS) {
    const int64_t i = base + t;
    const long long v = i < tiles ? tile_kept[i] : 0;
    long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      long long w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += u;
      }
      s_warp[lane] = w;                                         // inclusive over warps
    }
    __syncthreads();
    const long long before = s_carry + (warp ? s_warp[warp - 1] : 0) + inc - v;
    if (i < tiles) tile_offset[i] = before;
    __syncthreads();
    if (t == RS_SCAN_THREADS - 1) s_carry = before + v;
    __syncthreads();
  }
  if (t == 0) *n_kept = s_carry;
}

__global__ void __launch_bounds__(RS_THREADS)
ransac_filter_write_kernel(const float* __restrict__ points, int64_t n, const DbwRansacResult* __restrict__ result, float thresh,
                           const int64_t* __restrict__ tile_offset, float* __restrict__ kept, uint8_t* __restrict__ inlier) {
  __shared__ int s_warp[RS_WARPS];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const unsigned int bits = rs_kept_bits(points, n, blockIdx.x, t, result, thresh);
  const int cnt = __popc(bits);
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int before = inc - cnt;
  for (int w = 0; w < warp; ++w) before += s_warp[w];
  int64_t o = tile_offset[blockIdx.x] + before;
#pragma unroll
  for (int k = 0; k < RS_PTS; ++k) {
    const int64_t i = rs_point(blockIdx.x, t, k);
    if (i >= n) break;
    const bool keep = (bits >> k) & 1u;
    if (inlier) inlier[i] = keep ? 0 : 1;
    if (keep && kept) {
      kept[3 * o] = points[3 * i]; kept[3 * o + 1] = points[3 * i + 1]; kept[3 * o + 2] = points[3 * i + 2];
    }
    o += keep;
  }
}

static bool rs_points_ok(int64_t n_points) { return n_points >= 1 && n_points <= INT32_MAX; }

extern "C" int dbw_ransac_workspace_bytes(int64_t n_points, int32_t n_hyp, size_t* bytes) {
  if (!bytes) return dbw_fail_("dbw_ransac_workspace_bytes: null argument", cudaSuccess);
  if (!rs_points_ok(n_points) || n_hyp < 1 || n_hyp > DBW_RANSAC_MAX_HYPOTHESES)
    return dbw_fail_("dbw_ransac_workspace_bytes: n_points must be in [1, 2^31 - 1] and n_hyp in [1, DBW_RANSAC_MAX_HYPOTHESES]",
                     cudaSuccess);
  const size_t tiles = (size_t)rs_tiles(n_points);
  const size_t count = (size_t)n_hyp * tiles * sizeof(int), filter = 2 * tiles * sizeof(int64_t);
  *bytes = RS_TICKET_BYTES + (count > filter ? count : filter);
  return 0;
}

extern "C" int dbw_ransac_fit(int64_t n_points, const float* points, int32_t n_hyp, int32_t n_sample, const int64_t* sample_idx,
                              float* params, void* stream) {
  if (!points || !sample_idx || !params) return dbw_fail_("dbw_ransac_fit: null argument", cudaSuccess);
  if (!rs_points_ok(n_points) || n_hyp < 1 || n_hyp > DBW_RANSAC_MAX_HYPOTHESES || n_sample < 3 || n_sample > DBW_RANSAC_MAX_SAMPLE)
    return dbw_fail_("dbw_ransac_fit: n_points, n_hyp or n_sample out of range", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  ransac_fit_kernel<<<(n_hyp + 127) / 128, 128, 0, s>>>(points, n_hyp, n_sample, sample_idx, params);
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("ransac_fit_kernel", e);
}

extern "C" int dbw_ransac_count(int64_t n_points, const float* points, int32_t n_hyp, const float* params, float thresh,
                                int64_t* counts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!points || !params || !counts) return dbw_fail_("dbw_ransac_count: null argument", cudaSuccess);
  size_t need = 0;
  if (dbw_ransac_workspace_bytes(n_points, n_hyp, &need)) return 1;
  if (!workspace || workspace_bytes < need) return dbw_fail_("dbw_ransac_count: workspace too small", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  unsigned int* ticket = (unsigned int*)workspace;
  cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), s);
  if (e != cudaSuccess) return dbw_fail_("dbw_ransac_count: ticket reset", e);
  const size_t smem = (size_t)n_hyp * (3 * sizeof(float) + sizeof(int));
  if (smem > 48 * 1024) {
    e = cudaFuncSetAttribute(ransac_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return dbw_fail_("dbw_ransac_count: shared memory attribute", e);
  }
  ransac_count_kernel<<<(unsigned)rs_tiles(n_points), RS_THREADS, smem, s>>>(
      points, n_points, n_hyp, params, thresh, (int*)((char*)workspace + RS_TICKET_BYTES), ticket, counts);
  dbw_count_launch_();
  e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("ransac_count_kernel", e);
}

extern "C" int dbw_ransac_select(int32_t n_hyp, int32_t batch_size, const int64_t* counts, const float* params,
                                 DbwRansacResult* result, void* stream) {
  if (!counts || !params || !result) return dbw_fail_("dbw_ransac_select: null argument", cudaSuccess);
  if (n_hyp < 1 || n_hyp > DBW_RANSAC_MAX_HYPOTHESES || batch_size < 1 || n_hyp % batch_size)
    return dbw_fail_("dbw_ransac_select: n_hyp must be in [1, DBW_RANSAC_MAX_HYPOTHESES] and a multiple of batch_size",
                     cudaSuccess);
  ransac_select_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(n_hyp, batch_size, counts, params, result);
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("ransac_select_kernel", e);
}

extern "C" int dbw_ransac_filter(int64_t n_points, const float* points, const DbwRansacResult* result, float thresh, float* kept,
                                 uint8_t* inlier, int64_t* n_kept, void* workspace, size_t workspace_bytes, void* stream) {
  if (!points || !result || !n_kept) return dbw_fail_("dbw_ransac_filter: null argument", cudaSuccess);
  size_t need = 0;
  if (dbw_ransac_workspace_bytes(n_points, 1, &need)) return 1;
  if (!workspace || workspace_bytes < need) return dbw_fail_("dbw_ransac_filter: workspace too small", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t tiles = rs_tiles(n_points);
  int64_t* tile_kept = (int64_t*)((char*)workspace + RS_TICKET_BYTES);
  int64_t* tile_offset = tile_kept + tiles;
  ransac_filter_count_kernel<<<(unsigned)tiles, RS_THREADS, 0, s>>>(points, n_points, result, thresh, tile_kept);
  dbw_count_launch_();
  ransac_scan_kernel<<<1, RS_SCAN_THREADS, 0, s>>>(tile_kept, tiles, tile_offset, n_kept);
  dbw_count_launch_();
  ransac_filter_write_kernel<<<(unsigned)tiles, RS_THREADS, 0, s>>>(points, n_points, result, thresh, tile_offset, kept, inlier);
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("ransac_filter kernels", e);
}
