// dbw_eval.cu -- sm_90a kernels of the DTU chamfer evaluation (see include/dbw_render.h, "DTU chamfer evaluation").
//
// Replaces the CPU pipeline of the reference's utils/dtu_eval.evaluate_mesh (an mp.Pool of per-triangle numpy calls,
// a scikit-learn kd-tree and a Python loop over every sampled point) with:
//   sampling     per triangle (lattice size) -> per (triangle, row) (sample count, binary search) -> one warp per row
//                (sample write); the caller scans between the passes
//   downsample   the greedy loop `for curr: if mask[curr]: mask[neighbours] = 0` computes the lexicographically-first
//                maximal independent set of the graph dist <= r in shuffle order; it is reproduced exactly by parallel
//                rounds on a uniform grid (cell >= r): an undecided point is kept once every earlier neighbour is
//                removed and removed once one is kept.  Decisions are final, so a round may read states written by the
//                same round; the undecided point of smallest rank is always decided, so rounds <= N
//   1-NN         rings of 4x4x4-cell blocks around each query on a grid of the targets, empty blocks skipped by their
//                cell offsets, everything farther than the best distance so far (initially max_dist) pruned
// All geometry is fp64 without FMA contraction (dbw_eval_math.cuh).
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/dbw_render.h"
#include "dbw_eval_math.cuh"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);
#define EVAL_LAUNCH_CK(name) do { dbw_count_launch_(); cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return dbw_fail_(name, _e); } while (0)
#define EVAL_CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return dbw_fail_(#call, _e); } while (0)

enum { EV_UNDECIDED = 0, EV_KEPT = 1, EV_REMOVED = 2 };

static int ev_blocks(int64_t n, int threads) {
  const int64_t b = (n + threads - 1) / threads;
  return (int)(b < (1 << 20) ? (b > 0 ? b : 1) : (1 << 20));
}

#define GRID_STRIDE(i, n) for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// last f in [0, F) with begin[f] <= r (begin non-decreasing, begin[0] = 0 <= r)
__device__ __forceinline__ int64_t ev_owner(const int64_t* __restrict__ begin, int64_t F, int64_t r) {
  int64_t lo = 0, hi = F - 1;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if (begin[mid] <= r) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------ sampling
__global__ void ev_sample_setup_kernel(const double* __restrict__ verts, const int64_t* __restrict__ faces, int64_t F,
                                       double* __restrict__ tri, int64_t* __restrict__ n_rows) {
  GRID_STRIDE(f, F) {
    double t[3][3];
    for (int k = 0; k < 3; ++k) {
      const int64_t v = faces[3 * f + k];
      for (int a = 0; a < 3; ++a) t[k][a] = verts[3 * v + a];
    }
    n_rows[f] = ev_tri_setup(t[0], t[1], t[2], tri + DBW_EVAL_TRI_STRIDE * f);
  }
}

__global__ void ev_sample_count_kernel(const double* __restrict__ tri, const int64_t* __restrict__ row_begin, int64_t F,
                                       int64_t R, int64_t* __restrict__ row_count) {
  GRID_STRIDE(r, R) {
    const int64_t f = ev_owner(row_begin, F, r);
    row_count[r] = ev_row_count(tri + DBW_EVAL_TRI_STRIDE * f, r - row_begin[f]);
  }
}

__global__ void ev_sample_write_kernel(const double* __restrict__ tri, const int64_t* __restrict__ row_begin, int64_t F,
                                       int64_t R, const int64_t* __restrict__ row_count,
                                       const int64_t* __restrict__ sample_begin, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * blockDim.x / 32;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; r < R; r += warps) {
    const int64_t f = ev_owner(row_begin, F, r), i = r - row_begin[f], cnt = row_count[r];
    const double* rec = tri + DBW_EVAL_TRI_STRIDE * f;
    double* o = out + 3 * sample_begin[r];
    for (int64_t j = lane; j < cnt; j += 32) {
      double q[3];
      ev_sample(rec, i, j, q);
      o[3 * j] = q[0]; o[3 * j + 1] = q[1]; o[3 * j + 2] = q[2];
    }
  }
}

extern "C" int dbw_eval_sample_setup(const double* verts, const int64_t* faces, int64_t n_faces, double* tri, int64_t* n_rows,
                                     void* stream) {
  if (n_faces < 0) return dbw_fail_("dbw_eval_sample_setup: bad sizes", cudaSuccess);
  if (n_faces == 0) return 0;
  if (!verts || !faces || !tri || !n_rows) return dbw_fail_("dbw_eval_sample_setup: null pointer argument", cudaSuccess);
  ev_sample_setup_kernel<<<ev_blocks(n_faces, 256), 256, 0, (cudaStream_t)stream>>>(verts, faces, n_faces, tri, n_rows);
  EVAL_LAUNCH_CK("ev_sample_setup_kernel");
  return 0;
}

extern "C" int dbw_eval_sample_count(const double* tri, const int64_t* row_begin, int64_t n_faces, int64_t n_rows_total,
                                     int64_t* row_count, void* stream) {
  if (n_faces < 0 || n_rows_total < 0) return dbw_fail_("dbw_eval_sample_count: bad sizes", cudaSuccess);
  if (n_rows_total == 0) return 0;
  if (!tri || !row_begin || !row_count || n_faces == 0) return dbw_fail_("dbw_eval_sample_count: null pointer argument", cudaSuccess);
  ev_sample_count_kernel<<<ev_blocks(n_rows_total, 256), 256, 0, (cudaStream_t)stream>>>(tri, row_begin, n_faces, n_rows_total, row_count);
  EVAL_LAUNCH_CK("ev_sample_count_kernel");
  return 0;
}

extern "C" int dbw_eval_sample_write(const double* tri, const int64_t* row_begin, int64_t n_faces, int64_t n_rows_total,
                                     const int64_t* row_count, const int64_t* sample_begin, double* out, void* stream) {
  if (n_faces < 0 || n_rows_total < 0) return dbw_fail_("dbw_eval_sample_write: bad sizes", cudaSuccess);
  if (n_rows_total == 0) return 0;
  if (!tri || !row_begin || !row_count || !sample_begin || !out || n_faces == 0)
    return dbw_fail_("dbw_eval_sample_write: null pointer argument", cudaSuccess);
  ev_sample_write_kernel<<<ev_blocks(n_rows_total * 32, 256), 256, 0, (cudaStream_t)stream>>>(tri, row_begin, n_faces, n_rows_total,
                                                                                               row_count, sample_begin, out);
  EVAL_LAUNCH_CK("ev_sample_write_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ grid keys
__global__ void ev_cell_keys_kernel(const double* __restrict__ pts, int64_t n, DbwEvalGrid g, int64_t* __restrict__ keys) {
  GRID_STRIDE(i, n) {
    int64_t c[3];
    for (int a = 0; a < 3; ++a) {
      const double p = pts[3 * i + a];
      // NaN / huge coordinates: clamp before converting
      const double t = floor(__ddiv_rn(__dadd_rn(p, -g.origin[a]), g.cell));
      c[a] = t >= 0. ? (t < (double)g.dims[a] ? (int64_t)t : g.dims[a] - 1) : 0;
    }
    const int64_t B = g.block;
    if (B <= 1) {
      keys[i] = (c[2] * g.dims[1] + c[1]) * g.dims[0] + c[0];
    } else {
      const int64_t nbx = g.dims[0] / B, nby = g.dims[1] / B;
      const int64_t blk = ((c[2] / B) * nby + c[1] / B) * nbx + c[0] / B;
      keys[i] = blk * B * B * B + ((c[2] % B) * B + c[1] % B) * B + c[0] % B;
    }
  }
}

extern "C" int dbw_eval_cell_keys(const double* points, int64_t n, const DbwEvalGrid* grid, int64_t* keys, void* stream) {
  if (!grid || n < 0) return dbw_fail_("dbw_eval_cell_keys: bad arguments", cudaSuccess);
  if (n == 0) return 0;
  if (!points || !keys) return dbw_fail_("dbw_eval_cell_keys: null pointer argument", cudaSuccess);
  const int64_t B = grid->block;
  if (!(grid->cell > 0.) || B < 1 || grid->dims[0] < 1 || grid->dims[1] < 1 || grid->dims[2] < 1 ||
      grid->dims[0] % B || grid->dims[1] % B || grid->dims[2] % B)
    return dbw_fail_("dbw_eval_cell_keys: bad grid", cudaSuccess);
  ev_cell_keys_kernel<<<ev_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(points, n, *grid, keys);
  EVAL_LAUNCH_CK("ev_cell_keys_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ radius downsample
// first index in [0, C) with keys[idx] >= k (C if none)
__device__ __forceinline__ int64_t ev_lower_bound(const int64_t* __restrict__ keys, int64_t C, int64_t k) {
  int64_t lo = 0, hi = C;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void ev_cell_ranges_kernel(const int64_t* __restrict__ ckeys, const int64_t* __restrict__ cbegin, int64_t C,
                                      DbwEvalGrid g, int32_t* __restrict__ nb, int32_t* __restrict__ ne) {
  GRID_STRIDE(c, C) {
    const int64_t key = ckeys[c], nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
    const int64_t x = key % nx, y = (key / nx) % ny, z = key / (nx * ny);
    const int64_t xl = x > 0 ? x - 1 : 0, xh = x + 1 < nx ? x + 1 : nx - 1;
    for (int dz = -1; dz <= 1; ++dz)
      for (int dy = -1; dy <= 1; ++dy) {
        const int s = 9 * (int)c + (dz + 1) * 3 + (dy + 1);
        const int64_t yy = y + dy, zz = z + dz;
        if (yy < 0 || yy >= ny || zz < 0 || zz >= nz) { nb[s] = ne[s] = 0; continue; }
        const int64_t row = (zz * ny + yy) * nx;
        nb[s] = (int32_t)cbegin[ev_lower_bound(ckeys, C, row + xl)];
        ne[s] = (int32_t)cbegin[ev_lower_bound(ckeys, C, row + xh + 1)];
      }
  }
}

extern "C" int dbw_eval_cell_ranges(const int64_t* cell_keys, const int64_t* cell_begin, int64_t n_cells, const DbwEvalGrid* grid,
                                    int32_t* nbr_begin, int32_t* nbr_end, void* stream) {
  if (!grid || n_cells < 0 || grid->block != 1 || grid->dims[0] < 1 || grid->dims[1] < 1 || grid->dims[2] < 1)
    return dbw_fail_("dbw_eval_cell_ranges: bad arguments (needs a block = 1 grid)", cudaSuccess);
  if (n_cells == 0) return 0;
  if (!cell_keys || !cell_begin || !nbr_begin || !nbr_end) return dbw_fail_("dbw_eval_cell_ranges: null pointer argument", cudaSuccess);
  ev_cell_ranges_kernel<<<ev_blocks(n_cells, 256), 256, 0, (cudaStream_t)stream>>>(cell_keys, cell_begin, n_cells, *grid,
                                                                                     nbr_begin, nbr_end);
  EVAL_LAUNCH_CK("ev_cell_ranges_kernel");
  return 0;
}

// One round over the sorted points.  `state` is read and written in place: a state read here is either stale-undecided
// (the point waits one more round) or final, so every decision is the one the sequential loop makes.
__global__ void __launch_bounds__(256) ev_mis_round_kernel(const double* __restrict__ pts, const int64_t* __restrict__ rank,
                                                           const int32_t* __restrict__ cell_of, const int32_t* __restrict__ nb,
                                                           const int32_t* __restrict__ ne, int64_t n, double r2,
                                                           uint8_t* state, unsigned long long* undecided) {
  unsigned long long left = 0;
  GRID_STRIDE(s, n) {
    if (state[s] != EV_UNDECIDED) continue;
    const double p[3] = {pts[3 * s], pts[3 * s + 1], pts[3 * s + 2]};
    const int64_t my = rank[s];
    const int c = cell_of[s];
    bool waiting = false, removed = false;
    for (int k = 0; k < 9 && !removed; ++k) {
      const int e = ne[9 * c + k];
      for (int q = nb[9 * c + k]; q < e; ++q) {
        if (rank[q] >= my) continue;
        const uint8_t st = *(volatile uint8_t*)(state + q);
        if (st == EV_REMOVED) continue;
        if (ev_dist2(p, pts + 3 * q) > r2) continue;
        if (st == EV_KEPT) { removed = true; break; }
        waiting = true;
      }
    }
    if (removed) state[s] = EV_REMOVED;
    else if (!waiting) state[s] = EV_KEPT;
    else ++left;
  }
  // one atomic per warp
  for (int o = 16; o > 0; o >>= 1) left += __shfl_down_sync(0xffffffffu, left, o);
  if ((threadIdx.x & 31) == 0 && left) atomicAdd(undecided, left);
}

__global__ void ev_mis_keep_kernel(const int64_t* __restrict__ rank, const uint8_t* __restrict__ state, int64_t n,
                                   uint8_t* __restrict__ keep) {
  GRID_STRIDE(s, n) keep[rank[s]] = state[s] == EV_KEPT;
}

static size_t ev_align(size_t x) { return (x + 255) / 256 * 256; }

extern "C" int dbw_eval_downsample_workspace_bytes(int64_t n, size_t* bytes) {
  if (n < 0 || !bytes) return dbw_fail_("dbw_eval_downsample_workspace_bytes: bad arguments", cudaSuccess);
  *bytes = 256 + ev_align((size_t)n);
  return 0;
}

extern "C" int dbw_eval_radius_downsample(const double* points, const int64_t* rank, const int32_t* cell_of,
                                          const int32_t* nbr_begin, const int32_t* nbr_end, int64_t n, double radius,
                                          int32_t max_rounds, uint8_t* keep, int32_t* rounds_out, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  if (n < 0 || !(radius >= 0.) || max_rounds < 1 || !rounds_out) return dbw_fail_("dbw_eval_radius_downsample: bad arguments", cudaSuccess);
  *rounds_out = 0;
  if (n == 0) return 0;
  if (n > INT32_MAX) return dbw_fail_("dbw_eval_radius_downsample: more than 2^31 - 1 points", cudaSuccess);
  if (!points || !rank || !cell_of || !nbr_begin || !nbr_end || !keep || !workspace)
    return dbw_fail_("dbw_eval_radius_downsample: null pointer argument", cudaSuccess);
  size_t need = 0;
  dbw_eval_downsample_workspace_bytes(n, &need);
  if (workspace_bytes < need) return dbw_fail_("dbw_eval_radius_downsample: workspace too small", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* counter = (unsigned long long*)workspace;
  uint8_t* state = (uint8_t*)workspace + 256;
  EVAL_CK(cudaMemsetAsync(state, EV_UNDECIDED, (size_t)n, st));
  const double r2 = radius * radius;
  for (int round = 1;; ++round) {
    if (round > max_rounds) {
      char msg[160];
      snprintf(msg, sizeof(msg), "dbw_eval_radius_downsample: points still undecided after max_rounds = %d rounds", max_rounds);
      return dbw_fail_(msg, cudaSuccess);
    }
    EVAL_CK(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), st));
    ev_mis_round_kernel<<<ev_blocks(n, 256), 256, 0, st>>>(points, rank, cell_of, nbr_begin, nbr_end, n, r2, state, counter);
    EVAL_LAUNCH_CK("ev_mis_round_kernel");
    unsigned long long left = 0;
    EVAL_CK(cudaMemcpyAsync(&left, counter, sizeof(left), cudaMemcpyDeviceToHost, st));
    EVAL_CK(cudaStreamSynchronize(st));
    if (left == 0) { *rounds_out = round; break; }
  }
  ev_mis_keep_kernel<<<ev_blocks(n, 256), 256, 0, st>>>(rank, state, n, keep);
  EVAL_LAUNCH_CK("ev_mis_keep_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ nearest neighbour
// squared distance from p to the axis-aligned box [lo, lo + ext)
__device__ __forceinline__ double ev_box_d2(const double* p, const double* lo, double ext) {
  double d2 = 0.;
  for (int a = 0; a < 3; ++a) {
    const double u = lo[a] - p[a], v = p[a] - (lo[a] + ext);
    const double d = u > 0. ? u : (v > 0. ? v : 0.);
    d2 += d * d;
  }
  return d2;
}

__global__ void __launch_bounds__(256) ev_nn_kernel(const double* __restrict__ qs, int64_t nq, const double* __restrict__ tg,
                                                    const int32_t* __restrict__ cell_start, DbwEvalGrid g, double max_dist,
                                                    double* __restrict__ out) {
  const int B = g.block, B3 = B * B * B;
  const double h = g.cell, H = h * B;
  const int64_t nb[3] = {g.dims[0] / B, g.dims[1] / B, g.dims[2] / B};
  const double maxd2 = __dmul_rn(max_dist, max_dist);
  GRID_STRIDE(i, nq) {
    const double p[3] = {qs[3 * i], qs[3 * i + 1], qs[3 * i + 2]};
    double best2 = maxd2;
    bool found = false;
    // whole grid farther than max_dist (or a non-finite query): nothing to search
    const double glo[3] = {g.origin[0], g.origin[1], g.origin[2]};
    double gd2 = 0.;
    for (int a = 0; a < 3; ++a) {
      const double u = glo[a] - p[a], v = p[a] - (glo[a] + (double)g.dims[a] * h);
      const double d = u > 0. ? u : (v > 0. ? v : 0.);
      gd2 += d * d;
    }
    if (gd2 < maxd2) {
      int64_t bc[3];
      for (int a = 0; a < 3; ++a) bc[a] = (int64_t)floor((p[a] - glo[a]) / H);
      int64_t kmax = 0;
      for (int a = 0; a < 3; ++a) {
        const int64_t lo = bc[a], hi = nb[a] - 1 - bc[a];
        kmax = max(kmax, max(lo, hi));
      }
      for (int64_t k = 0; k <= kmax; ++k) {
        if (k > 0) {
          // anything in ring k lies outside the box of rings < k: at least `lb` away
          double lb = 1e300;
          for (int a = 0; a < 3; ++a) {
            const double lo = glo[a] + (double)(bc[a] - k + 1) * H, hi = glo[a] + (double)(bc[a] + k) * H;
            lb = fmin(lb, fmin(p[a] - lo, hi - p[a]));
          }
          if (lb > 0. && lb * lb >= best2) break;
        }
        // the blocks of ring k that lie in the grid: the (z, y) rows clamped to it, x over the whole row on the ring's
        // faces and only its two ends inside
        const int64_t z0 = max(bc[2] - k, (int64_t)0), z1 = min(bc[2] + k, nb[2] - 1);
        const int64_t y0 = max(bc[1] - k, (int64_t)0), y1 = min(bc[1] + k, nb[1] - 1);
        const int64_t x0 = max(bc[0] - k, (int64_t)0), x1 = min(bc[0] + k, nb[0] - 1);
        for (int64_t z = z0; z <= z1; ++z) {
          for (int64_t y = y0; y <= y1; ++y) {
            const bool face = k == 0 || z == bc[2] - k || z == bc[2] + k || y == bc[1] - k || y == bc[1] + k;
            for (int64_t x = face ? x0 : bc[0] - k; x <= x1; x = (face || x >= bc[0] + k) ? x + 1 : bc[0] + k) {
              if (x < x0) continue;
              const int64_t blk = (z * nb[1] + y) * nb[0] + x;
              const int32_t b0 = cell_start[blk * B3], b1 = cell_start[(blk + 1) * B3];
              if (b0 == b1) continue;
              const double blo[3] = {glo[0] + (double)x * H, glo[1] + (double)y * H, glo[2] + (double)z * H};
              if (ev_box_d2(p, blo, H) >= best2) continue;
              int32_t c1 = b0;
              for (int sc = 0; sc < B3 && c1 < b1; ++sc) {
                const int32_t c0 = c1;
                c1 = cell_start[blk * B3 + sc + 1];
                if (c0 == c1) continue;
                const double clo[3] = {blo[0] + (double)(sc % B) * h, blo[1] + (double)((sc / B) % B) * h,
                                       blo[2] + (double)(sc / (B * B)) * h};
                if (ev_box_d2(p, clo, h) >= best2) continue;
                for (int32_t t = c0; t < c1; ++t) {
                  const double d2 = ev_dist2(p, tg + 3 * (int64_t)t);
                  if (d2 < best2) { best2 = d2; found = true; }
                }
              }
            }
          }
        }
      }
    }
    const double d = found ? __dsqrt_rn(best2) : INFINITY;
    out[i] = d < max_dist ? d : INFINITY;
  }
}

extern "C" int dbw_eval_nn_distance(const double* queries, int64_t n_queries, const double* targets, const int32_t* cell_start,
                                    const DbwEvalGrid* grid, double max_dist, double* dist, void* stream) {
  if (!grid || n_queries < 0 || !(max_dist > 0.)) return dbw_fail_("dbw_eval_nn_distance: bad arguments", cudaSuccess);
  if (n_queries == 0) return 0;
  const int64_t B = grid->block;
  if (!(grid->cell > 0.) || B < 2 || B > 8 || grid->dims[0] < B || grid->dims[1] < B || grid->dims[2] < B ||
      grid->dims[0] % B || grid->dims[1] % B || grid->dims[2] % B)
    return dbw_fail_("dbw_eval_nn_distance: bad grid (block in [2, 8], dims multiples of it)", cudaSuccess);
  if (!queries || !targets || !cell_start || !dist) return dbw_fail_("dbw_eval_nn_distance: null pointer argument", cudaSuccess);
  ev_nn_kernel<<<ev_blocks(n_queries, 256), 256, 0, (cudaStream_t)stream>>>(queries, n_queries, targets, cell_start, *grid,
                                                                             max_dist, dist);
  EVAL_LAUNCH_CK("ev_nn_kernel");
  return 0;
}
