// dbw_knn.cu -- sm_90a exact k-nearest neighbours between batched 3-D point clouds (see include/dbw_render.h, "k-nearest
// neighbours").  Serves pytorch3d.ops.knn_points (dbw_b200/pointcloud.py), the search under the reference's chamfer
// distance, ChamferLoss and gradient_icp.
//
// Brute force, no cutoff: each thread holds Q queries and their top-K lists in registers; the CTA streams the targets of
// its batch element through shared memory in tiles of KNN_TILE points, double-buffered through registers (the next
// tile's global loads are in flight while the current one is searched; one barrier per tile).  Every thread scans the
// targets in ascending index order, so a strict `<` against the K-th entry and a (distance, index) order inside the
// list give ties to the lower index.  The squared distance is (dx*dx + dy*dy) + dz*dz in round-to-nearest fp32 without
// contraction: a numpy float32 restatement (oracle/knn.py) reproduces dists and idx bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);
#define KNN_LAUNCH_CK(name) do { dbw_count_launch_(); cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return dbw_fail_(name, _e); } while (0)

constexpr int KNN_THREADS = 128;
constexpr int KNN_TILE = 512;                        // targets per tile: 8 KB of float4, two buffers
constexpr int KNN_LOADS = KNN_TILE / KNN_THREADS;    // targets each thread stages per tile
constexpr int KNN_EMPTY = 0x7fffffff;                // index of an unfilled slot (sorts after every real one)

__device__ __forceinline__ float knn_d2(float qx, float qy, float qz, float4 p) {
  const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ int64_t knn_clamp_len(const int64_t* lengths, int n, int64_t P) {
  const int64_t l = lengths[n];
  return l < 0 ? 0 : (l > P ? P : l);
}

// Candidate j (larger than every index in the list) at distance d.  Only a distance strictly below the K-th entry gets
// in, so +inf and NaN never do; the displaced entries bubble down in (distance, index) order.
template <int K>
__device__ __forceinline__ void knn_insert(float (&bd)[K], int (&bi)[K], float d, int j) {
  if constexpr (K == 1) {
    if (d < bd[0]) { bd[0] = d; bi[0] = j; }
  } else {
    if (!(d < bd[K - 1])) return;
    float cd = d;
    int ci = j;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (cd < bd[k] || (cd == bd[k] && ci < bi[k])) {
        const float td = bd[k];
        const int ti = bi[k];
        bd[k] = cd; bi[k] = ci; cd = td; ci = ti;
      }
    }
  }
}

template <int KB, int Q>
__global__ void __launch_bounds__(KNN_THREADS) knn_forward_kernel(const float* __restrict__ p1, const float* __restrict__ p2,
                                                                  const int64_t* __restrict__ lengths1,
                                                                  const int64_t* __restrict__ lengths2, int P1, int P2, int K,
                                                                  float* __restrict__ dists, int64_t* __restrict__ idx) {
  __shared__ float4 tile[2][KNN_TILE];
  const int n = blockIdx.y, tid = threadIdx.x;
  const int len1 = (int)knn_clamp_len(lengths1, n, P1), len2 = (int)knn_clamp_len(lengths2, n, P2);
  const int i0 = blockIdx.x * (KNN_THREADS * Q) + tid;
  const int64_t row0 = (int64_t)n * P1;

  float qx[Q], qy[Q], qz[Q], bd[Q][KB];
  int bi[Q][KB];
#pragma unroll
  for (int s = 0; s < Q; ++s) {
    const int i = i0 + s * KNN_THREADS;
    const float* q = p1 + 3 * (row0 + (i < len1 ? i : 0));
    qx[s] = i < len1 ? q[0] : 0.f; qy[s] = i < len1 ? q[1] : 0.f; qz[s] = i < len1 ? q[2] : 0.f;
#pragma unroll
    for (int k = 0; k < KB; ++k) { bd[s][k] = __int_as_float(0x7f800000); bi[s][k] = KNN_EMPTY; }
  }

  // a CTA with no valid query skips the search (uniformly: no barrier is reached) and writes its padding rows
  if (blockIdx.x * (KNN_THREADS * Q) < len1) {
    const float* t2 = p2 + 3 * (int64_t)n * P2;
    const int n_tiles = (len2 + KNN_TILE - 1) / KNN_TILE;
    float4 pre[KNN_LOADS];
    auto stage = [&](int t) {
#pragma unroll
      for (int r = 0; r < KNN_LOADS; ++r) {
        const int j = t * KNN_TILE + r * KNN_THREADS + tid;
        pre[r] = j < len2 ? make_float4(t2[3 * j], t2[3 * j + 1], t2[3 * j + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
    if (n_tiles > 0) stage(0);
    for (int t = 0; t < n_tiles; ++t) {
      float4* buf = tile[t & 1];
#pragma unroll
      for (int r = 0; r < KNN_LOADS; ++r) buf[r * KNN_THREADS + tid] = pre[r];
      __syncthreads();
      if (t + 1 < n_tiles) stage(t + 1);
      const int base = t * KNN_TILE, cnt = min(KNN_TILE, len2 - base);
#pragma unroll 4
      for (int jj = 0; jj < cnt; ++jj) {
        const float4 p = buf[jj];
#pragma unroll
        for (int s = 0; s < Q; ++s) knn_insert<KB>(bd[s], bi[s], knn_d2(qx[s], qy[s], qz[s], p), base + jj);
      }
    }
  }

#pragma unroll
  for (int s = 0; s < Q; ++s) {
    const int i = i0 + s * KNN_THREADS;
    if (i >= P1) continue;
    float* od = dists + (row0 + i) * K;
    int64_t* oi = idx + (row0 + i) * K;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      if (k >= K) break;
      const bool filled = i < len1 && bi[s][k] != KNN_EMPTY;     // PyTorch3D's padding: 0 and 0
      od[k] = filled ? bd[s][k] : 0.f;
      oi[k] = filled ? (int64_t)bi[s][k] : 0;
    }
  }
}

// one thread per query row: grad_p1 without atomics, grad_p2 by RED
__global__ void __launch_bounds__(256) knn_backward_kernel(const float* __restrict__ p1, const float* __restrict__ p2,
                                                           const int64_t* __restrict__ lengths1,
                                                           const int64_t* __restrict__ lengths2, const int64_t* __restrict__ idx,
                                                           const float* __restrict__ grad_dists, int64_t N, int P1, int P2, int K,
                                                           float* __restrict__ grad_p1, float* __restrict__ grad_p2) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < N * P1; r += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(r / P1), i = (int)(r - (int64_t)n * P1);
    const int64_t len1 = knn_clamp_len(lengths1, n, P1), len2 = knn_clamp_len(lengths2, n, P2);
    if (i >= len1) continue;
    const int kmax = (int)(K < len2 ? K : len2);
    const float qx = p1[3 * r], qy = p1[3 * r + 1], qz = p1[3 * r + 2];
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int k = 0; k < kmax; ++k) {
      const int64_t j = idx[r * K + k];
      if (j < 0 || j >= len2) continue;
      const float g = 2.f * grad_dists[r * K + k];
      const float* t = p2 + 3 * ((int64_t)n * P2 + j);
      const float dx = g * (qx - t[0]), dy = g * (qy - t[1]), dz = g * (qz - t[2]);
      gx += dx; gy += dy; gz += dz;
      float* o = grad_p2 + 3 * ((int64_t)n * P2 + j);
      atomicAdd(o, -dx); atomicAdd(o + 1, -dy); atomicAdd(o + 2, -dz);
    }
    grad_p1[3 * r] += gx; grad_p1[3 * r + 1] += gy; grad_p1[3 * r + 2] += gz;
  }
}

static int knn_check_sizes(const char* what, int64_t N, int64_t P1, int64_t P2, int32_t K) {
  if (N < 0 || P1 < 0 || P2 < 0 || K < 1 || K > DBW_KNN_MAX_K) return dbw_fail_(what, cudaSuccess);
  if (N > 65535 || P1 >= KNN_EMPTY || P2 >= KNN_EMPTY) return dbw_fail_(what, cudaSuccess);
  return 0;
}

template <int KB, int Q>
static void knn_launch(const float* p1, const float* p2, const int64_t* l1, const int64_t* l2, int64_t N, int64_t P1, int64_t P2,
                       int K, float* dists, int64_t* idx, cudaStream_t st) {
  const dim3 grid((unsigned)((P1 + KNN_THREADS * Q - 1) / (KNN_THREADS * Q)), (unsigned)N);
  knn_forward_kernel<KB, Q><<<grid, KNN_THREADS, 0, st>>>(p1, p2, l1, l2, (int)P1, (int)P2, K, dists, idx);
}

extern "C" int dbw_knn_forward(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2, int64_t N,
                               int64_t P1, int64_t P2, int32_t K, float* dists, int64_t* idx, void* stream) {
  if (const int rc = knn_check_sizes("dbw_knn_forward: bad sizes (N <= 65535, P < 2^31 - 1, 1 <= K <= DBW_KNN_MAX_K)", N, P1, P2, K)) return rc;
  if (N == 0 || P1 == 0) return 0;
  if (!p1 || (P2 > 0 && !p2) || !lengths1 || !lengths2 || !dists || !idx)
    return dbw_fail_("dbw_knn_forward: null pointer argument", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  if (K <= 1) knn_launch<1, 2>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  else if (K <= 2) knn_launch<2, 2>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  else if (K <= 4) knn_launch<4, 2>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  else if (K <= 8) knn_launch<8, 2>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  else if (K <= 16) knn_launch<16, 1>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  else knn_launch<32, 1>(p1, p2, lengths1, lengths2, N, P1, P2, K, dists, idx, st);
  KNN_LAUNCH_CK("knn_forward_kernel");
  return 0;
}

extern "C" int dbw_knn_backward(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2,
                                const int64_t* idx, const float* grad_dists, int64_t N, int64_t P1, int64_t P2, int32_t K,
                                float* grad_p1, float* grad_p2, void* stream) {
  if (const int rc = knn_check_sizes("dbw_knn_backward: bad sizes (N <= 65535, P < 2^31 - 1, 1 <= K <= DBW_KNN_MAX_K)", N, P1, P2, K)) return rc;
  if (N == 0 || P1 == 0 || P2 == 0) return 0;
  if (!p1 || !p2 || !lengths1 || !lengths2 || !idx || !grad_dists || !grad_p1 || !grad_p2)
    return dbw_fail_("dbw_knn_backward: null pointer argument", cudaSuccess);
  const int64_t rows = N * P1;
  const int blocks = (int)((rows + 255) / 256 < (1 << 20) ? (rows + 255) / 256 : (1 << 20));
  knn_backward_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p1, p2, lengths1, lengths2, idx, grad_dists, N, (int)P1, (int)P2,
                                                               K, grad_p1, grad_p2);
  KNN_LAUNCH_CK("knn_backward_kernel");
  return 0;
}
