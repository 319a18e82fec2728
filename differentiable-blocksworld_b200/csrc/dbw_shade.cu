// dbw_shade.cu -- sm_90a vertex normals of Phong shading (see include/dbw_render.h, "Phong shading"; the per-element math is
// dbw_shade_math.cuh).
//
// Meshes.verts_normals_packed scatters each face's normal into its three vertices with index_add, whose float atomics make the
// sums' order (and so their last bits) vary between calls.  Here the scatter is inverted once per topology into a vertex ->
// face list (dbw_vertex_face_list: integer counts, a scan, a fill, then each vertex's faces sorted), and every vertex gathers
// its faces' normals in that fixed order (dbw_vertex_normals): two calls give the same bits.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_shade_math.cuh"

#define SHADE_NT 256
#define SHADE_SCAN_NT 1024

#define SHADE_LAUNCH_CK(name) do { dbw_count_launch_(); cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return dbw_fail_(name, _e); } while (0)

// corner i = 3 f + c of faces: count[v] += 1 (count must start at 0)
__global__ void vf_count_kernel(const int* __restrict__ faces, int n_corners, int V, int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_corners) return;
  const int v = __ldg(faces + i);
  if (v >= 0 && v < V) atomicAdd(count + v, 1);
}

// exclusive prefix sum of x[0, n) in place, one CTA: each thread scans a contiguous chunk, the chunk totals are scanned in
// shared memory
__global__ void __launch_bounds__(SHADE_SCAN_NT) vf_scan_kernel(int* __restrict__ x, int n) {
  __shared__ int s_tot[SHADE_SCAN_NT];
  const int t = threadIdx.x;
  const int per = (n + SHADE_SCAN_NT - 1) / SHADE_SCAN_NT;
  const int lo = min(t * per, n), hi = min(lo + per, n);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += x[i];
  s_tot[t] = sum;
  __syncthreads();
  for (int off = 1; off < SHADE_SCAN_NT; off <<= 1) {        // inclusive Hillis-Steele scan of the chunk totals
    const int add = t >= off ? s_tot[t - off] : 0;
    __syncthreads();
    s_tot[t] += add;
    __syncthreads();
  }
  int run = t ? s_tot[t - 1] : 0;
  for (int i = lo; i < hi; ++i) { const int c = x[i]; x[i] = run; run += c; }
}

// corner 3 f + c on vertex v takes the next free entry of v's range; afterwards cursor[v] is the END of v's range
__global__ void vf_fill_kernel(const int* __restrict__ faces, int n_corners, int V, int* __restrict__ cursor, int* __restrict__ list) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_corners) return;
  const int v = __ldg(faces + i);
  if (v >= 0 && v < V) list[atomicAdd(cursor + v, 1)] = i / 3;
}

// the fill's order depends on the atomics: each vertex sorts its range (insertion sort: a vertex has a handful of faces)
__global__ void vf_sort_kernel(const int* __restrict__ vf_end, int V, int* __restrict__ list) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int lo = v ? vf_end[v - 1] : 0, hi = vf_end[v];
  for (int i = lo + 1; i < hi; ++i) {
    const int key = list[i];
    int j = i - 1;
    while (j >= lo && list[j] > key) { list[j + 1] = list[j]; --j; }
    list[j + 1] = key;
  }
}

__global__ void vertex_normals_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int V,
                                      const int* __restrict__ vf_end, const int* __restrict__ vf_faces, float* __restrict__ normals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int lo = v ? __ldg(vf_end + v - 1) : 0, hi = __ldg(vf_end + v);
  DbwVec3 n = shade_v3(0.f, 0.f, 0.f);
  for (int k = lo; k < hi; ++k) {
    const int f = __ldg(vf_faces + k);
    const DbwVec3 fn = shade_face_normal(shade_load3(verts + 3 * __ldg(faces + 3 * f)), shade_load3(verts + 3 * __ldg(faces + 3 * f + 1)),
                                         shade_load3(verts + 3 * __ldg(faces + 3 * f + 2)));
    n = shade_v3(n.x + fn.x, n.y + fn.y, n.z + fn.z);
  }
  n = shade_normalize(n);
  normals[3 * v] = n.x; normals[3 * v + 1] = n.y; normals[3 * v + 2] = n.z;
}

extern "C" int dbw_vertex_face_list(const int32_t* faces, int32_t n_faces, int32_t n_verts, int32_t* vf_end, int32_t* vf_faces,
                                    void* stream) {
  if (n_faces < 0 || n_verts < 1) return dbw_fail_("dbw_vertex_face_list: n_faces must be >= 0 and n_verts >= 1", cudaSuccess);
  if (3LL * n_faces > INT32_MAX) return dbw_fail_("dbw_vertex_face_list: too many faces", cudaSuccess);
  if (!vf_end || (n_faces && (!faces || !vf_faces))) return dbw_fail_("dbw_vertex_face_list: null pointer argument", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  const int n3 = 3 * n_faces;
  cudaError_t e = cudaMemsetAsync(vf_end, 0, (size_t)n_verts * sizeof(int32_t), st);
  if (e != cudaSuccess) return dbw_fail_("dbw_vertex_face_list: memset", e);
  if (n3) {
    vf_count_kernel<<<(n3 + SHADE_NT - 1) / SHADE_NT, SHADE_NT, 0, st>>>(faces, n3, n_verts, vf_end);
    SHADE_LAUNCH_CK("vf_count_kernel");
  }
  vf_scan_kernel<<<1, SHADE_SCAN_NT, 0, st>>>(vf_end, n_verts);
  SHADE_LAUNCH_CK("vf_scan_kernel");
  if (n3) {
    vf_fill_kernel<<<(n3 + SHADE_NT - 1) / SHADE_NT, SHADE_NT, 0, st>>>(faces, n3, n_verts, vf_end, vf_faces);
    SHADE_LAUNCH_CK("vf_fill_kernel");
  }
  vf_sort_kernel<<<(n_verts + SHADE_NT - 1) / SHADE_NT, SHADE_NT, 0, st>>>(vf_end, n_verts, vf_faces);
  SHADE_LAUNCH_CK("vf_sort_kernel");
  return 0;
}

extern "C" int dbw_vertex_normals(const float* verts, const int32_t* faces, int32_t n_verts, const int32_t* vf_end,
                                  const int32_t* vf_faces, float* normals, void* stream) {
  if (n_verts < 1) return dbw_fail_("dbw_vertex_normals: n_verts must be >= 1", cudaSuccess);
  if (!verts || !faces || !vf_end || !vf_faces || !normals) return dbw_fail_("dbw_vertex_normals: null pointer argument", cudaSuccess);
  vertex_normals_kernel<<<(n_verts + SHADE_NT - 1) / SHADE_NT, SHADE_NT, 0, (cudaStream_t)stream>>>(verts, faces, n_verts, vf_end,
                                                                                                    vf_faces, normals);
  SHADE_LAUNCH_CK("vertex_normals_kernel");
  return 0;
}
