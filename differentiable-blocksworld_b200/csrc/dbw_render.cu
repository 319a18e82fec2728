// dbw_render.cu -- sm_90a kernels + C-ABI of the differentiable primitive renderer (see include/dbw_render.h).
//
// Replaces, for the reference's render hot path (src/model/renderer.py:84-98, 219-273):
//   PerspectiveCameras/MeshRasterizer.transform, clip_faces, _C.rasterize_meshes{,_backward},
//   interpolate_face_attributes, F.grid_sample on the (B*K)-replicated atlas, and the ~15 eager kernels of
//   layered_rgb_blend -- with  project -> face setup (z-clip) -> ONE fused raster+shade+blend kernel per pass,
//   and the mirror-image backward.  No fragments tensors (pix_to_face/zbuf/bary/dists, 28 B/px/K) are ever written:
//   the forward keeps the per-pixel top-K in registers and stores only K int32 slot ids per pixel for the backward.
//
// Layout in HBM (all fp32 / int32):
//   verts_ndc  (B,V,3)            projected vertices (x_ndc, y_ndc, z_view)
//   bbox       (B,2F) float4      blur-expanded NDC bbox of each face slot (xmin,xmax,ymin,ymax); xmin=+inf: empty
//   rec        (B,2F,4) float4    v0xy v1xy | v2xy z0 z1 | z2 face neighbor flags | 1/area, 1/|e01|^2, 1/|e02|^2, 1/|e12|^2
//   rec2       (B,2F,2) float4    u0 v0 u1 v1 | u2 v2 map_id -   (static per face, replicated per view: one load level after the
//                                 face id); the map table itself (first texel, H, W of each map) is staged in shared memory
//   maps4      (sum H*W) float4   the caller's (H,W,3) maps re-packed as RGB+pad texels: one 128-bit load per bilinear tap
//   conv       (B,2F,9)           barycentric conversion (clipped -> original face), only for clipped slots
//   slots [0,F) hold each face's (first) triangle, slots [F,2F) the second triangle of a z-clipped quad.
//   frag       (B,K,H,W,2) float4 optional saved fragment state (u, v, signed dist, r | g, b, -, -): two 128-bit stores per kept
//                                 fragment (only where one exists); lets the detach_bary backward stream instead of re-deriving geometry
//   out_rgba   (B,4,H,W), topk_ids (B,K,H,W) planar so that every warp store is a run of full 32 B sectors.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include "../../include/dbw_render.h"
#include "dbw_math.cuh"
#include "dbw_fraglist.cuh"
#include "dbw_camera.cuh"
#include "dbw_viz_math.cuh"
#include "dbw_shade_math.cuh"
#include "dbw_depth_math.cuh"

// ------------------------------------------------------------------------------------------------ error plumbing
static thread_local char g_err[512] = "";
static uint64_t g_launches = 0;

static int fail(const char* what, cudaError_t e = cudaSuccess) {
  if (e != cudaSuccess) snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  else snprintf(g_err, sizeof(g_err), "%s", what);
  return -1;
}
// shared with dbw_scene.cu
int dbw_fail_(const char* what, cudaError_t e) { return fail(what, e); }
void dbw_count_launch_(void) { ++g_launches; }
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(#call, _e); } while (0)
#define LAUNCH_CK(name) do { ++g_launches; cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return fail(name, _e); } while (0)

// CTAs of 256 threads for a grid-stride kernel over n items: at most `per_sm` per SM of the current device; -1 if the
// device cannot be queried
static int stride_grid(long long n, int per_sm) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return -1;
  const long long blocks = (n + 255) / 256, cap = (long long)sms * per_sm;
  return (int)(blocks < cap ? blocks : cap);
}

static int g_no_hard_kernel = 0;
// test hook: 1 routes hard single-layer renders through the generic kernel (the two must agree bit for bit)
extern "C" void dbw_debug_generic_kernel_only(int on) { g_no_hard_kernel = on; }
static int g_generic_blocks_loss = 0;
// test / benchmark hook: 1 routes the coarse phase's blocks loss pass through raster_forward_kernel<128, true> instead of
// blocks_loss_kernel (the two give the same loss bit for bit)
extern "C" void dbw_debug_generic_blocks_loss(int on) { g_generic_blocks_loss = on; }
static int g_keep_unread = 0;
// test hook: 1 keeps the outputs no backward reads -- the colour records of a pass without an opacity or distance path, and
// the alpha plane of a loss epilogue's g_env -- so that a test can compare against the computation that still writes them
extern "C" void dbw_debug_keep_unread_outputs(int on) { g_keep_unread = on; }
extern "C" int dbw_abi_version(void) { return DBW_ABI_VERSION; }
extern "C" size_t dbw_sizeof_settings(void) { return sizeof(DbwRenderSettings); }
extern "C" const char* dbw_last_error(void) { return g_err; }
extern "C" uint64_t dbw_launch_count(void) { return g_launches; }

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------ optional per-kernel timing
// CUDA events recorded on the launch stream around the two raster kernels (bench.py's live roofline measurement).
#include <vector>
struct TimedLaunch { int kind, K; cudaEvent_t a, b; };
static bool g_timing = false;
static std::vector<TimedLaunch> g_timed;
struct ScopedTimer {
  cudaStream_t st; bool on; TimedLaunch t;
  ScopedTimer(int kind, int K, cudaStream_t s) : st(s), on(g_timing) {
    if (!on) return;
    t.kind = kind; t.K = K; cudaEventCreate(&t.a); cudaEventCreate(&t.b); cudaEventRecord(t.a, st);
  }
  ~ScopedTimer() { if (on) { cudaEventRecord(t.b, st); g_timed.push_back(t); } }
};
extern "C" void dbw_timing_enable(int on) { g_timing = on != 0; }
extern "C" int dbw_timing_read(int kind, int K, double* total_ms, int* count) {
  double tot = 0; int n = 0;
  for (auto& t : g_timed) {
    if (t.kind != kind || (K > 0 && t.K != K)) continue;
    if (cudaEventSynchronize(t.b) != cudaSuccess) return fail("dbw_timing_read: event sync failed");
    float ms = 0.f; cudaEventElapsedTime(&ms, t.a, t.b); tot += ms; ++n;
  }
  if (total_ms) *total_ms = tot;
  if (count) *count = n;
  return 0;
}
extern "C" void dbw_timing_reset(void) {
  for (auto& t : g_timed) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
  g_timed.clear();
}

#ifndef DBW_CBIN
#define DBW_CBIN 64            // coarse bin edge in pixels (a multiple of every raster tile's width and height)
#endif
struct Workspace {
  float* verts_ndc; float4* bbox; float4* rec; float4* rec2; float* conv; int* view_flags; int* view_bbox; float4* maps4;
  int* view_nvis; int* vis_list;
  int* cbin_count; int* cbin_list; int cbin_nx, cbin_ny;       // coarse bins (DBW_CBIN x DBW_CBIN pixels): slot lists per (view, bin)
  float4* frag; float4* frag_rgb; unsigned char* nfrag; size_t total;
};
// Does the forward keep each fragment's colour?  The backward reads it only for colour . gradient, which feeds nothing but
// the suffix pass of the opacity and distance gradients.  A single-layer hard pass (sigma = 0: no distance path) whose
// caller declared it free of opacities (save_fragment_state = 2) has neither.
static bool keeps_colours(const DbwRenderSettings& s) {
  if (!s.save_fragment_state) return false;
  return g_keep_unread || !(s.save_fragment_state == 2 && s.faces_per_pixel == 1 && s.sigma == 0.f);
}
// bins = false: no coarse bins (a hard single-layer render never reads them; the resolving render leaves them out)
static Workspace carve(const DbwRenderSettings& s, void* base, bool bins = true) {
  Workspace w; char* p = (char*)base; size_t off = 0;
  const size_t B = s.n_views, V = s.n_verts, S = 2 * (size_t)s.n_faces;
  w.verts_ndc = (float*)(p + off); off += align_up(B * V * 3 * sizeof(float));
  w.bbox = (float4*)(p + off);     off += align_up(B * S * sizeof(float4));
  w.rec = (float4*)(p + off);      off += align_up(B * S * 4 * sizeof(float4));
  w.rec2 = (float4*)(p + off);     off += align_up(B * S * 2 * sizeof(float4));
  w.conv = (float*)(p + off);      off += align_up(B * S * 9 * sizeof(float));
  w.view_flags = (int*)(p + off);  off += align_up(B * sizeof(int));
  w.view_bbox = (int*)(p + off);   off += align_up(B * 4 * sizeof(int));
  w.view_nvis = (int*)(p + off);   off += align_up(B * sizeof(int));
  w.vis_list = (int*)(p + off);    off += align_up(B * S * sizeof(int));
  // coarse bins: every list can hold all 2F slots (worst case), so they are only used while that stays below 1 GB
  w.cbin_nx = (s.width + DBW_CBIN - 1) / DBW_CBIN; w.cbin_ny = (s.height + DBW_CBIN - 1) / DBW_CBIN;
  const size_t nb = (size_t)w.cbin_nx * w.cbin_ny;
  const bool use_bins = bins && B * nb * S * sizeof(int) <= ((size_t)1 << 30) && nb > 1;
  w.cbin_count = use_bins ? (int*)(p + off) : nullptr;  off += use_bins ? align_up(B * nb * sizeof(int)) : 0;
  w.cbin_list = use_bins ? (int*)(p + off) : nullptr;   off += use_bins ? align_up(B * nb * S * sizeof(int)) : 0;
  w.maps4 = (float4*)(p + off);    off += s.maps_are_texels4 ? 0 : align_up((size_t)(s.n_map_floats / 3) * sizeof(float4));
  const size_t npx = B * (size_t)s.height * s.width;
  w.frag = (float4*)(p + off);     off += s.save_fragment_state ? align_up(npx * (size_t)s.faces_per_pixel * sizeof(float4)) : 0;
  const bool rgb = keeps_colours(s);
  w.frag_rgb = rgb ? (float4*)(p + off) : nullptr; off += rgb ? align_up(npx * (size_t)s.faces_per_pixel * sizeof(float4)) : 0;
  w.nfrag = (unsigned char*)(p + off); off += s.save_fragment_state ? align_up(npx) : 0;
  w.total = off; return w;
}
struct BwdScratch { float* g_tri; float* g_conv; float* g_verts_ndc; float4* g_maps4; float4* g_cells; int* bary_flags; float* g_alpha; size_t total; };
static size_t bary_flag_count(const DbwRenderSettings& s);
static BwdScratch carve_bwd(const DbwRenderSettings& s, void* base) {
  BwdScratch w; char* p = (char*)base; size_t off = 0;
  const size_t B = s.n_views, V = s.n_verts, S = 2 * (size_t)s.n_faces;
  w.g_tri = (float*)(p + off);        off += align_up(B * S * 9 * sizeof(float));
  w.g_conv = (float*)(p + off);       off += align_up(B * S * 9 * sizeof(float));
  w.g_verts_ndc = (float*)(p + off);  off += align_up(B * V * 3 * sizeof(float));
  w.g_maps4 = (float4*)(p + off);     off += s.maps_are_texels4 ? 0 : align_up((size_t)(s.n_map_floats / 3) * sizeof(float4));
  // cell-map gradients: DBW_CELL_GRAD_COPIES copies of the whole map array (a CTA adds into one of them)
  w.g_cells = (float4*)(p + off);     off += s.maps_are_texels4 == 2 ? align_up((size_t)DBW_CELL_GRAD_COPIES * (s.n_map_floats / 3) * sizeof(float4)) : 0;
  w.bary_flags = (int*)(p + off);     off += align_up(bary_flag_count(s) * sizeof(int));
  // unscaled opacity gradient of a loss-epilogue forward that differentiates itself (dbw_render_forward_loss_grad)
  const size_t n_alpha = s.n_faces / (s.alpha_group > 0 ? s.alpha_group : 1);
  w.g_alpha = (float*)(p + off);      off += align_up(B * n_alpha * sizeof(float));
  w.total = off; return w;
}

extern "C" int dbw_workspace_bytes(const DbwRenderSettings* s, size_t* fwd, size_t* bwd) {
  if (!s) return fail("dbw_workspace_bytes: null settings");
  if (fwd) *fwd = carve(*s, nullptr).total;
  if (bwd) *bwd = carve_bwd(*s, nullptr).total;
  return 0;
}

static int validate(const DbwRenderSettings* s) {
  if (!s) return fail("null settings");
  if (s->n_views <= 0 || s->height <= 0 || s->width <= 0) return fail("n_views, height, width must be positive");
  if (s->faces_per_pixel <= 0 || s->faces_per_pixel > DBW_MAX_FACES_PER_PIXEL) return fail("faces_per_pixel out of range [1, 64]");
  if (s->n_verts <= 0 || s->n_faces <= 0 || s->n_maps <= 0) return fail("n_verts, n_faces, n_maps must be positive");
  const int ag = s->alpha_group > 0 ? s->alpha_group : 1;
  if (s->n_faces % ag) return fail("n_faces must be a multiple of alpha_group");
  if (s->alpha_view_stride != 0 && s->alpha_view_stride != s->n_faces / ag) return fail("alpha_view_stride must be 0 or n_faces / alpha_group");
  if (s->n_static_faces < 0 || s->n_static_faces > s->n_faces) return fail("n_static_faces out of range [0, n_faces]");
  if (s->save_fragment_state < 0 || s->save_fragment_state > 2) return fail("save_fragment_state must be 0, 1 or 2");
  if (2 * (long long)s->n_faces > DBW_FRAG_SLOT_MASK) return fail("too many faces: triangle slots are stored in 20 bits");
  if (s->n_maps > DBW_FRAG_MAX_MAPS) return fail("too many texture maps: a fragment's map is stored in 9 bits");
  if (s->sigma < 0.f || s->blur_radius < 0.f) return fail("sigma and blur_radius must be >= 0");
  if (s->n_map_floats <= 0 || s->n_map_floats % 3 != 0) return fail("n_map_floats must be a positive multiple of 3");
  if (s->maps_are_texels4 < 0 || s->maps_are_texels4 > 2) return fail("maps_are_texels4 must be 0, 1 or 2");
  return 0;
}

// ------------------------------------------------------------------------------------------------ texel repack
__global__ void maps_to_float4_kernel(const float* __restrict__ maps, float4* __restrict__ maps4, int n_texels) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_texels; i += gridDim.x * blockDim.x)
    maps4[i] = make_float4(maps[3 * i], maps[3 * i + 1], maps[3 * i + 2], 0.f);
}
// g_maps += the sum of the DBW_CELL_GRAD_COPIES cell-gradient copies (maps_are_texels4 = 2), times the device scalar *scale
// (NULL = 1)
__global__ void fold_gcells_kernel(const float4* __restrict__ gc, float4* __restrict__ g_maps, int n, const float* __restrict__ scale) {
  const float s = scale ? __ldg(scale) : 1.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 t = gc[i];
#pragma unroll
    for (int r = 1; r < DBW_CELL_GRAD_COPIES; ++r) {
      const float4 c = gc[(size_t)r * n + i];
      t.x += c.x; t.y += c.y; t.z += c.z;
    }
    float4 a = g_maps[i];
    a.x += s * t.x; a.y += s * t.y; a.z += s * t.z;
    g_maps[i] = a;
  }
}
// dst += *scale * src
__global__ void scale_add_kernel(float* __restrict__ dst, const float* __restrict__ src, int n, const float* __restrict__ scale) {
  const float s = __ldg(scale);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] += s * src[i];
}
__global__ void fold_gmaps_kernel(const float4* __restrict__ g4, float* __restrict__ g_maps, int n_texels) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_texels; i += gridDim.x * blockDim.x) {
    const float4 g = g4[i];
    g_maps[3 * i] += g.x; g_maps[3 * i + 1] += g.y; g_maps[3 * i + 2] += g.z;
  }
}

// ------------------------------------------------------------------------------------------------ projection (A1)
__global__ void project_verts_kernel(const float* __restrict__ vw, const float* __restrict__ R, const float* __restrict__ T,
                                     float fx, float fy, float px, float py, float eps, int B, int V, float* __restrict__ out,
                                     int* __restrict__ view_bbox, int* __restrict__ view_flags, int* __restrict__ view_nvis) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  // per-view state face_setup accumulates into (it runs after this kernel on the same stream): reset here, no extra launch
  if (i < B * 4) view_bbox[i] = (i & 1) ? (int)0x807fffff : (int)0x7f800000;     // f2ord(-inf) : f2ord(+inf)
  if (i < B) { view_flags[i] = 0; view_nvis[i] = 0; }
  if (i >= B * V) return;
  const int b = i / V, v = i - b * V;
  const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
  const float* r = R + b * 9; const float* t = T + b * 3;
  const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
  const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
  const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
  const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
  const float den = sgn * fmaxf(fabsf(zv), eps);
  out[i * 3] = (fx * xv + px * zv) / den;
  out[i * 3 + 1] = (fy * yv + py * zv) / den;
  out[i * 3 + 2] = zv;
}

// one warp per vertex: lanes stride over the views, shuffle-reduce, lane 0 accumulates (deterministic, no atomics)
__global__ void project_verts_backward_kernel(const float* __restrict__ vw, const float* __restrict__ R, const float* __restrict__ T,
                                              float fx, float fy, float px, float py, float eps, int B, int V,
                                              const float* __restrict__ g_ndc, float* __restrict__ g_vw) {
  const int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (v >= V) return;
  const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (int b = lane; b < B; b += 32) {
    const float* r = R + b * 9; const float* t = T + b * 3;
    const float* g = g_ndc + ((size_t)b * V + v) * 3;
    float gxv, gyv, gzv;
    dbw_project_backward(X, Y, Z, r, t, fx, fy, px, py, eps, g[0], g[1], g[2], gxv, gyv, gzv);
    ax += r[0] * gxv + r[1] * gyv + r[2] * gzv;
    ay += r[3] * gxv + r[4] * gyv + r[5] * gzv;
    az += r[6] * gxv + r[7] * gyv + r[8] * gzv;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ax += __shfl_xor_sync(0xffffffffu, ax, o); ay += __shfl_xor_sync(0xffffffffu, ay, o); az += __shfl_xor_sync(0xffffffffu, az, o);
  }
  if (lane == 0) { g_vw[v * 3] += ax; g_vw[v * 3 + 1] += ay; g_vw[v * 3 + 2] += az; }
}

// Gradient of the camera poses: one CTA per view sums X_world (x) g_view over the vertices (g_view: the same Jacobian as
// project_verts_backward_kernel) in a fixed order -- per thread, then xor-shuffles, then the warps in index order -- and
// adds the view's 9 + 3 sums into g_R / g_T.  Each element receives one atomic add per call, so the two passes of a fused
// step may accumulate into the same buffers from two streams and still sum to the same bits.
#define DBW_CAM_NT 256
__global__ void __launch_bounds__(DBW_CAM_NT) camera_grad_kernel(const float* __restrict__ vw, const float* __restrict__ R,
                                                                 const float* __restrict__ T, float fx, float fy, float px, float py,
                                                                 float eps, int V, const float* __restrict__ g_ndc,
                                                                 float* __restrict__ g_R, float* __restrict__ g_T) {
  __shared__ float s_part[DBW_CAM_NT / 32][12];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* r = R + b * 9; const float* t = T + b * 3;
  float acc[12] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};     // g_R (9), g_T (3)
  for (int v = tid; v < V; v += DBW_CAM_NT) {
    const float* g = g_ndc + ((size_t)b * V + v) * 3;
    const float gx = g[0], gy = g[1], gz = g[2];
    if (gx == 0.f && gy == 0.f && gz == 0.f) continue;          // a vertex no face of this view differentiated
    const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
    float gxv, gyv, gzv;
    dbw_project_backward(X, Y, Z, r, t, fx, fy, px, py, eps, gx, gy, gz, gxv, gyv, gzv);
    dbw_camera_accumulate(X, Y, Z, gxv, gyv, gzv, acc, acc + 9);
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 12; ++k) s_part[warp][k] = acc[k];
  }
  __syncthreads();
  if (tid < 12) {
    float s = 0.f;
    for (int w = 0; w < DBW_CAM_NT / 32; ++w) s += s_part[w][tid];
    float* dst = tid < 9 ? (g_R ? g_R + b * 9 + tid : nullptr) : (g_T ? g_T + b * 3 + (tid - 9) : nullptr);
    if (dst && s != 0.f) atomicAdd(dst, s);
  }
}

// ------------------------------------------------------------------------------------------------ per-view projection
// dbw_camera_project: project_verts_kernel's arithmetic with each view's own (fx, fy, px, py) read from intr (B,4)
__global__ void camera_project_kernel(const float* __restrict__ vw, const float* __restrict__ R, const float* __restrict__ T,
                                      const float* __restrict__ intr, float eps, int B, int V, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * V) return;
  const int b = i / V, v = i - b * V;
  const float fx = intr[b * 4], fy = intr[b * 4 + 1], px = intr[b * 4 + 2], py = intr[b * 4 + 3];
  const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
  const float* r = R + b * 9; const float* t = T + b * 3;
  const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
  const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
  const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
  const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
  const float den = sgn * fmaxf(fabsf(zv), eps);
  out[i * 3] = (fx * xv + px * zv) / den;
  out[i * 3 + 1] = (fy * yv + py * zv) / den;
  out[i * 3 + 2] = zv;
}

// world-vertex gradient of dbw_camera_project: project_verts_backward_kernel with per-view intrinsics (one warp per vertex,
// lanes over the views, no atomics: g_vw receives one add per element)
__global__ void camera_project_verts_backward_kernel(const float* __restrict__ vw, const float* __restrict__ R,
                                                     const float* __restrict__ T, const float* __restrict__ intr, float eps,
                                                     int B, int V, const float* __restrict__ g_ndc, float* __restrict__ g_vw) {
  const int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (v >= V) return;
  const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (int b = lane; b < B; b += 32) {
    const float* r = R + b * 9; const float* t = T + b * 3; const float* k = intr + b * 4;
    const float* g = g_ndc + ((size_t)b * V + v) * 3;
    float gxv, gyv, gzv;
    dbw_project_backward(X, Y, Z, r, t, k[0], k[1], k[2], k[3], eps, g[0], g[1], g[2], gxv, gyv, gzv);
    ax += r[0] * gxv + r[1] * gyv + r[2] * gzv;
    ay += r[3] * gxv + r[4] * gyv + r[5] * gzv;
    az += r[6] * gxv + r[7] * gyv + r[8] * gzv;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ax += __shfl_xor_sync(0xffffffffu, ax, o); ay += __shfl_xor_sync(0xffffffffu, ay, o); az += __shfl_xor_sync(0xffffffffu, az, o);
  }
  if (lane == 0) { g_vw[v * 3] += ax; g_vw[v * 3 + 1] += ay; g_vw[v * 3 + 2] += az; }
}

// camera gradient of dbw_camera_project: camera_grad_kernel's fixed-order per-view sums, with the view's 4 intrinsics
// sums after its 9 + 3 pose sums; each element of g_R / g_T / g_intr receives one atomic add per call
#define DBW_CAMK_N 16
__global__ void __launch_bounds__(DBW_CAM_NT) camera_project_camera_backward_kernel(
    const float* __restrict__ vw, const float* __restrict__ R, const float* __restrict__ T, const float* __restrict__ intr,
    float eps, int V, const float* __restrict__ g_ndc, float* __restrict__ g_R, float* __restrict__ g_T, float* __restrict__ g_intr) {
  __shared__ float s_part[DBW_CAM_NT / 32][DBW_CAMK_N];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* r = R + b * 9; const float* t = T + b * 3;
  const float fx = intr[b * 4], fy = intr[b * 4 + 1], px = intr[b * 4 + 2], py = intr[b * 4 + 3];
  float acc[DBW_CAMK_N];                                         // g_R (9), g_T (3), g_intr (4)
#pragma unroll
  for (int k = 0; k < DBW_CAMK_N; ++k) acc[k] = 0.f;
  for (int v = tid; v < V; v += DBW_CAM_NT) {
    const float* g = g_ndc + ((size_t)b * V + v) * 3;
    const float gx = g[0], gy = g[1], gz = g[2];
    if (gx == 0.f && gy == 0.f && gz == 0.f) continue;          // a vertex no face of this view differentiated
    const float X = vw[v * 3], Y = vw[v * 3 + 1], Z = vw[v * 3 + 2];
    float gxv, gyv, gzv;
    dbw_project_backward(X, Y, Z, r, t, fx, fy, px, py, eps, gx, gy, gz, gxv, gyv, gzv);
    dbw_camera_accumulate(X, Y, Z, gxv, gyv, gzv, acc, acc + 9);
    dbw_intrinsics_accumulate(X, Y, Z, r, t, eps, gx, gy, acc + 12);
  }
#pragma unroll
  for (int k = 0; k < DBW_CAMK_N; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < DBW_CAMK_N; ++k) s_part[warp][k] = acc[k];
  }
  __syncthreads();
  if (tid < DBW_CAMK_N) {
    float s = 0.f;
    for (int w = 0; w < DBW_CAM_NT / 32; ++w) s += s_part[w][tid];
    float* dst = tid < 9 ? (g_R ? g_R + b * 9 + tid : nullptr)
               : tid < 12 ? (g_T ? g_T + b * 3 + (tid - 9) : nullptr)
                          : (g_intr ? g_intr + b * 4 + (tid - 12) : nullptr);
    if (dst && s != 0.f) atomicAdd(dst, s);
  }
}

static int check_camera_project(const char* who, int32_t n_views, int32_t n_verts, const float* verts, const float* R,
                                const float* T, const float* intrinsics, float eps) {
  char msg[200];
  const char* why = (n_views <= 0 || n_verts <= 0) ? "n_views and n_verts must be positive"
                  : ((long long)n_views * n_verts * 3 > 0x7fffffffLL || (long long)n_verts * 32 > 0x7fffffffLL)
                      ? "too many views or vertices for one call (32-bit indexing)"
                  : (!verts || !R || !T || !intrinsics) ? "verts, R, T and intrinsics are required"
                  : !(eps > 0.f) ? "eps must be positive"
                  : nullptr;
  if (!why) return 0;
  snprintf(msg, sizeof(msg), "%s: %s", who, why);
  return fail(msg);
}

extern "C" int dbw_camera_project(int32_t n_views, int32_t n_verts, const float* verts, const float* R, const float* T,
                                  const float* intrinsics, float eps, float* verts_ndc, void* stream) {
  if (check_camera_project("dbw_camera_project", n_views, n_verts, verts, R, T, intrinsics, eps)) return -1;
  if (!verts_ndc) return fail("dbw_camera_project: verts_ndc is required");
  const int n = n_views * n_verts;
  camera_project_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(verts, R, T, intrinsics, eps, n_views, n_verts, verts_ndc);
  LAUNCH_CK("camera_project_kernel");
  return 0;
}

extern "C" int dbw_camera_project_backward(int32_t n_views, int32_t n_verts, const float* verts, const float* R, const float* T,
                                           const float* intrinsics, float eps, const float* g_ndc, float* g_verts, float* g_R,
                                           float* g_T, float* g_intrinsics, void* stream) {
  if (check_camera_project("dbw_camera_project_backward", n_views, n_verts, verts, R, T, intrinsics, eps)) return -1;
  if (!g_ndc) return fail("dbw_camera_project_backward: g_ndc is required");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_verts) {
    camera_project_verts_backward_kernel<<<(n_verts * 32 + 127) / 128, 128, 0, st>>>(verts, R, T, intrinsics, eps, n_views, n_verts,
                                                                                      g_ndc, g_verts);
    LAUNCH_CK("camera_project_verts_backward_kernel");
  }
  if (g_R || g_T || g_intrinsics) {
    camera_project_camera_backward_kernel<<<n_views, DBW_CAM_NT, 0, st>>>(verts, R, T, intrinsics, eps, n_verts, g_ndc, g_R, g_T,
                                                                          g_intrinsics);
    LAUNCH_CK("camera_project_camera_backward_kernel");
  }
  return 0;
}

// order-preserving float <-> int map, so that atomicMin/atomicMax on ints order floats of either sign
__device__ __forceinline__ int f2ord(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// ------------------------------------------------------------------------------------------------ face setup + z-clip (A3)
#include "dbw_clip.cuh"

__device__ __forceinline__ void write_slot(float4* bbox, float4* rec, float4* rec2, float* conv, size_t slot, const float* tri,
                                           const float* cv, bool clipped, int face, int neighbor, float sqrt_blur,
                                           float4 uv01, float4 uv2m) {
  rec2[slot * 2] = uv01; rec2[slot * 2 + 1] = uv2m;
  const float x0 = tri[0], y0 = tri[1], z0 = tri[2], x1 = tri[3], y1 = tri[4], z1 = tri[5], x2 = tri[6], y2 = tri[7], z2 = tri[8];
  const float zmin = fminf(fminf(z0, z1), z2);
  const f2 a = {x0, y0}, b = {x1, y1}, c = {x2, y2};
  const float area = edge_nc(c, a, b);
  const bool degenerate = (area <= DBW_KEPS && area >= -DBW_KEPS);
  const bool valid = !(zmin < DBW_KEPS) && !degenerate;
  float4 bb;
  if (valid) {
    bb.x = fminf(fminf(x0, x1), x2) - sqrt_blur; bb.y = fmaxf(fmaxf(x0, x1), x2) + sqrt_blur;
    bb.z = fminf(fminf(y0, y1), y2) - sqrt_blur; bb.w = fmaxf(fmaxf(y0, y1), y2) + sqrt_blur;
  } else {
    bb.x = INFINITY; bb.y = -INFINITY; bb.z = INFINITY; bb.w = -INFINITY;
  }
  bbox[slot] = bb;
  rec[slot * 4 + 0] = make_float4(x0, y0, x1, y1);
  rec[slot * 4 + 1] = make_float4(x2, y2, z0, z1);
  rec[slot * 4 + 2] = make_float4(z2, __int_as_float(face), __int_as_float(neighbor), __int_as_float(clipped ? 1 : 0));
  const float l01 = (x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0), l02 = (x2 - x0) * (x2 - x0) + (y2 - y0) * (y2 - y0);
  const float l12 = (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1);
  rec[slot * 4 + 3] = make_float4(1.f / __fadd_rn(area, DBW_KEPS), l01 <= DBW_KEPS ? -1.f : 1.f / l01,
                                  l02 <= DBW_KEPS ? -1.f : 1.f / l02, l12 <= DBW_KEPS ? -1.f : 1.f / l12);
  if (clipped) {
#pragma unroll
    for (int i = 0; i < 9; ++i) conv[slot * 9 + i] = cv[i];
  }
}

__global__ void init_view_bbox_kernel(int* vb, int* flags, int* nvis, int B) {      // only when the vertices come in as NDC
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * 4) vb[i] = (i & 1) ? f2ord(-INFINITY) : f2ord(INFINITY);
  if (i < B) { flags[i] = 0; nvis[i] = 0; }
}

__global__ void face_setup_kernel(const float* __restrict__ verts_ndc, const int* __restrict__ faces, int B, int V, int F,
                                  float z_clip, int persp, float sqrt_blur, const float* __restrict__ faces_uvs,
                                  const int* __restrict__ face_map, const DbwMapDesc* __restrict__ map_table,
                                  float4* __restrict__ bbox, float4* __restrict__ rec, float4* __restrict__ rec2,
                                  float* __restrict__ conv, int* __restrict__ view_flags, int* __restrict__ view_bbox,
                                  int* __restrict__ view_nvis, int* __restrict__ vis_list, float screen_x, float screen_y) {
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  const bool tail = i0 >= B * F;                    // tail lanes redo the last face (idempotent writes) so that the warp
  const int i = tail ? B * F - 1 : i0;              // stays converged for the shuffles below
  const int b = i / F, f = i - b * F;
  float a[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float* v = verts_ndc + ((size_t)b * V + faces[f * 3 + j]) * 3;
    a[j][0] = v[0]; a[j][1] = v[1]; a[j][2] = v[2];
  }
  ClipResult r;
  clip_face(a, z_clip, persp != 0, r);
  const size_t s0 = (size_t)b * 2 * F + f, s1 = s0 + F;
  const float inval[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};     // zmin = 0 < eps -> marked empty
  const float* fu = faces_uvs + (size_t)f * 6;
  const int mid = face_map[f];
  if (mid < 0) r.ntri = 0;                                 // face disabled by the caller (e.g. a killed block): never rasterized
  const DbwMapDesc md = map_table[mid < 0 ? 0 : mid];
  const float4 uv01 = make_float4(fu[0], fu[1], fu[2], fu[3]);
  (void)md;
  const float4 uv2m = make_float4(fu[4], fu[5], __int_as_float(mid < 0 ? 0 : mid), 0.f);
  write_slot(bbox, rec, rec2, conv, s0, r.ntri >= 1 ? r.tri[0] : inval, r.conv[0], r.clipped, f, r.ntri == 2 ? F + f : -1, sqrt_blur, uv01, uv2m);
  write_slot(bbox, rec, rec2, conv, s1, r.ntri == 2 ? r.tri[1] : inval, r.conv[1], r.clipped, f, r.ntri == 2 ? f : -1, sqrt_blur, uv01, uv2m);
  if (r.ntri == 2) atomicOr(&view_flags[b], 1);
  // the view's list of slots whose (blur-expanded) box reaches the screen at all: the hard single-layer kernel scans this
  // instead of all 2F slots (32-40 of the 896 environment slots at the DTU cameras)
  if (!tail) {
    for (int q = 0; q < r.ntri; ++q) {
      const size_t sl = q == 0 ? s0 : s1;
      const float4 bb = bbox[sl];
      if (bb.x <= screen_x && bb.y >= -screen_x && bb.z <= screen_y && bb.w >= -screen_y)
        vis_list[(size_t)b * 2 * F + atomicAdd(&view_nvis[b], 1)] = q == 0 ? f : F + f;
    }
  }
  // union of the (blur-expanded) face boxes of the view: tiles outside it skip the binning scan altogether
  float ux0 = INFINITY, ux1 = -INFINITY, uy0 = INFINITY, uy1 = -INFINITY;
  for (int q = 0; q < r.ntri; ++q) {
    const float4 bb = bbox[q == 0 ? s0 : s1];
    ux0 = fminf(ux0, bb.x); ux1 = fmaxf(ux1, bb.y); uy0 = fminf(uy0, bb.z); uy1 = fmaxf(uy1, bb.w);
  }
  // one atomic set per warp
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ux0 = fminf(ux0, __shfl_xor_sync(0xffffffffu, ux0, o)); ux1 = fmaxf(ux1, __shfl_xor_sync(0xffffffffu, ux1, o));
    uy0 = fminf(uy0, __shfl_xor_sync(0xffffffffu, uy0, o)); uy1 = fmaxf(uy1, __shfl_xor_sync(0xffffffffu, uy1, o));
  }
  const int b_lead = __shfl_sync(0xffffffffu, b, 0);
  if (__all_sync(0xffffffffu, b == b_lead)) {
    if ((threadIdx.x & 31) == 0 && ux0 <= ux1) {
      atomicMin(&view_bbox[b * 4], f2ord(ux0)); atomicMax(&view_bbox[b * 4 + 1], f2ord(ux1));
      atomicMin(&view_bbox[b * 4 + 2], f2ord(uy0)); atomicMax(&view_bbox[b * 4 + 3], f2ord(uy1));
    }
  } else if (r.ntri > 0) {          // warp straddles two views: recompute this lane's own box
    float lx0 = INFINITY, lx1 = -INFINITY, ly0 = INFINITY, ly1 = -INFINITY;
    for (int q = 0; q < r.ntri; ++q) {
      const float4 bb = bbox[q == 0 ? s0 : s1];
      lx0 = fminf(lx0, bb.x); lx1 = fmaxf(lx1, bb.y); ly0 = fminf(ly0, bb.z); ly1 = fmaxf(ly1, bb.w);
    }
    if (lx0 <= lx1) {
      atomicMin(&view_bbox[b * 4], f2ord(lx0)); atomicMax(&view_bbox[b * 4 + 1], f2ord(lx1));
      atomicMin(&view_bbox[b * 4 + 2], f2ord(ly0)); atomicMax(&view_bbox[b * 4 + 3], f2ord(ly1));
    }
  }
}

// ------------------------------------------------------------------------------------------------ coarse binning
// One CTA per (view, 64 x 64 pixel bin): the slots whose blur-expanded box reaches the bin, compacted into the bin's list.
// A raster tile then scans its bin's list (tens of slots) instead of the view's 2F (800 - 8000): at the stress shape the
// per-tile scan of all 8000 slots was half of the forward's instructions.  A view with z-clipped slots lists them in
// frag_order_key order (the clipped mesh's face order, dbw_fraglist.cuh): slots are scanned in that order and compacted in
// order (a block prefix over the warps' counts per batch), so that the raster kernel's chunked path offers them in it.  Other
// views cannot depend on the order: one shared atomic per warp and batch, no barrier.
__global__ void coarse_bin_kernel(const float4* __restrict__ bbox, const int* __restrict__ view_flags, int F, int H, int W,
                                  int nbx, int nby, int* __restrict__ cbin_count, int* __restrict__ cbin_list) {
  __shared__ int s_n;
  __shared__ int s_wn[32];
  const int view = blockIdx.x, bin = blockIdx.y, bx = bin % nbx, by = bin / nbx;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  if (tid == 0) s_n = 0;
  __syncthreads();
  const int x0 = bx * DBW_CBIN, x1 = min(x0 + DBW_CBIN, W) - 1, y0 = by * DBW_CBIN, y1 = min(y0 + DBW_CBIN, H) - 1;
  // NDC extents of the bin's pixel centres (+X is left, +Y is up: the last column / row has the smallest coordinate)
  const float xmin = pix_to_ndc(W - 1 - x1, W, H), xmax = pix_to_ndc(W - 1 - x0, W, H);
  const float ymin = pix_to_ndc(H - 1 - y1, H, W), ymax = pix_to_ndc(H - 1 - y0, H, W);
  const bool split = view_flags[view] & 1;
  const int nslots = split ? 2 * F : F;
  const float4* bb = bbox + (size_t)view * 2 * F;
  int* list = cbin_list + ((size_t)view * gridDim.y + bin) * 2 * F;
  int n = 0;                        // entries listed so far in order (the same in every thread)
  for (int base = 0; base < nslots; base += blockDim.x) {
    const int i = base + tid;
    const int sl = split ? frag_order_slot(i, F) : i;
    bool hit = false;
    if (i < nslots) { const float4 b = __ldg(&bb[sl]); hit = !(b.x > xmax || b.y < xmin || b.z > ymax || b.w < ymin); }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (split) {
      if (lane == 0) s_wn[warp] = __popc(m);
      __syncthreads();
      int pos = n;
      for (int w = 0; w < n_warps; ++w) { const int c = s_wn[w]; pos += w < warp ? c : 0; n += c; }
      if (hit) list[pos + __popc(m & ((1u << lane) - 1u))] = sl;
      __syncthreads();              // s_wn is read before the next batch writes it
    } else if (m) {
      int wbase = 0;
      if (lane == 0) wbase = atomicAdd(&s_n, __popc(m));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      if (hit) list[wbase + __popc(m & ((1u << lane) - 1u))] = sl;
    }
  }
  __syncthreads();
  if (tid == 0) cbin_count[(size_t)view * gridDim.y + bin] = split ? n : s_n;
}

// ------------------------------------------------------------------------------------------------ raster + shade + blend, forward
struct RasterParams {
  int B, H, W, K, V, F, M;
  int alpha_stride;
  float inv_alpha_group;     // 1 / (faces sharing one opacity entry): alpha index = floor((face + 0.5) * inv_alpha_group)
  int n_alpha;               // opacity entries per view = F / alpha_group
  int n_static_faces;        // faces [0, n_static_faces) have constant vertices: the backward skips their vertex gradient
  const int* view_rows;      // (B,2) [row_begin, row_end) rendered of each view, or NULL = all rows (row-band sharding)
  float sigma, blur, sqrt_blur, bg0, bg1, bg2;
  int clip_inside, persp, clipb, detach_bary;
  const float4* bbox; const float4* rec; const float4* rec2; const float* conv; const int* view_flags; const int* view_bbox;
  const int* view_nvis; const int* vis_list;
  const int* cbin_count; const int* cbin_list; int cbin_nx, cbin_ny;
  const float4* maps4;
  const float* faces_alpha;
  float* out_rgba; int* topk;        // topk may be NULL
  const DbwMapDesc* map_table;   // (M) device: offset (3 * first texel), height, width of each map
  float4* frag;              // (B,K,H,W) saved fragment records {bits, u, v, signed dist} or NULL
  float4* frag_rgb;          // (B,K,H,W) their colours {r, g, b, -}: the backward's d/d(opacity) needs colour . gradient
  unsigned char* nfrag;      // (B,H,W) number of records written per pixel
  const float* face_shade;   // (B,F,3) per-view per-face colour multiplier (flat shading) or NULL
  float* out_dists;          // (B,K,H,W) signed squared distances of the kept fragments (-1 = empty) or NULL
  // backward only (and the forward with ep_grad)
  const float* grad_rgba; float* g_tri; float* g_conv; float* g_faces_alpha; float4* g_maps4;
  float4* g_cells; int n_cells;   // cell-map gradient copies (DBW_CELL_GRAD_COPIES x n_cells) or NULL: cell taps go to g_maps4
  const float* grad_scale;   // device scalar multiplied into grad_rgba (the upstream gradient of a fused loss) or NULL
  int* bary_flags;           // (B, tile columns, strips) of a non-detached single-layer pass: strip needs the barycentric path
  // fused compositing + MSE epilogue of the forward (DbwLossEpilogue); ep_target == NULL: plain render
  const float* ep_env; const float* ep_target; float* ep_g_env; float* ep_rec; float* ep_partials;
  float ep_inv_count; int ep_part_mask;
  int ep_skip_env_alpha;     // DbwLossEpilogue.env_alpha_unread: the alpha plane of ep_g_env is not written
  // the epilogue also differentiates the pass (dbw_render_forward_loss_grad): unscaled gradients into g_tri / g_cells /
  // g_faces_alpha, which then point at the backward scratch
  int ep_grad;
};
// Depth outputs and their gradients (dbw_render_forward_depth / dbw_render_backward_depth): a kernel argument of the DEPTH
// instantiations only, so that RasterParams -- and with it every other kernel -- is unchanged.
struct DepthIO {
  float* zbuf;               // (B,K,H,W) view-space depth of each kept fragment (-1 = empty) or NULL
  float* depth;              // (B,1,H,W) the fragments' depths blended with the colour weights (background 0) or NULL
  const float* g_zbuf; const float* g_depth;   // their gradients, multiplied by *grad_scale as read (either may be NULL)
};

// Raster CTAs: the 8x4-pixel patches of a CTA's warps tile a 16 x (NT / 16) pixel tile.  The backward kernels and the
// K > 4 forward use 128 threads (finer scheduling granularity, less waiting on the slowest warp of a tile), the K <= 4
// forward 256 (the bin scan is amortised over more pixels).
#ifndef DBW_FWD_NT_SMALLK
#define DBW_FWD_NT_SMALLK 256
#endif
#ifndef DBW_FWD_NT
#define DBW_FWD_NT 128
#endif
#ifndef DBW_BWD_NT
#define DBW_BWD_NT 128
#endif
#define TILE_W 16
#ifndef DBW_AGG_MIN
#define DBW_AGG_MIN 2         // groups of at most this many lanes use plain atomics instead of a warp reduction
#endif
#define DBW_ALPHA_SMEM_MAX 512      // opacity entries per view that a CTA may pre-accumulate in shared memory

// opacity of one fragment from its signed squared distance (layered_rgb_blend, src/model/renderer.py:252-257)
__device__ __forceinline__ float frag_alpha(float d, float sigma, int clip_inside) {
  if (sigma == 0.f) return d <= 0.f ? 1.f : 0.f;
  // __expf: ex2.approx-based, relative error ~1e-6 over the halo range |d/sigma| <= 9.3 -- far inside the 1e-4 image tolerance
  if (clip_inside) return __expf(-fmaxf(d, 0.f) / sigma);
  return 1.f / (1.f + __expf(d / sigma));
}

// index of a face's opacity entry: faces_alpha holds one value per group of `alpha_group` consecutive faces
__device__ __forceinline__ int alpha_index(const RasterParams& P, int view, int face) {
  return view * P.alpha_stride + __float2int_rd(((float)face + 0.5f) * P.inv_alpha_group);
}

// bilinear colour of a fragment from its UV (shared by forward shading and the detach_bary backward)
struct Texel4 { TexTap tap; f3 c00, c01, c10, c11, color; };
// the map table in shared memory: (first texel, H, W, DBW_MAP_CELLS or 0) per map, staged once per CTA -- a fragment's tap addresses then
// depend on no global load
__device__ __forceinline__ void stage_map_table(const RasterParams& P, int4* s_desc, int tid, int nthreads) {
  for (int m = tid; m < P.M; m += nthreads) {
    const DbwMapDesc d = P.map_table[m];
    s_desc[m] = make_int4(d.offset / 3, d.height, d.width, d.reserved);
  }
}
// taps of (u, v) in map d: texel indices, or cell indices for a cell map (d.w != 0)
__device__ __forceinline__ TexTap map_tap(float u, float v, int4 d) {
  TexTap t = tex_tap(u, v, d.x, d.y, d.z);
  if (d.w) tap_to_cells(t, d.x, d.y, d.w);
  return t;
}
__device__ __forceinline__ void tap_only(float u, float v, int4 d, Texel4& s) { s.tap = map_tap(u, v, d); }
// CELLS: the caller knows that d is a cell map (d.w != 0)
template <bool CELLS = false>
__device__ __forceinline__ void fetch_color(const RasterParams& P, float u, float v, int4 d, Texel4& s) {
  s.tap = map_tap(u, v, d);
  s.c00 = ld_texel(P.maps4, s.tap.i00);
  if (CELLS || d.w) { // cell map: the four taps usually share one cell (49 of 64 footprints at f = 8); each distinct cell is loaded once
    s.c01 = s.tap.i01 == s.tap.i00 ? s.c00 : ld_texel(P.maps4, s.tap.i01);
    s.c10 = s.tap.i10 == s.tap.i00 ? s.c00 : ld_texel(P.maps4, s.tap.i10);
    s.c11 = s.tap.i11 == s.tap.i01 ? s.c01 : (s.tap.i11 == s.tap.i10 ? s.c10 : ld_texel(P.maps4, s.tap.i11));
  } else {
    s.c01 = ld_texel(P.maps4, s.tap.i01); s.c10 = ld_texel(P.maps4, s.tap.i10); s.c11 = ld_texel(P.maps4, s.tap.i11);
  }
  s.color.x = s.c00.x * s.tap.w00 + s.c01.x * s.tap.w01 + s.c10.x * s.tap.w10 + s.c11.x * s.tap.w11;
  s.color.y = s.c00.y * s.tap.w00 + s.c01.y * s.tap.w01 + s.c10.y * s.tap.w10 + s.c11.y * s.tap.w11;
  s.color.z = s.c00.z * s.tap.w00 + s.c01.z * s.tap.w01 + s.c10.z * s.tap.w10 + s.c11.z * s.tap.w11;
}

// geometry of fragment (slot) at pixel p, re-derived from the face records (the barycentric-path backward needs all of it)
struct Shade {
  TriGeom t; Bary b; f3 bu;       // bu: barycentrics w.r.t. the ORIGINAL face (after un-clipping)
  float4 uv01; float u2, v2;      // per-face-vertex UVs
  float u, v; int map_id;
};

__device__ __forceinline__ void shade_geometry(const RasterParams& P, int view, int slot, f2 p, Shade& s) {
  const size_t gs = (size_t)view * 2 * P.F + slot;
  const float4 r0 = __ldg(&P.rec[gs * 4]), r1 = __ldg(&P.rec[gs * 4 + 1]), r2 = __ldg(&P.rec[gs * 4 + 2]), r3 = __ldg(&P.rec[gs * 4 + 3]);
  const float4 q0 = __ldg(&P.rec2[gs * 2]);
  const float4 q1 = __ldg(&P.rec2[gs * 2 + 1]);
  s.map_id = __float_as_int(q1.z);
  s.t = unpack_tri(r0, r1, r2, r3);
  s.b = eval_bary(p, s.t, P.persp, P.clipb);
  s.bu = s.b.bc;
  if (s.t.flags & 1) {
    const float* cv = P.conv + gs * 9;
    s.bu.x = s.b.bc.x * cv[0] + s.b.bc.y * cv[3] + s.b.bc.z * cv[6];
    s.bu.y = s.b.bc.x * cv[1] + s.b.bc.y * cv[4] + s.b.bc.z * cv[7];
    s.bu.z = s.b.bc.x * cv[2] + s.b.bc.y * cv[5] + s.b.bc.z * cv[8];
  }
  s.uv01 = q0; s.u2 = q1.x; s.v2 = q1.y;
  s.u = s.bu.x * q0.x + s.bu.y * q0.z + s.bu.z * q1.x;
  s.v = s.bu.x * q0.y + s.bu.y * q0.w + s.bu.z * q1.y;
}

// Resident CTAs per SM each raster kernel is compiled for (register cap = 65536 / (threads * CTAs)).
#ifndef DBW_FWD_SMALLK_MINB
#define DBW_FWD_SMALLK_MINB 5     // CTAs of DBW_FWD_NT_SMALLK threads (51 registers)
#endif
#ifndef DBW_FWD_MINB
#define DBW_FWD_MINB 7            // CTAs of DBW_FWD_NT threads: shared memory (25.6 KB of lists at K = 10 + 5 KB tile list) allows 7
                                  // of the 227 KB an H100 SM gives its CTAs (72 registers)
#endif
#ifndef DBW_BWD_DETACH_MINB
#define DBW_BWD_DETACH_MINB 7     // backward without the barycentric path, CTAs of DBW_BWD_NT threads (72 registers)
#endif
#ifndef DBW_BWD_BARY_MINB
#define DBW_BWD_BARY_MINB 4       // backward with the barycentric path: more live state (128 registers)
#endif
#ifndef DBW_BWD_GEOM_MINB
#define DBW_BWD_GEOM_MINB 5       // barycentric path of a single-layer pass alone (raster_bary_backward_kernel, 93 registers)
#endif

// CTA -> (view, tile) mapping of the raster kernels.  CTAs are dispatched in linear grid order, so the grid is laid out as
// (view, tile column, tile row RANK) with the rows ranked centre-out: every view's central rows -- where the blocks are and the
// CTAs run longest -- are dispatched first, the cheap border rows last.  With the few waves a view-sharded rank has (8750 CTAs
// at 8 GPUs = 8 waves), the last wave otherwise holds the heavy tiles of the last view while most SMs idle.
__device__ __forceinline__ int centre_out(int rank, int n) {
  const int c = n >> 1;
  return (rank & 1) ? c - ((rank + 1) >> 1) : c + (rank >> 1);
}

template <bool BLOCKS>
__device__ __forceinline__ void epilogue_backward(const RasterParams& P, float4* lA, float* lV, int stride, const int4* s_desc,
                                                  float* s_galpha, bool live, int n, f2 p, const float (&g)[4], int view,
                                                  int lane, int warp);

// One body for every K: the per-pixel list of the K nearest fragments lives in (dynamic) shared memory (dbw_fraglist.cuh).
// EP: with the compositing + MSE loss epilogue (DbwLossEpilogue); a template flag so that plain renders carry none of it.
// With P.ep_grad the epilogue then also runs the pass's detach_bary backward on the list still in shared memory
// (epilogue_backward): no fragment record and no gradient image goes through HBM.
// BLOCKS (with EP, NT = 128: blocks_loss_kernel): the coarse phase's blocks loss pass, which the dispatch sends here only with
// ep_grad, cell maps, no optional output (fragment records, ids, distances, flat shading, image) and at most
// DBW_ALPHA_SMEM_MAX opacity entries per view.  The branches it never takes are compiled out, and the view's opacity table
// is staged in shared memory beside the opacity sums, so that the shading loop and the backward's pass 1 read no global
// memory but the texels.  Every decision and every loss term is the generic instantiation's; the gradients differ only by
// the order of their atomics.
// DEPTH (depth_forward_kernel): also writes each kept fragment's depth (its pz, DepthIO.zbuf) and the depth blended with
// the colour weights (DepthIO.depth), and keeps the records of the layers behind a fully opaque one too (their zbuf still has
// a gradient); the image is the plain instantiation's bit for bit.
template <int NT, bool EP, bool BLOCKS, bool DEPTH = false>
__device__ __forceinline__ void raster_forward_body(const RasterParams& P, const DepthIO& Dz = DepthIO{}) {
  static_assert(!DEPTH || !EP, "depth has no loss epilogue");
  static_assert(!BLOCKS || (EP && NT == 128), "the blocks loss pass is a loss-epilogue pass of 128 threads");
  // faces a tile lists at once (more: chunked path)
#ifndef DBW_LIST_CAP
#define DBW_LIST_CAP 64      // tile lists average 17 faces (max 64) at cfg 2: 5 KB instead of 10.5 KB buys a 7th resident CTA
#endif
  constexpr int CAP = NT <= 128 ? DBW_LIST_CAP : 256;
  static_assert(CAP >= NT || CAP == 64, "a scan batch adds up to NT entries");
  __shared__ float4 s_bbox[CAP];
  __shared__ float4 s_rec[CAP * 4];
  __shared__ int s_slot[CAP];
  __shared__ int s_count;
  __shared__ __align__(8) uint64_t s_bar;      // mbarrier of the TMA record gather
  extern __shared__ float4 s_dyn[];            // fragment lists: K*NT float4 (pz, bits, sd, u), K*NT float (v); then the map table
                                               // (and with ep_grad the opacity sums, then with BLOCKS the opacity table)
  uint32_t bar_phase = 0;

  constexpr int TILE_H = NT / 16;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = blockIdx.x;
  const int tile_y = centre_out(blockIdx.z, gridDim.z);
  const int tx0 = blockIdx.y * TILE_W, ty0 = tile_y * TILE_H;
  // a warp covers an 8x4 pixel patch; 2x4 warps cover the 16x16 tile
  const int xi = tx0 + (warp & 1) * 8 + (lane & 7);
  const int yi = ty0 + (warp >> 1) * 4 + (lane >> 3);
  int row_lo = 0, row_hi = P.H;
  if (P.view_rows) { row_lo = P.view_rows[view * 2]; row_hi = P.view_rows[view * 2 + 1]; }
  if (ty0 >= row_hi || ty0 + TILE_H <= row_lo) return;       // this view's rows of the tile belong to another rank
  const bool live = xi < P.W && yi < P.H && yi >= row_lo && yi < row_hi;
  // NDC coordinates of the tile's 16 pixel columns and 16 rows (+X is left, +Y is up): 32 exact evaluations per CTA,
  // shared through shared memory, instead of two per thread
  __shared__ float s_ndc[TILE_W + TILE_H];
  if (tid < TILE_W) s_ndc[tid] = pix_to_ndc(P.W - 1 - min(tx0 + tid, P.W - 1), P.W, P.H);
  else if (tid < TILE_W + TILE_H) s_ndc[tid] = pix_to_ndc(P.H - 1 - min(ty0 + tid - TILE_W, P.H - 1), P.H, P.W);
  if (tid == 0) { s_count = 0; mbar_init(&s_bar, 1); }
  // the map table goes to shared memory too: this thread's entry is loaded now and stored just before the barrier that follows
  // the bin scan, so that nobody waits for it
  int4* const s_desc = reinterpret_cast<int4*>(reinterpret_cast<float*>(s_dyn + (size_t)P.K * NT) + (size_t)P.K * NT);
  float* const s_galpha = reinterpret_cast<float*>(s_desc + P.M);
  float* const s_alpha = s_galpha + P.n_alpha;
  const bool alpha_sums = EP && (BLOCKS || (P.ep_grad && P.n_alpha <= DBW_ALPHA_SMEM_MAX)) && P.faces_alpha && P.g_faces_alpha;
  if (alpha_sums) for (int i = tid; i < P.n_alpha; i += NT) s_galpha[i] = 0.f;
  DbwMapDesc my_desc = {0, 0, 0, 0};
  if (tid < P.M) my_desc = P.map_table[tid];
  float my_alpha = 0.f;          // BLOCKS: this thread's opacity entry, stored with its map-table entry
  if (BLOCKS && P.faces_alpha && tid < P.n_alpha) my_alpha = __ldg(&P.faces_alpha[(size_t)view * P.alpha_stride + tid]);
  const int4 vbox = __ldg(reinterpret_cast<const int4*>(P.view_bbox) + view);      // in flight across the barrier
  const int vflags = __ldg(P.view_flags + view);
  __syncthreads();
  const f2 p = {s_ndc[xi - tx0], s_ndc[TILE_W + yi - ty0]};
  const int tx1 = min(tx0 + TILE_W, P.W) - 1, ty1 = min(ty0 + TILE_H, P.H) - 1;
  const float t_xmin = s_ndc[tx1 - tx0], t_xmax = s_ndc[0], t_ymin = s_ndc[TILE_W + ty1 - ty0], t_ymax = s_ndc[TILE_W];
  // tiles outside the union of the view's face boxes have nothing to rasterize: no scan
  const bool tile_empty = ord2f(vbox.x) > t_xmax || ord2f(vbox.y) < t_xmin || ord2f(vbox.z) > t_ymax || ord2f(vbox.w) < t_ymin;

  const int K = P.K;
  float4* const lA = s_dyn + tid;                                            // this thread's list column
  float* const lV = reinterpret_cast<float*>(s_dyn + (size_t)K * NT) + tid;
  int n = 0;

  // the slots this tile scans: its coarse bin's list when there is one, else every slot of the view
  const int* clist = nullptr;
  int nslots = tile_empty ? 0 : ((vflags & 1) ? 2 * P.F : P.F);
  if (P.cbin_list && !tile_empty) {
    const size_t b = (size_t)view * P.cbin_nx * P.cbin_ny + (size_t)(ty0 / DBW_CBIN) * P.cbin_nx + tx0 / DBW_CBIN;
    clist = P.cbin_list + b * 2 * P.F;
    nslots = __ldg(P.cbin_count + b);
  }
  const size_t slot_base = (size_t)view * 2 * P.F;
  const float4* bbox = P.bbox + slot_base;
  const float4* rec = P.rec + slot_base * 4;
  const bool dist_inside = (!P.clip_inside && P.sigma > 0.f) || (!BLOCKS && P.out_dists != nullptr);

  // stage the records of the `cnt` listed faces in shared memory, then test every pixel against every listed face
  auto raster_list = [&](int cnt) {
    // ---- stage the records of the listed faces in shared memory: one 64 B TMA bulk copy per face, all landing on s_bar
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // earlier generic reads of s_rec precede the async writes
    if (tid == 0) mbar_arrive_expect_tx(&s_bar, (uint32_t)cnt * 64u);
    for (int j = tid; j < cnt; j += NT) bulk_copy_g2s(&s_rec[j * 4], &rec[(size_t)s_slot[j] * 4], 64u, &s_bar);
    mbar_wait(&s_bar, bar_phase);
    bar_phase ^= 1u;
    // ---- per pixel: test every listed face, keep the K nearest (SURVEY A4, A5)
    if (live) {
      for (int j = 0; j < cnt; ++j) {
        const float4 b4 = s_bbox[j];
        if (p.x > b4.y || p.x < b4.x || p.y > b4.w || p.y < b4.z) continue;
        const TriGeom t = unpack_tri(s_rec[j * 4], s_rec[j * 4 + 1], s_rec[j * 4 + 2], s_rec[j * 4 + 3]);
        // cheap, exact part first: edge functions -> inside; pixels outside the face and beyond the halo leave here
        const Edges ed = eval_edges(p, t);
        if (!ed.inside && P.blur == 0.f) continue;      // hard pass: nothing outside a face can be within a zero halo
        float dist = 1.f; int edge = 0;
        const bool need_dist = !ed.inside || dist_inside || t.neighbor >= 0;
        if (need_dist) dist = tri_dist2_edge(p, t, edge);
        if (!ed.inside && dist >= P.blur) continue;
        const Bary b = bary_from_edges(ed, t, P.persp, P.clipb);
        if (b.pz < 0.f) continue;
        const int slot = s_slot[j];
        // a full list only admits what sorts before its last entry (the z-clipped halves first settle their exclusion rule)
        if (n == K && t.neighbor < 0 && !frag_key_less(__float_as_uint(b.pz + 0.f), slot, lA[(K - 1) * NT])) continue;
        // texture coordinates now, while the barycentrics are in registers: shading never re-derives geometry
        const size_t gs = slot_base + slot;
        f3 bu = b.bc;
        if (t.flags & 1) {
          const float* cv = P.conv + gs * 9;
          bu.x = b.bc.x * cv[0] + b.bc.y * cv[3] + b.bc.z * cv[6];
          bu.y = b.bc.x * cv[1] + b.bc.y * cv[4] + b.bc.z * cv[7];
          bu.z = b.bc.x * cv[2] + b.bc.y * cv[5] + b.bc.z * cv[8];
        }
        const float4 q0 = __ldg(&P.rec2[gs * 2]), q1 = __ldg(&P.rec2[gs * 2 + 1]);
        const float u = bu.x * q0.x + bu.y * q0.z + bu.z * q1.x;
        const float v = bu.x * q0.y + bu.y * q0.w + bu.z * q1.y;
        n = fraglist_offer(lA, lV, NT, n, K, b.pz, slot, edge, b.inside ? -dist : dist, dist, t.neighbor, u, v, __float_as_int(q1.z));
      }
    }
    // no barrier here: on the fast path nothing rewrites the list, and warps that finish early start shading (and hide
    // the texel latency of the others); the chunked path synchronises at its call site before refilling the list
  };

  // ---- bin: which face slots of the view touch the tile?  A slot is listed when its blur-expanded box overlaps the tile
  // AND no edge line of its triangle has the whole (halo-expanded) tile on its outer side.  Fast path: every batch of NT
  // slots is tested and compacted with NO block barrier in between (ballot + one shared atomic per warp); hits beyond the
  // list capacity are counted but not stored, and only then the chunked path below (barrier per batch) is taken.
  const float rx0 = t_xmin - P.sqrt_blur, rx1 = t_xmax + P.sqrt_blur, ry0 = t_ymin - P.sqrt_blur, ry1 = t_ymax + P.sqrt_blur;
  // (the chunked path scans in frag_order_key order: the coarse bin's list is in it, the view's 2F slots are mapped to it)
  const bool split = vflags & 1;
  auto scan_hit = [&](int& s, float4& bb) -> bool {
    if (s >= nslots) return false;
    if (clist) s = __ldg(clist + s);
    else if (split) s = frag_order_slot(s, P.F);
    bb = __ldg(&bbox[s]);
    if (bb.x > t_xmax || bb.y < t_xmin || bb.z > t_ymax || bb.w < t_ymin) return false;
    const float4 r0 = __ldg(&rec[(size_t)s * 4]);
    const float2 r1 = __ldg(reinterpret_cast<const float2*>(&rec[(size_t)s * 4 + 1]));
    return tri_overlaps_rect({r0.x, r0.y}, {r0.z, r0.w}, {r1.x, r1.y}, rx0, rx1, ry0, ry1);
  };
  // four batches per trip, their box loads issued together: the scan is a chain of L2 latencies otherwise
  for (int base = 0; base < nslots; base += 4 * NT) {
    float4 bb[4]; int sid[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = base + q * NT + tid;
      sid[q] = i < nslots ? (clist ? __ldg(clist + i) : i) : -1;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) bb[q] = sid[q] >= 0 ? __ldg(&bbox[sid[q]]) : make_float4(INFINITY, -INFINITY, INFINITY, -INFINITY);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int sl = sid[q];
      bool hit = !(bb[q].x > t_xmax || bb[q].y < t_xmin || bb[q].z > t_ymax || bb[q].w < t_ymin);
      if (hit) {
        const float4 r0 = __ldg(&rec[(size_t)sl * 4]);
        const float2 r1 = __ldg(reinterpret_cast<const float2*>(&rec[(size_t)sl * 4 + 1]));
        hit = tri_overlaps_rect({r0.x, r0.y}, {r0.z, r0.w}, {r1.x, r1.y}, rx0, rx1, ry0, ry1);
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m == 0u) continue;
      int wbase = 0;
      if (lane == 0) wbase = atomicAdd(&s_count, __popc(m));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      const int pos = wbase + __popc(m & ((1u << lane) - 1u));
      if (hit && pos < CAP) { s_slot[pos] = sl; s_bbox[pos] = bb[q]; }
    }
  }
  if (tid < P.M) s_desc[tid] = make_int4(my_desc.offset / 3, my_desc.height, my_desc.width, my_desc.reserved);
  for (int m = tid + NT; m < P.M; m += NT) { const DbwMapDesc d = P.map_table[m]; s_desc[m] = make_int4(d.offset / 3, d.height, d.width, d.reserved); }
  if (BLOCKS && P.faces_alpha) {
    if (tid < P.n_alpha) s_alpha[tid] = my_alpha;
    for (int i = tid + NT; i < P.n_alpha; i += NT) s_alpha[i] = __ldg(&P.faces_alpha[(size_t)view * P.alpha_stride + i]);
  }
  __syncthreads();
  const int total = s_count;
  if (total <= CAP) {
    // the warps above listed their hits in the order they won the atomic; where the offer order can matter (a view with
    // z-clipped slots, dbw_fraglist.cuh), the list is sorted into frag_order_key order first: each entry moves to its rank.
    // (Flagging the tiles that list a second half instead costs all views a shared store per hit in the scan: slower.)
    if (split && total > 1) {
      constexpr int PER = (CAP + NT - 1) / NT;
      int sl[PER], rk[PER]; float4 bx[PER];
#pragma unroll
      for (int r = 0; r < PER; ++r) {
        const int j = tid + r * NT;
        if (j < total) { sl[r] = s_slot[j]; bx[r] = s_bbox[j]; rk[r] = frag_order_rank(s_slot, total, j, P.F); }
      }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < PER; ++r)
        if (tid + r * NT < total) { s_slot[rk[r]] = sl[r]; s_bbox[rk[r]] = bx[r]; }
      __syncthreads();
    }
    if (total > 0) raster_list(total);
  } else {
    // chunked path (more than CAP faces touch this tile): re-scan in frag_order_key order, compacting each batch in order (a
    // block prefix over the warps' counts), and flush the list whenever it may overflow
    __shared__ int s_wcount[NT / 32];
    constexpr int BS = NT < CAP ? NT : CAP;          // slots scanned per batch: a batch never overflows an empty list
    int cnt = 0;                                     // entries listed (the same in every thread)
    for (int base = 0; base < nslots; base += BS) {
      float4 bb = make_float4(0, 0, 0, 0);
      int sl = base + tid;
      const bool hit = tid < BS && scan_hit(sl, bb);
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) s_wcount[warp] = __popc(m);
      __syncthreads();
      int pos = cnt;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) { const int c = s_wcount[w]; pos += w < warp ? c : 0; cnt += c; }
      if (hit) {
        pos += __popc(m & ((1u << lane) - 1u));
        s_slot[pos] = sl; s_bbox[pos] = bb;
      }
      __syncthreads();                // the batch is listed; s_wcount is read before the next batch writes it
      const bool last = base + BS >= nslots;
      if (cnt > CAP - BS || last) {
        raster_list(cnt);
        __syncthreads();              // every warp is done with the list before it is refilled
        cnt = 0;
      }
    }
  }

  float ep_sq = 0.f;          // this pixel's squared error (fused loss epilogue)
  float ep_g[4] = {0.f, 0.f, 0.f, 0.f};      // d loss / d (this render's RGBA) at the pixel (fused loss epilogue)
  int n_saved = 0;            // layers blended: those in front of the first fully opaque one
  if (live) {
  // ---- shade + blend the sorted fragments front to back (layered_rgb_blend, Appendix B)
  float occ = 1.f, r = 0.f, g = 0.f, bl = 0.f;
  float dep = 0.f;              // DEPTH: blended depth
  const size_t plane = (size_t)P.H * P.W;
  const size_t pix = (size_t)yi * P.W + xi;
  float ep_e[3] = {0.f, 0.f, 0.f}, ep_t[3] = {0.f, 0.f, 0.f};
  if (EP) {                     // the epilogue's environment / target pixels: in flight while the fragments are shaded
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      ep_e[c] = __ldg(P.ep_env + (size_t)view * 4 * plane + (size_t)c * plane + pix);
      ep_t[c] = __ldg(P.ep_target + (size_t)view * 3 * plane + (size_t)c * plane + pix);
    }
  }
#pragma unroll 1
  for (int k = 0; k < n; ++k) {
    if (BLOCKS && occ == 0.f) break;      // no per-layer output: every later layer contributes exactly 0
    const float4 e = lA[k * NT];
    const int bits = __float_as_int(e.y), slot = bits & DBW_FRAG_SLOT_MASK;
    const float d0 = e.z;
    if (!BLOCKS && P.topk) P.topk[((size_t)view * K + k) * plane + pix] = slot;
    if (!BLOCKS && P.out_dists) P.out_dists[((size_t)view * K + k) * plane + pix] = d0;
    if (DEPTH && Dz.zbuf) Dz.zbuf[((size_t)view * K + k) * plane + pix] = e.x;
    // behind a fully opaque fragment (fine phase: alpha = 1 inside a face): contributes exactly 0 (DEPTH with records: the layer
    // is still recorded, for the gradient of its zbuf; its weight is 0, so the blend is unchanged)
    if (occ == 0.f && !(DEPTH && P.frag)) continue;
    n_saved = k + 1;
    const float v = lV[k * NT];
    const int face = slot >= P.F ? slot - P.F : slot;
    Texel4 tx;
    fetch_color<BLOCKS>(P, e.w, v, s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT], tx);
    float a = frag_alpha(d0, P.sigma, P.clip_inside);
    if (P.faces_alpha) a *= BLOCKS ? s_alpha[alpha_index(P, 0, face)] : __ldg(&P.faces_alpha[alpha_index(P, view, face)]);
    if (!BLOCKS && P.face_shade) {          // flat shading: colour = texel * (ambient + diffuse * relu(n . l)) per (view, face)
      const float* m = P.face_shade + ((size_t)view * P.F + face) * 3;
      tx.color.x *= __ldg(m); tx.color.y *= __ldg(m + 1); tx.color.z *= __ldg(m + 2);
    }
    if (!BLOCKS && P.frag) {      // what the backward streams instead of re-deriving geometry and texels: two 16 B records
      const size_t fi = ((size_t)view * K + k) * plane + pix;
      P.frag[fi] = make_float4(e.y, e.w, v, d0);
      if (P.frag_rgb) P.frag_rgb[fi] = make_float4(tx.color.x, tx.color.y, tx.color.z, 0.f);
    }
    const float w = occ * a;
    r += w * tx.color.x; g += w * tx.color.y; bl += w * tx.color.z;
    if (DEPTH) dep += w * e.x;
    occ *= (1.f - a);
  }
  if (DEPTH && Dz.depth) Dz.depth[(size_t)view * plane + pix] = dep;
  if (!BLOCKS && P.nfrag) P.nfrag[(size_t)view * plane + pix] = (unsigned char)n_saved;
  for (int k = n; k < K; ++k) {
    if (!BLOCKS && P.topk) P.topk[((size_t)view * K + k) * plane + pix] = -1;
    if (!BLOCKS && P.out_dists) P.out_dists[((size_t)view * K + k) * plane + pix] = -1.f;
    if (DEPTH && Dz.zbuf) Dz.zbuf[((size_t)view * K + k) * plane + pix] = -1.f;
  }
  float* o = P.out_rgba + (size_t)view * 4 * plane + pix;
  const float fc[3] = {r + occ * P.bg0, g + occ * P.bg1, bl + occ * P.bg2};
  const float m = 1.f - occ;
  if (!EP) {
    o[0] = fc[0]; o[plane] = fc[1]; o[2 * plane] = fc[2]; o[3 * plane] = m;
  } else {
    // fused epilogue (same arithmetic as composite_mse_kernel): composite over the environment render, squared error
    // against the target, and the gradients of the MSE w.r.t. both layers -- out_rgba (when not NULL) receives
    // d loss / d (this render)
    float* ge = P.ep_g_env + (size_t)view * 4 * plane + pix;
    float gm = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float ec = ep_e[c];
      const float rc = fc[c] * m + (1.f - m) * ec;
      const float diff = rc - ep_t[c];
      ep_sq += diff * diff;
      if (P.ep_rec) P.ep_rec[(size_t)view * 3 * plane + (size_t)c * plane + pix] = rc;
      const float gr = 2.f * diff * P.ep_inv_count;
      ep_g[c] = gr * m;
      ge[(size_t)c * plane] = gr * (1.f - m);
      gm += gr * (fc[c] - ec);
    }
    ep_g[3] = gm;
    if (!BLOCKS && P.out_rgba) { o[0] = ep_g[0]; o[plane] = ep_g[1]; o[2 * plane] = ep_g[2]; o[3 * plane] = gm; }
    if (!P.ep_skip_env_alpha) ge[3 * plane] = 0.f;
  }
  }   // live
  if (BLOCKS || (EP && P.ep_grad)) epilogue_backward<BLOCKS>(P, lA, lV, NT, s_desc, s_galpha, live, n_saved, p, ep_g, view, lane, warp);
  if (EP) {
    // one atomic per warp into a strip of partial sums (the caller adds them up): no single hot address
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ep_sq += __shfl_xor_sync(0xffffffffu, ep_sq, off);
    if (lane == 0 && ep_sq != 0.f) {
      const unsigned cta = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;      // any spread over the strip will do
      atomicAdd(&P.ep_partials[(cta * (NT / 32) + warp) & P.ep_part_mask], ep_sq * P.ep_inv_count);
    }
  }
  if (alpha_sums) {
    __syncthreads();                 // one global atomic per (CTA, opacity entry), as in raster_backward_kernel
    for (int i = tid; i < P.n_alpha; i += NT) {
      const float v = s_galpha[i];
      if (v != 0.f) atomicAdd(&P.g_faces_alpha[(size_t)view * P.alpha_stride + i], v);
    }
  }
}

template <int NT, bool EP>
__global__ void __launch_bounds__(NT, NT <= 128 ? DBW_FWD_MINB : DBW_FWD_SMALLK_MINB) raster_forward_kernel(const RasterParams P) {
  raster_forward_body<NT, EP, false>(P);
}
__global__ void __launch_bounds__(128, DBW_FWD_MINB) blocks_loss_kernel(const RasterParams P) { raster_forward_body<128, true, true>(P); }
// the generic forward with the depth outputs (dbw_render_forward_depth)
template <int NT>
__global__ void __launch_bounds__(NT, NT <= 128 ? DBW_FWD_MINB : DBW_FWD_SMALLK_MINB) depth_forward_kernel(const RasterParams P, const DepthIO Dz) {
  raster_forward_body<NT, false, false, true>(P, Dz);
}

// ------------------------------------------------------------------------------------------------ hard single-layer forward
// K = 1, sigma = 0 (the environment pass, src/model/dbw.py:135-138,219; VizMeshRenderer's 4x supersampled renders,
// renderer.py:56-60): the nearest face that CONTAINS the pixel -- no halo, no distances, no per-pixel list.  The generic
// kernel spends two thirds of its instructions on machinery this case does not need (a scan of all 2F slots per tile, TMA
// staging, the shared-memory fragment lists); here a tile tests only the view's visible slots (face_setup's vis_list), keeps
// the best fragment in registers and derives its texture coordinates once, after the walk.  Results (image, records, ids) are
// identical to the generic kernel's: same edge functions, same (depth, slot) order.
#define HARD_NT 256
#define HARD_CAP 64
// Outputs of the resolving variant (VIZ): the settings describe the 4H x 4W sample grid, these the H x W frames.
struct VizOut {
  const float* bkg; int bkg_stride;    // (1 or B, 3, H, W) background composited under the frame, or NULL; stride 0 or 3HW
  float* rgba;                         // (B, 4, H, W) resolved RGBA (RGB composited when bkg), or NULL
  unsigned char* rgb8;                 // (B, H, W, 3) uint8 frames, or NULL
};
__device__ __forceinline__ void hard_viz_resolve(const RasterParams& P, const VizOut& Z, bool live, int view, int xi, int yi,
                                                 int lane, const float (&c)[4]);
// texture coordinates (its record is read back from global memory: the tile list may have been recycled), colour and opacity
// of the winning fragment of a hard single-layer pass.  The same operations as the tail of the plain kernel below, which keeps
// its own copy: routing it through this function changes its instruction schedule (same registers, same results).
struct HardShade { f3 color; float u, v, a; int map_id; };
__device__ __forceinline__ HardShade hard_shade(const RasterParams& P, const int4* s_desc, int view, int best_slot, f3 best_bc) {
  const size_t gs = (size_t)view * 2 * P.F + best_slot;
  f3 bu = best_bc;
  if (__float_as_int(__ldg(&P.rec[gs * 4 + 2]).w) & 1) {
    const float* cv = P.conv + gs * 9;
    bu.x = best_bc.x * cv[0] + best_bc.y * cv[3] + best_bc.z * cv[6];
    bu.y = best_bc.x * cv[1] + best_bc.y * cv[4] + best_bc.z * cv[7];
    bu.z = best_bc.x * cv[2] + best_bc.y * cv[5] + best_bc.z * cv[8];
  }
  const float4 q0 = __ldg(&P.rec2[gs * 2]), q1 = __ldg(&P.rec2[gs * 2 + 1]);
  HardShade w;
  w.u = bu.x * q0.x + bu.y * q0.z + bu.z * q1.x;
  w.v = bu.x * q0.y + bu.y * q0.w + bu.z * q1.y;
  w.map_id = __float_as_int(q1.z);
  Texel4 tx;
  fetch_color(P, w.u, w.v, s_desc[w.map_id], tx);
  const int face = best_slot >= P.F ? best_slot - P.F : best_slot;
  w.a = 1.f;                                         // inside a face of a hard pass: opacity 1 (x the face's entry)
  if (P.faces_alpha) w.a *= __ldg(&P.faces_alpha[alpha_index(P, view, face)]);
  if (P.face_shade) {
    const float* m = P.face_shade + ((size_t)view * P.F + face) * 3;
    tx.color.x *= __ldg(m); tx.color.y *= __ldg(m + 1); tx.color.z *= __ldg(m + 2);
  }
  w.color = tx.color;
  return w;
}

// Inputs of the Phong-shaded variants (dbw_render_forward_phong): a kernel argument of their own, so that RasterParams -- and
// with it every other kernel -- is unchanged.
struct PhongIn {
  const float* verts;        // (V,3) world-space vertices
  const float* normals;      // (V,3) vertex normals (dbw_vertex_normals)
  const int* faces;          // (F,3)
  const float* R; const float* T;   // (B,3,3), (B,3): the per-view light direction and camera centre
  DbwPhongShading light;
};
// hard_shade with the texel Phong-shaded: vertex normal and world position interpolated with the same barycentrics bu as the
// texture coordinates.  A copy of hard_shade rather than a branch in it, so that the existing kernels keep their code.
__device__ __forceinline__ HardShade hard_shade_phong(const RasterParams& P, const PhongIn& L, const int4* s_desc, int view,
                                                      int best_slot, f3 best_bc) {
  const size_t gs = (size_t)view * 2 * P.F + best_slot;
  f3 bu = best_bc;
  if (__float_as_int(__ldg(&P.rec[gs * 4 + 2]).w) & 1) {
    const float* cv = P.conv + gs * 9;
    bu.x = best_bc.x * cv[0] + best_bc.y * cv[3] + best_bc.z * cv[6];
    bu.y = best_bc.x * cv[1] + best_bc.y * cv[4] + best_bc.z * cv[7];
    bu.z = best_bc.x * cv[2] + best_bc.y * cv[5] + best_bc.z * cv[8];
  }
  const float4 q0 = __ldg(&P.rec2[gs * 2]), q1 = __ldg(&P.rec2[gs * 2 + 1]);
  HardShade w;
  w.u = bu.x * q0.x + bu.y * q0.z + bu.z * q1.x;
  w.v = bu.x * q0.y + bu.y * q0.w + bu.z * q1.y;
  w.map_id = __float_as_int(q1.z);
  Texel4 tx;
  fetch_color(P, w.u, w.v, s_desc[w.map_id], tx);
  const int face = best_slot >= P.F ? best_slot - P.F : best_slot;
  w.a = 1.f;
  if (P.faces_alpha) w.a *= __ldg(&P.faces_alpha[alpha_index(P, view, face)]);
  const int i0 = __ldg(L.faces + 3 * face), i1 = __ldg(L.faces + 3 * face + 1), i2 = __ldg(L.faces + 3 * face + 2);
  DbwVec3 n, p;
  n.x = bu.x * __ldg(L.normals + 3 * i0) + bu.y * __ldg(L.normals + 3 * i1) + bu.z * __ldg(L.normals + 3 * i2);
  n.y = bu.x * __ldg(L.normals + 3 * i0 + 1) + bu.y * __ldg(L.normals + 3 * i1 + 1) + bu.z * __ldg(L.normals + 3 * i2 + 1);
  n.z = bu.x * __ldg(L.normals + 3 * i0 + 2) + bu.y * __ldg(L.normals + 3 * i1 + 2) + bu.z * __ldg(L.normals + 3 * i2 + 2);
  p.x = bu.x * __ldg(L.verts + 3 * i0) + bu.y * __ldg(L.verts + 3 * i1) + bu.z * __ldg(L.verts + 3 * i2);
  p.y = bu.x * __ldg(L.verts + 3 * i0 + 1) + bu.y * __ldg(L.verts + 3 * i1 + 1) + bu.z * __ldg(L.verts + 3 * i2 + 1);
  p.z = bu.x * __ldg(L.verts + 3 * i0 + 2) + bu.y * __ldg(L.verts + 3 * i1 + 2) + bu.z * __ldg(L.verts + 3 * i2 + 2);
  float Rv[9], Tv[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) Rv[k] = __ldg(L.R + 9 * view + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) Tv[k] = __ldg(L.T + 3 * view + k);
  DbwVec3 light, camera;
  shade_view_setup(L.light, Rv, Tv, light, camera);
  const DbwVec3 c = shade_phong(L.light, shade_v3(tx.color.x, tx.color.y, tx.color.z), n, p, light, camera);
  w.color.x = c.x; w.color.y = c.y; w.color.z = c.z;
  return w;
}

// PHONG: the Phong-shaded variants (phong_hard_forward_kernel, phong_resolve_hard_viz_kernel), which shade the winner with
// hard_shade_phong; the code of the other instantiations is unchanged.  DEPTH (depth_hard_forward_kernel): also the winner's
// depth (DepthIO.zbuf, -1 where nothing is hit) and its depth times its opacity (DepthIO.depth, 0 where nothing is hit).
template <bool VIZ, bool PHONG = false, bool DEPTH = false>
__device__ __forceinline__ void hard_forward_body(const RasterParams& P, const VizOut& Z, const PhongIn& L = PhongIn{},
                                                  const DepthIO& Dz = DepthIO{}) {
  static_assert(!DEPTH || (!VIZ && !PHONG), "depth is a plain hard render's");
  __shared__ float4 s_bbox[HARD_CAP];
  __shared__ float4 s_rec[HARD_CAP * 4];
  __shared__ int s_slot[HARD_CAP];
  __shared__ int s_count;
  __shared__ float s_ndc[32];
  extern __shared__ float4 s_dyn[];            // the map table
  int4* const s_desc = reinterpret_cast<int4*>(s_dyn);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = blockIdx.x;
  const int tile_y = centre_out(blockIdx.z, gridDim.z);
  const int tx0 = blockIdx.y * 16, ty0 = tile_y * 16;
  const int xi = tx0 + (warp & 1) * 8 + (lane & 7);
  const int yi = ty0 + (warp >> 1) * 4 + (lane >> 3);
  int row_lo = 0, row_hi = P.H;
  if (P.view_rows) { row_lo = P.view_rows[view * 2]; row_hi = P.view_rows[view * 2 + 1]; }
  if (ty0 >= row_hi || ty0 + 16 <= row_lo) return;
  const bool live = xi < P.W && yi < P.H && yi >= row_lo && yi < row_hi;
  if (tid < 16) s_ndc[tid] = pix_to_ndc(P.W - 1 - min(tx0 + tid, P.W - 1), P.W, P.H);
  else if (tid < 32) s_ndc[tid] = pix_to_ndc(P.H - 1 - min(ty0 + tid - 16, P.H - 1), P.H, P.W);
  if (tid == 0) s_count = 0;
  const int nvis = __ldg(P.view_nvis + view);
  const size_t slot_base = (size_t)view * 2 * P.F;
  const int* vis = P.vis_list + slot_base;
  for (int m = tid; m < P.M; m += HARD_NT) { const DbwMapDesc d = P.map_table[m]; s_desc[m] = make_int4(d.offset / 3, d.height, d.width, d.reserved); }
  __syncthreads();
  const f2 p = {s_ndc[xi - tx0], s_ndc[16 + yi - ty0]};
  const int tx1 = min(tx0 + 16, P.W) - 1, ty1 = min(ty0 + 16, P.H) - 1;
  const float t_xmin = s_ndc[tx1 - tx0], t_xmax = s_ndc[0], t_ymin = s_ndc[16 + ty1 - ty0], t_ymax = s_ndc[16];
  // the nearest containing fragment of this pixel
  unsigned best_pz = 0xffffffffu; int best_slot = 0x7fffffff, best_j = -1;
  f3 best_bc = {0.f, 0.f, 0.f};
  for (int base = 0; base < nvis; base += HARD_NT) {
    // ---- which visible slots touch the tile?  (box overlap, then no edge line with the whole tile on its outer side)
    const int i = base + tid;
    bool hit = false; int slot = 0; float4 bb = make_float4(0, 0, 0, 0);
    if (i < nvis) {
      slot = __ldg(vis + i);
      bb = __ldg(&P.bbox[slot_base + slot]);
      hit = !(bb.x > t_xmax || bb.y < t_xmin || bb.z > t_ymax || bb.w < t_ymin);
      if (hit) {
        const float4 r0 = __ldg(&P.rec[(slot_base + slot) * 4]);
        const float2 r1 = __ldg(reinterpret_cast<const float2*>(&P.rec[(slot_base + slot) * 4 + 1]));
        hit = tri_overlaps_rect({r0.x, r0.y}, {r0.z, r0.w}, {r1.x, r1.y}, t_xmin, t_xmax, t_ymin, t_ymax);
      }
    }
    // lists of at most HARD_CAP entries per round: ballots in warp order, the overflow is taken in further rounds
    bool pending = hit;
    while (__syncthreads_or(pending)) {
      const unsigned m = __ballot_sync(0xffffffffu, pending);
      int wbase = 0;
      if (lane == 0 && m) wbase = atomicAdd(&s_count, __popc(m));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      const int pos = wbase + __popc(m & ((1u << lane) - 1u));
      if (pending && pos < HARD_CAP) {
        s_slot[pos] = slot; s_bbox[pos] = bb;
        const float4* r = &P.rec[(slot_base + slot) * 4];
        s_rec[pos * 4] = __ldg(r); s_rec[pos * 4 + 1] = __ldg(r + 1); s_rec[pos * 4 + 2] = __ldg(r + 2); s_rec[pos * 4 + 3] = __ldg(r + 3);
        pending = false;
      }
      __syncthreads();
      const int cnt = min(s_count, HARD_CAP);
      if (live) {
        for (int j = 0; j < cnt; ++j) {
          const float4 b4 = s_bbox[j];
          if (p.x > b4.y || p.x < b4.x || p.y > b4.w || p.y < b4.z) continue;
          const TriGeom t = unpack_tri(s_rec[j * 4], s_rec[j * 4 + 1], s_rec[j * 4 + 2], s_rec[j * 4 + 3]);
          const Edges ed = eval_edges(p, t);
          if (!ed.inside) continue;
          const Bary b = bary_from_edges(ed, t, P.persp, P.clipb);
          if (b.pz < 0.f) continue;
          const unsigned pzb = __float_as_uint(b.pz + 0.f);
          const int sl = s_slot[j];
          if (pzb < best_pz || (pzb == best_pz && sl < best_slot)) { best_pz = pzb; best_slot = sl; best_bc = b.bc; best_j = j; }
        }
      }
      __syncthreads();
      if (tid == 0) s_count = 0;
      // (the next round's atomics come after the barrier at the top of the loop)
    }
  }
  if (VIZ) {
    // every lane takes part in the resolve's shuffles: a sample outside the image belongs to a frame pixel outside it
    float c[4] = {P.bg0, P.bg1, P.bg2, 0.f};
    if (live && best_j >= 0) {
      const HardShade w = PHONG ? hard_shade_phong(P, L, s_desc, view, best_slot, best_bc) : hard_shade(P, s_desc, view, best_slot, best_bc);
      const float occ = 1.f - w.a;
      c[0] = w.a * w.color.x + occ * P.bg0; c[1] = w.a * w.color.y + occ * P.bg1; c[2] = w.a * w.color.z + occ * P.bg2; c[3] = w.a;
    }
    hard_viz_resolve(P, Z, live, view, xi, yi, lane, c);
    return;
  }
  if (!live) return;
  const size_t plane = (size_t)P.H * P.W;
  const size_t pix = (size_t)yi * P.W + xi;
  float* o = P.out_rgba + (size_t)view * 4 * plane + pix;
  if (best_j < 0) {
    o[0] = P.bg0; o[plane] = P.bg1; o[2 * plane] = P.bg2; o[3 * plane] = 0.f;
    if (P.nfrag) P.nfrag[(size_t)view * plane + pix] = 0;
    if (P.topk) P.topk[(size_t)view * plane + pix] = -1;
    if (DEPTH && Dz.zbuf) Dz.zbuf[(size_t)view * plane + pix] = -1.f;
    if (DEPTH && Dz.depth) Dz.depth[(size_t)view * plane + pix] = 0.f;
    return;
  }
  if constexpr (PHONG) {         // no fragment records: a phong render has no backward
    const HardShade w = hard_shade_phong(P, L, s_desc, view, best_slot, best_bc);
    if (P.topk) P.topk[(size_t)view * plane + pix] = best_slot;
    const float occ = 1.f - w.a;
    o[0] = w.a * w.color.x + occ * P.bg0; o[plane] = w.a * w.color.y + occ * P.bg1; o[2 * plane] = w.a * w.color.z + occ * P.bg2;
    o[3 * plane] = w.a;
    return;
  }
  // texture coordinates of the winner (its record is read back from global memory: the tile list may have been recycled)
  const size_t gs = slot_base + best_slot;
  f3 bu = best_bc;
  if (__float_as_int(__ldg(&P.rec[gs * 4 + 2]).w) & 1) {
    const float* cv = P.conv + gs * 9;
    bu.x = best_bc.x * cv[0] + best_bc.y * cv[3] + best_bc.z * cv[6];
    bu.y = best_bc.x * cv[1] + best_bc.y * cv[4] + best_bc.z * cv[7];
    bu.z = best_bc.x * cv[2] + best_bc.y * cv[5] + best_bc.z * cv[8];
  }
  const float4 q0 = __ldg(&P.rec2[gs * 2]), q1 = __ldg(&P.rec2[gs * 2 + 1]);
  const float u = bu.x * q0.x + bu.y * q0.z + bu.z * q1.x;
  const float v = bu.x * q0.y + bu.y * q0.w + bu.z * q1.y;
  const int map_id = __float_as_int(q1.z);
  Texel4 tx;
  fetch_color(P, u, v, s_desc[map_id], tx);
  const int face = best_slot >= P.F ? best_slot - P.F : best_slot;
  float a = 1.f;                                     // inside a face of a hard pass: opacity 1 (x the face's entry)
  if (P.faces_alpha) a *= __ldg(&P.faces_alpha[alpha_index(P, view, face)]);
  if (P.face_shade) {
    const float* m = P.face_shade + ((size_t)view * P.F + face) * 3;
    tx.color.x *= __ldg(m); tx.color.y *= __ldg(m + 1); tx.color.z *= __ldg(m + 2);
  }
  if (P.frag) {
    const size_t fi = (size_t)view * plane + pix;
    P.frag[fi] = make_float4(__int_as_float(best_slot | (map_id << DBW_FRAG_MAP_SHIFT)), u, v, -1.f);
    if (P.frag_rgb) P.frag_rgb[fi] = make_float4(tx.color.x, tx.color.y, tx.color.z, 0.f);
    P.nfrag[fi] = 1;
  }
  if (P.topk) P.topk[(size_t)view * plane + pix] = best_slot;
  const float occ = 1.f - a;
  o[0] = a * tx.color.x + occ * P.bg0; o[plane] = a * tx.color.y + occ * P.bg1; o[2 * plane] = a * tx.color.z + occ * P.bg2;
  o[3 * plane] = a;
  if (DEPTH) {
    const float z = __uint_as_float(best_pz);
    if (Dz.zbuf) Dz.zbuf[(size_t)view * plane + pix] = z;
    if (Dz.depth) Dz.depth[(size_t)view * plane + pix] = a * z;
  }
}

__global__ void __launch_bounds__(HARD_NT, 5) raster_hard_forward_kernel(const RasterParams P) { hard_forward_body<false>(P, VizOut{}); }
// the hard single-layer forward with the depth outputs (dbw_render_forward_depth)
__global__ void __launch_bounds__(HARD_NT, 5) depth_hard_forward_kernel(const RasterParams P, const DepthIO Dz) {
  hard_forward_body<false, false, true>(P, VizOut{}, PhongIn{}, Dz);
}

// The resolving variant renders the VizMeshRenderer frame (hard render on the 4H x 4W sample grid, avg_pool2d(., 4)) without
// the sample image: a warp's 8 x 4 samples are the 4 x 4 samples of two frame pixels, which its lanes sum in registers.
__global__ void __launch_bounds__(HARD_NT, 5) resolve_hard_viz_kernel(const RasterParams P, const VizOut Z) { hard_forward_body<true>(P, Z); }

// Phong-shaded hard render (dbw_render_forward_phong, factor 1) and its resolving variant (factor 4)
__global__ void __launch_bounds__(HARD_NT, 5) phong_hard_forward_kernel(const RasterParams P, const PhongIn L) {
  hard_forward_body<false, true>(P, VizOut{}, L);
}
__global__ void __launch_bounds__(HARD_NT, 5) phong_resolve_hard_viz_kernel(const RasterParams P, const VizOut Z, const PhongIn L) {
  hard_forward_body<true, true>(P, Z, L);
}

// The 16 samples of a frame pixel are lanes (g + c) + 8 r, r, c in [0, 4), g = 0 or 4.  Each sum runs in avg_pool2d's order
// (dbw_viz_math.cuh), so the frame equals avg_pool2d(render at 4H x 4W, 4) bit for bit.
__device__ __forceinline__ void hard_viz_resolve(const RasterParams& P, const VizOut& Z, bool live, int view, int xi, int yi,
                                                 int lane, const float (&c)[4]) {
  const int g = lane & 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) acc[ch] = dbw_viz_box_add(acc[ch], __shfl_sync(0xffffffffu, c[ch], r * 8 + g + k));
  if (!live || (lane & ~4)) return;
  const int H = P.H >> 2, W = P.W >> 2;
  const size_t plane = (size_t)H * W, pix = (size_t)(yi >> 2) * W + (xi >> 2);
  float f[4];
#pragma unroll
  for (int ch = 0; ch < 4; ++ch) f[ch] = dbw_viz_box_mean(acc[ch]);
  if (Z.bkg) {
    const float* b = Z.bkg + (size_t)view * Z.bkg_stride + pix;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) f[ch] = dbw_viz_composite(f[ch], f[3], __ldg(b + ch * plane));
  }
  if (Z.rgba) {
    float* o = Z.rgba + (size_t)view * 4 * plane + pix;
    o[0] = f[0]; o[plane] = f[1]; o[2 * plane] = f[2]; o[3 * plane] = f[3];
  }
  if (Z.rgb8) {
    unsigned char* o = Z.rgb8 + ((size_t)view * plane + pix) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch] = dbw_viz_u8(f[ch]);
  }
}

// ------------------------------------------------------------------------------------------------ backward
// Warp-aggregated accumulation: lanes of a warp that hold a contribution for the same key (face slot) are summed with
// shuffles and ONE lane issues the atomics -- a 16x16 tile typically sees 1-3 distinct faces per layer, so this
// removes the same-address contention that otherwise serialises the L2 atomic units (every pixel of a big face hitting
// the same 9 floats).  Must be called by all 32 lanes (key < 0: nothing to add).
// Transposed multi-value warp reduction: NP (power of two) values per lane are summed over the 32 lanes with
// NP-1 + (5 - log2 NP) shuffles instead of 5*NP -- at every level a lane hands HALF of its partial sums to its partner
// and keeps the other half, so the totals end up spread over the warp: lane l returns the total of value l >> (5 - log2 NP).
// The totals are then written by NP different lanes in ONE (predicated) atomic instruction instead of NP sequential ones.
template <int NP>
__device__ __forceinline__ float warp_sum_spread(float (&x)[NP], int lane) {
  static_assert(NP == 1 || NP == 2 || NP == 4 || NP == 8 || NP == 16 || NP == 32, "NP must be a power of two <= 32");
  constexpr int L = NP == 1 ? 0 : NP == 2 ? 1 : NP == 4 ? 2 : NP == 8 ? 3 : NP == 16 ? 4 : 5;
#pragma unroll
  for (int l = 0; l < 5; ++l) {
    const int o = 16 >> l;
    if (l < L) {
      const int c = NP >> (l + 1);
      const bool upper = (lane & o) != 0;
      // constant trip count: the inner loop is unrolled before the outer one, and a bound that depends on l would leave
      // it a loop with run-time indices into x -- which puts x in local memory
#pragma unroll
      for (int j = 0; j < NP / 2; ++j) {
        if (j >= c) break;
        const float send = upper ? x[j] : x[j + c];
        const float keep = upper ? x[j + c] : x[j];
        x[j] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    } else {
      x[0] += __shfl_xor_sync(0xffffffffu, x[0], o);
    }
  }
  return x[0];
}
template <int N> struct Pow2Ceil { static constexpr int v = N <= 1 ? 1 : N <= 2 ? 2 : N <= 4 ? 4 : N <= 8 ? 8 : N <= 16 ? 16 : 32; };
template <int NP> struct SpreadShift { static constexpr int v = NP == 1 ? 5 : NP == 2 ? 4 : NP == 4 ? 3 : NP == 8 ? 2 : NP == 16 ? 1 : 0; };

template <int N>
__device__ __forceinline__ void warp_agg_add(float* __restrict__ dst, int stride, int key, const float (&v)[N], int lane) {
  constexpr int NP = Pow2Ceil<N>::v, SH = SpreadShift<NP>::v;
  unsigned todo = __ballot_sync(0xffffffffu, key >= 0);
  while (todo) {
    const int leader = __ffs(todo) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = (key == lk);
    const unsigned grp = __ballot_sync(0xffffffffu, mine);
    if (__popc(grp) <= DBW_AGG_MIN) {              // (almost) alone: plain atomics are cheaper than a reduction
      if (mine) {
#pragma unroll
        for (int i = 0; i < N; ++i) if (v[i] != 0.f) atomicAdd(dst + (size_t)lk * stride + i, v[i]);
      }
    } else {
      float x[NP];
#pragma unroll
      for (int i = 0; i < NP; ++i) x[i] = (i < N && mine) ? v[i] : 0.f;
      const float r = warp_sum_spread<NP>(x, lane);
      const int idx = lane >> SH;
      if ((lane & ((1 << SH) - 1)) == 0 && idx < N && r != 0.f) atomicAdd(dst + (size_t)lk * stride + idx, r);
    }
    todo &= ~grp;
  }
}

// Texture-gradient scatter of one fragment: 4 bilinear taps x RGB, i.e. the colour gradient g times the tap weights w.
// Only those 7 floats are carried; the 12 products are formed where they are consumed, so the scatter keeps no
// 12-float array live across the fragment loop (which spilled to local memory).  Under magnification (the environment
// maps: several pixels per texel) the lanes of a warp fall into a few groups that share a 2x2 texel footprint.
// Groups of >= DBW_TEX_AGG_MIN lanes (found with one match.any) are reduced (16-wide spread reduction: total i lands in
// lane 2i and is added to channel i % 3 of tap i / 3); the other lanes issue plain vector reds.  On an H100 SXM, 4 lanes
// beat 8: 0.495 vs 0.504 ms for the dtu environment backward, 1.19 vs 1.25 ms for the blocks backward (per step).
#ifndef DBW_TEX_AGG_MIN
#define DBW_TEX_AGG_MIN 4
#endif
// Cell maps (DbwMapDesc.reserved != 0): a lane first merges its taps that share a cell (one cell carries all four weights
// for 49 of 64 footprints at f = 8) and issues one red.v4 per distinct cell instead of four, one tap slot per round, into
// one of DBW_CELL_GRAD_COPIES copies of the cell gradients (cell_grad_copy): a cell collects what 64 texels did, and with a
// single copy the reds of all the warps that cover it serialise at the L2.
//  - MATCH (single-layer passes: the environment maps, magnified, a warp often inside one cell): the lanes of every group of
//    >= DBW_CELL_AGG_MIN lanes found by match.any are warp-reduced first and their leader issues one red.v4.
//  - otherwise (the blocks pass): no warp reduction.  On an H100 at 400 W (dtu, blocks backward): 1.12 ms, against 1.27 ms
//    with the groups found in lane order and reduced, and 1.25 ms for the texel-space scatter of atlas maps.
#ifndef DBW_CELL_AGG_MIN
#define DBW_CELL_AGG_MIN 4
#endif
template <bool MATCH>
__device__ __forceinline__ void warp_cell_scatter(float4* __restrict__ gm, int k00, int k01, int k10, int k11,
                                                  const float (&g)[3], const float (&w)[4], int lane) {
  // merge this lane's taps that share a cell (kept in the first of them; k = -1: no tap)
  float m00 = w[0], m01 = w[1], m10 = w[2], m11 = w[3];
  if (k01 >= 0 && k01 == k00) { m00 += m01; k01 = -1; }
  if (k10 >= 0 && k10 == k00) { m00 += m10; k10 = -1; }
  if (k11 >= 0 && k11 == k00) { m00 += m11; k11 = -1; }
  else if (k11 >= 0 && k11 == k01) { m01 += m11; k11 = -1; }
  else if (k11 >= 0 && k11 == k10) { m10 += m11; k11 = -1; }
  // one tap slot per round, the slots rotated through registers (a rolled loop: the scatter stays small)
#pragma unroll 1
  while (__any_sync(0xffffffffu, (k00 & k01 & k10 & k11) != -1)) {
    const int key = k00;
    const float v0 = g[0] * m00, v1 = g[1] * m00, v2 = g[2] * m00;
    // groups to reduce: one bit per group, its leader; `big`: this lane's value goes into a group sum
    unsigned todo = 0;
    bool big = false;
    if (MATCH) {
      const unsigned grp = __match_any_sync(0xffffffffu, key);
      big = key >= 0 && __popc(grp) >= DBW_CELL_AGG_MIN;
      todo = __ballot_sync(0xffffffffu, big && (__ffs(grp) - 1) == lane);
    }
    while (todo) {
      const int leader = __ffs(todo) - 1;
      const int lk = __shfl_sync(0xffffffffu, key, leader);
      const bool mine = big && key == lk;
      float x[4] = {mine ? v0 : 0.f, mine ? v1 : 0.f, mine ? v2 : 0.f, 0.f};
      const float r = warp_sum_spread<4>(x, lane);          // total c in lanes 8c .. 8c + 7
      const float r0 = __shfl_sync(0xffffffffu, r, 0), r1 = __shfl_sync(0xffffffffu, r, 8), r2 = __shfl_sync(0xffffffffu, r, 16);
      if (lane == leader) red_add_v4(gm + lk, r0, r1, r2);
      todo &= todo - 1;
    }
    if (key >= 0 && !big) red_add_v4(gm + key, v0, v1, v2);
    k00 = k01; k01 = k10; k10 = k11; k11 = -1;
    m00 = m01; m01 = m10; m10 = m11;
  }
}

// cells: this lane's map is a cell map (the taps are cell indices).  A warp with any such lane takes the cell path for all
// its lanes: it is correct for texel taps too (a lane's four texels are distinct, so nothing merges), and only one of the two
// paths is live at a time.
// the copy of the cell-map gradients a warp adds into (re-derived where it is used: no register held across the loops).
// Neighbouring CTAs and the warps of a CTA cover neighbouring pixels, i.e. mostly the same cells, and spread over the copies.
__device__ __forceinline__ float4* cell_grad_copy(const RasterParams& P, int warp) {
  if (!P.g_cells) return P.g_maps4;
  const unsigned c = (blockIdx.y + 3 * blockIdx.z + 5 * blockIdx.x + 2 * warp) & (DBW_CELL_GRAD_COPIES - 1);
  return P.g_cells + (size_t)c * P.n_cells;
}
template <bool K1>
__device__ __forceinline__ void warp_tex_scatter(const RasterParams& P, int key, int i01, int i10, int i11, bool cells,
                                                 const float (&g)[3], const float (&w)[4], int lane, int warp) {
  float4* const gm = P.g_maps4;
  if (__any_sync(0xffffffffu, key >= 0 && cells)) {
    warp_cell_scatter<K1>(cell_grad_copy(P, warp), key, i01, i10, i11, g, w, lane);
    return;
  }
  const unsigned grp_mine = __match_any_sync(0xffffffffu, key);
  const bool big = key >= 0 && __popc(grp_mine) >= DBW_TEX_AGG_MIN;
  // one bit per group to reduce: its lowest lane
  unsigned todo = __ballot_sync(0xffffffffu, big && (__ffs(grp_mine) - 1) == lane);
  while (todo) {
    const int leader = __ffs(todo) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = big && key == lk;
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = (i < 12 && mine) ? g[i % 3] * w[i / 3] : 0.f;
    const float r = warp_sum_spread<16>(x, lane);
    // the footprint (i00 = key, i01, i10, i11) is the same for every lane of the group: fetch it from the leader
    const int l01 = __shfl_sync(0xffffffffu, i01, leader), l10 = __shfl_sync(0xffffffffu, i10, leader);
    const int l11 = __shfl_sync(0xffffffffu, i11, leader);
    const int idx = lane >> 1, tap = idx / 3, ch = idx - tap * 3;
    const int texel = tap == 0 ? lk : (tap == 1 ? l01 : (tap == 2 ? l10 : l11));
    if ((lane & 1) == 0 && idx < 12 && texel >= 0 && r != 0.f) atomicAdd(reinterpret_cast<float*>(gm + texel) + ch, r);
    todo &= todo - 1;
  }
  if (key >= 0 && !big) {
    red_add_v4(gm + key, g[0] * w[0], g[1] * w[0], g[2] * w[0]);
    if (i01 >= 0) red_add_v4(gm + i01, g[0] * w[1], g[1] * w[1], g[2] * w[1]);
    if (i10 >= 0) red_add_v4(gm + i10, g[0] * w[2], g[1] * w[2], g[2] * w[2]);
    if (i11 >= 0) red_add_v4(gm + i11, g[0] * w[3], g[1] * w[3], g[2] * w[3]);
  }
}

// Single-value aggregation keyed by an opacity entry: lanes sharing the key are summed with a 5-step butterfly and one lane
// issues the atomic.  A patch usually sees one or two blocks per layer, so this loop runs once or twice.
__device__ __forceinline__ void warp_agg_add1(float* __restrict__ dst, int key, float v, int lane) {
  unsigned todo = __ballot_sync(0xffffffffu, key >= 0);
  while (todo) {
    const int leader = __ffs(todo) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = (key == lk);
    const unsigned grp = __ballot_sync(0xffffffffu, mine);
    float x = mine ? v : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == leader && x != 0.f) atomicAdd(dst + lk, x);
    todo &= ~grp;
  }
}

// Distance-path vertex gradient of one layer, keyed by (triangle slot, closest edge): 4 values = (x, y) of the edge's two
// vertices.  Vertex pair of the edge: 0 = (v0, v1), 1 = (v0, v2), 2 = (v1, v2); vertex j's (x, y) live at floats 3j, 3j+1.
__device__ __forceinline__ void warp_agg_add_edge(float* __restrict__ g_tri, int key, const float (&v)[4], int lane) {
  // A patch's halo fragments of one layer lie along many edges, mostly one or two lanes per (slot, edge): every lane adds
  // its four values with plain atomics, all in the same pass.  Finding the groups first and reducing them one after the
  // other (a ballot, a shuffle and a ballot per group before any atomic) cost more than the atomics it saved: on an H100
  // (700 W) at dtu, 2.05 ms for the fused blocks kernel with groups of more than 2 lanes reduced, 2.01 ms with more than
  // 4, 1.88 ms with none
  if (key >= 0) {
    const int edge = key & 3;
    const int ia = edge == 2 ? 3 : 0, ib = edge == 0 ? 3 : 6;
    float* d = g_tri + (size_t)(key >> 2) * 9;
    if (v[0] != 0.f) atomicAdd(d + ia, v[0]);
    if (v[1] != 0.f) atomicAdd(d + ia + 1, v[1]);
    if (v[2] != 0.f) atomicAdd(d + ib, v[2]);
    if (v[3] != 0.f) atomicAdd(d + ib + 1, v[3]);
  }
}

// Barycentric-path gradient of one fragment with colour gradient (gcx, gcy, gcz): colour -> (ix, iy) -> (u, v) ->
// barycentrics -> vertices (grid_sample backward + A6).  Writes the slot's 9 vertex gradients; returns true when the face
// is z-clipped and gc9 holds the gradient of its conversion matrix too.
__device__ __forceinline__ bool bary_frag_backward(const RasterParams& P, size_t gsl, f2 p, const Shade& s, const Texel4& tx,
                                                   float gcx, float gcy, float gcz, float (&gv9)[9], float (&gc9)[9]) {
  const float fx0 = (float)tx.tap.x0, fy0 = (float)tx.tap.y0;
  const float ex = fx0 + 1.f - tx.tap.ix, wx = tx.tap.ix - fx0, ey = fy0 + 1.f - tx.tap.iy, wy = tx.tap.iy - fy0;
  const float d00 = tx.c00.x * gcx + tx.c00.y * gcy + tx.c00.z * gcz, d01 = tx.c01.x * gcx + tx.c01.y * gcy + tx.c01.z * gcz;
  const float d10 = tx.c10.x * gcx + tx.c10.y * gcy + tx.c10.z * gcz, d11 = tx.c11.x * gcx + tx.c11.y * gcy + tx.c11.z * gcz;
  const float gix = (d01 - d00) * ey + (d11 - d10) * wy;
  const float giy = (d10 - d00) * ex + (d11 - d01) * wx;
  const float gu = gix * tx.tap.mx, gv = giy * tx.tap.my;
  f3 gbu = {gu * s.uv01.x + gv * s.uv01.y, gu * s.uv01.z + gv * s.uv01.w, gu * s.u2 + gv * s.v2};
  f3 gbc = gbu;
  const bool clipped = s.t.flags & 1;
  if (clipped) {
    // z-clipped face (the ground plane under the camera is one): bu = bc @ conv, so the conversion matrix gets
    // gradient too; it is accumulated per slot with the same warp aggregation as the vertex gradient
    const float* cv = P.conv + gsl * 9;
    gbc.x = cv[0] * gbu.x + cv[1] * gbu.y + cv[2] * gbu.z;
    gbc.y = cv[3] * gbu.x + cv[4] * gbu.y + cv[5] * gbu.z;
    gbc.z = cv[6] * gbu.x + cv[7] * gbu.y + cv[8] * gbu.z;
    gc9[0] = s.b.bc.x * gbu.x; gc9[1] = s.b.bc.x * gbu.y; gc9[2] = s.b.bc.x * gbu.z;
    gc9[3] = s.b.bc.y * gbu.x; gc9[4] = s.b.bc.y * gbu.y; gc9[5] = s.b.bc.y * gbu.z;
    gc9[6] = s.b.bc.z * gbu.x; gc9[7] = s.b.bc.z * gbu.y; gc9[8] = s.b.bc.z * gbu.z;
  }
  float gz0 = 0.f, gz1 = 0.f, gz2 = 0.f;
  f3 gb_ = gbc;
  if (P.clipb) gb_ = clip_backward(s.b.bp, gb_);
  if (P.persp) gb_ = persp_backward(s.b.b0, s.t.z0, s.t.z1, s.t.z2, gb_, gz0, gz1, gz2);
  f2 g0 = {0.f, 0.f}, g1 = {0.f, 0.f}, g2 = {0.f, 0.f};
  bary_backward(p, s.t, gb_, g0, g1, g2);
  gv9[0] = g0.x; gv9[1] = g0.y; gv9[2] = gz0; gv9[3] = g1.x; gv9[4] = g1.y; gv9[5] = gz1; gv9[6] = g2.x; gv9[7] = g2.y; gv9[8] = gz2;
  return clipped;
}

// Pass 2 of a pixel's backward: its n fragments back to front with the division-free suffix recurrence of SURVEY Appendix B,
// on what pass 1 left in shared memory -- q = (alpha, cdot, e, occ) and the record bits of layer k at s_q[k * stride] and
// s_bits[k * stride] -- handing d/d(alpha_k) to the opacity sums and, for halo fragments, to the two vertices of the closest
// edge.  (gr, gg, gb, ga): d loss / d this pass's RGBA at the pixel.  Warp-uniform: every lane makes n_warp (the warp's
// largest n) trips, so that the aggregation helpers run converged.
__device__ __forceinline__ void suffix_backward(const RasterParams& P, const float4* s_q, const int* s_bits, int stride, int n,
                                                int n_warp, f2 p, float gr, float gg, float gb, float ga, int view,
                                                size_t slot_base, bool want_alpha, bool alpha_in_smem, float* s_galpha,
                                                bool want_dist, int lane) {
  if (!want_alpha && !want_dist) return;
  float Tacc = P.bg0 * gr + P.bg1 * gg + P.bg2 * gb - ga;
  // the edge geometry of a halo fragment (2 vertices + 1 / |edge|^2, from the face record) is loaded one layer ahead
  struct EdgeGeom { float4 r0; float2 r1; float4 r3; };
  auto load_edge = [&](int kk, EdgeGeom& g) {
    g.r0 = make_float4(0.f, 0.f, 0.f, 0.f); g.r1 = make_float2(0.f, 0.f); g.r3 = g.r0;
    if (!want_dist || kk < 0 || kk >= n) return;
    const int bits = s_bits[kk * stride];
    if (P.clip_inside && !(bits & DBW_FRAG_OUTSIDE_BIT)) return;          // clamp(d, 0): no distance gradient inside the face
    const size_t gsl = slot_base + (bits & DBW_FRAG_SLOT_MASK);
    g.r0 = __ldg(&P.rec[gsl * 4]); g.r3 = __ldg(&P.rec[gsl * 4 + 3]);
    g.r1 = __ldg(reinterpret_cast<const float2*>(&P.rec[gsl * 4 + 1]));
  };
  EdgeGeom eg_next;
  load_edge(n_warp - 1, eg_next);
  for (int k = n_warp - 1; k >= 0; --k) {
    const EdgeGeom eg = eg_next;
    load_edge(k - 1, eg_next);
    int akey = -1, vkey = -1;
    float aval = 0.f;
    float gv4[4] = {0.f, 0.f, 0.f, 0.f};        // (x, y) of the two vertices of the closest edge
    if (k < n) {
      const float4 q = s_q[k * stride];        // (alpha, cdot, e, occ)
      const float g_alpha = q.w * (q.y - Tacc);
      Tacc = q.x * q.y + (1.f - q.x) * Tacc;
      if (g_alpha != 0.f) {
        const int bits = s_bits[k * stride], slot = bits & DBW_FRAG_SLOT_MASK;
        const int face = slot >= P.F ? slot - P.F : slot;
        if (want_alpha) { akey = alpha_index(P, alpha_in_smem ? 0 : view, face); aval = g_alpha * q.z; }
        if (want_dist && face >= P.n_static_faces) {        // a static face's vertices are constants
          // gradient w.r.t. the SIGNED squared distance: alpha = e(d) * fa, so fa * e = alpha
          const bool inside = !(bits & DBW_FRAG_OUTSIDE_BIT);
          float g_sd = 0.f;
          if (P.clip_inside) { if (!inside) g_sd = g_alpha * (-q.x / P.sigma); }          // clamp(d, 0): flat inside the face
          else g_sd = g_alpha * (-q.x * (1.f - q.z) / P.sigma);
          const float g_dist = inside ? -g_sd : g_sd;    // signed = inside ? -dist : dist
          if (g_dist != 0.f) {
            const int edge = (bits >> DBW_FRAG_EDGE_SHIFT) & 3;
            const f2 v0 = {eg.r0.x, eg.r0.y}, v1 = {eg.r0.z, eg.r0.w}, v2 = {eg.r1.x, eg.r1.y};
            const f2 ea = edge == 2 ? v1 : v0, eb = edge == 0 ? v1 : v2;
            const float il = edge == 0 ? eg.r3.y : (edge == 1 ? eg.r3.z : eg.r3.w);
            f2 g_a = {0.f, 0.f}, g_b = {0.f, 0.f};
            seg_backward(p, ea, eb, il, g_dist, g_a, g_b);
            vkey = slot * 4 + edge;
            gv4[0] = g_a.x; gv4[1] = g_a.y; gv4[2] = g_b.x; gv4[3] = g_b.y;
          }
        }
      }
    }
    if (want_alpha && __ballot_sync(0xffffffffu, akey >= 0)) warp_agg_add1(alpha_in_smem ? s_galpha : P.g_faces_alpha, akey, aval, lane);
    if (want_dist && __ballot_sync(0xffffffffu, vkey >= 0)) warp_agg_add_edge(P.g_tri + slot_base * 9, vkey, gv4, lane);
  }
}

// The loss epilogue's own backward (raster_forward_kernel<NT, true> with P.ep_grad): the detach_bary backward of the pixel,
// run right after the epilogue formed g = d loss / d RGBA, unscaled (dbw_render_backward_deferred applies the upstream
// gradient when it folds the scratch).  The pixel's sorted fragment list is still in shared memory -- lA (pz, bits, signed
// dist, u) and lV (v), `stride` apart -- so pass 1 re-fetches each layer's texels (L1/L2-resident), scatters the texture
// gradient into the CTA's cell-gradient copy and overwrites the entry, whose depth and UV are dead by then, with what pass 2
// needs: (alpha, cdot, e, occ) in lA and the bits in lV.  Pass 2 is suffix_backward.  n: the layers the shading loop
// blended.  Called by every lane of the warp (lanes that are not `live` take part with empty keys).  BLOCKS (blocks_loss_kernel):
// cell maps, the opacities from the table staged after the sums, and the sums always in shared memory.
template <bool BLOCKS>
__device__ __forceinline__ void epilogue_backward(const RasterParams& P, float4* lA, float* lV, int stride, const int4* s_desc,
                                                  float* s_galpha, bool live, int n, f2 p, const float (&g)[4], int view,
                                                  int lane, int warp) {
  const float gr = g[0], gg = g[1], gb = g[2], ga = g[3];
  const bool any_grad = live && ((gr != 0.f) || (gg != 0.f) || (gb != 0.f) || (ga != 0.f));
  const int n_px = any_grad ? n : 0;
  int n_warp = n_px;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_warp = max(n_warp, __shfl_xor_sync(0xffffffffu, n_warp, o));
  float occ = 1.f;
  for (int k = 0; k < n_warp; ++k) {
    int tkey = -1, t01 = -1, t10 = -1, t11 = -1;
    bool tcells = false;
    float tg[3] = {0.f, 0.f, 0.f}, tw[4] = {0.f, 0.f, 0.f, 0.f};      // texture gradient = tg x tw (colour x tap weights)
    if (k < n_px) {
      const float4 e = lA[k * stride];
      const int bits = __float_as_int(e.y), slot = bits & DBW_FRAG_SLOT_MASK;
      const int face = slot >= P.F ? slot - P.F : slot;
      const int4 desc = s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT];
      Texel4 tx;
      fetch_color<BLOCKS>(P, e.w, lV[k * stride], desc, tx);
      const float ea = frag_alpha(e.z, P.sigma, P.clip_inside);
      const float a = !P.faces_alpha ? ea : ea * (BLOCKS ? s_galpha[P.n_alpha + alpha_index(P, 0, face)]
                                                         : __ldg(&P.faces_alpha[alpha_index(P, view, face)]));
      const float cdot = tx.color.x * gr + tx.color.y * gg + tx.color.z * gb;
      lA[k * stride] = make_float4(a, cdot, ea, occ);
      lV[k * stride] = __int_as_float(bits);
      const float w = occ * a;                 // d RGB / d colour_k
      if (w != 0.f && P.g_maps4) {
        tkey = tx.tap.i00; t01 = tx.tap.i01; t10 = tx.tap.i10; t11 = tx.tap.i11; tcells = desc.w != 0;
        tg[0] = w * gr; tg[1] = w * gg; tg[2] = w * gb;
        tw[0] = tx.tap.w00; tw[1] = tx.tap.w01; tw[2] = tx.tap.w10; tw[3] = tx.tap.w11;
      }
      occ *= (1.f - a);
    }
    if (P.g_maps4) warp_tex_scatter<false>(P, tkey, t01, t10, t11, tcells, tg, tw, lane, warp);
  }
  const bool want_alpha = P.faces_alpha != nullptr && P.g_faces_alpha != nullptr;
  suffix_backward(P, lA, reinterpret_cast<const int*>(lV), stride, n_px, n_warp, p, gr, gg, gb, ga, view, (size_t)view * 2 * P.F,
                  want_alpha, BLOCKS || (want_alpha && P.n_alpha <= DBW_ALPHA_SMEM_MAX), s_galpha, P.sigma > 0.f && P.g_tri != nullptr, lane);
}

// One thread per pixel.  Pass 1 streams the pixel's saved fragment records {slot, u, v, signed distance} front to back,
// re-fetches the four texels of each (the float4 atlas is L2-resident), scatters the texture gradient and -- unless
// detach_bary -- re-derives the geometry for the barycentric-path vertex gradient (skipped for faces whose vertices are
// constants; a single-layer pass leaves it to raster_bary_backward_kernel); pass 2 walks back to front with the division-free suffix recurrence of SURVEY Appendix B for d/d(alpha_k)
// -> opacity and distance -> vertex gradients.  Loops are warp-uniform (trip count = warp max) so that the aggregation
// helpers run converged.
// 16 x 8 tiles a backward CTA walks (each warp its own patch of every tile, no barrier between, the next patch's first-level
// loads in flight).  A single-layer pass is a chain of DRAM latencies per pixel and gains from 8 tiles (on an H100 SXM,
// 4 tiles: 0.51 ms instead of 0.50 ms for the dtu environment backward); the K = 10 blocks pass walks one (more tiles
// make longer CTAs and worse tails)
#ifndef DBW_BWD_TILES_K1
#define DBW_BWD_TILES_K1 8
#endif
#define DBW_BWD_TILES_KN 1

// K1: faces_per_pixel == 1 (the environment pass): no record prefetch registers, at most one trip through the loops
// depth_backward_kernel below is a copy of this walk with the depth terms: a fix here belongs there too.
template <bool DETACH, bool ALPHA, bool K1>
__global__ void __launch_bounds__(DBW_BWD_NT, DETACH ? DBW_BWD_DETACH_MINB : DBW_BWD_BARY_MINB) raster_backward_kernel(const RasterParams P) {
  extern __shared__ float4 s_dyn[];             // [k][tid] (alpha, cdot, e, occ), [k][tid] record bits, the map table, opacity sums
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = blockIdx.x;
  constexpr int DBW_BWD_TILES = K1 ? DBW_BWD_TILES_K1 : DBW_BWD_TILES_KN;
  const int strip = centre_out(blockIdx.z, gridDim.z);          // DBW_BWD_TILES vertically adjacent 16 x 8 tiles per CTA
  const int xi = blockIdx.y * TILE_W + (warp & 1) * 8 + (lane & 7);
  int row_lo = 0, row_hi = P.H;
  if (P.view_rows) { row_lo = P.view_rows[view * 2]; row_hi = P.view_rows[view * 2 + 1]; }
  constexpr int TH = DBW_BWD_NT / 16;
  if (strip * DBW_BWD_TILES * TH >= row_hi || (strip + 1) * DBW_BWD_TILES * TH <= row_lo) return;
  const size_t plane = (size_t)P.H * P.W;
  float4* const s_q = s_dyn + tid;
  int* const s_bits = reinterpret_cast<int*>(s_dyn + (size_t)P.K * DBW_BWD_NT) + tid;
  int4* const s_desc = reinterpret_cast<int4*>(reinterpret_cast<int*>(s_dyn + (size_t)P.K * DBW_BWD_NT) + (size_t)P.K * DBW_BWD_NT);
  float* const s_galpha = reinterpret_cast<float*>(s_desc + P.M);
  const float gs = P.grad_scale ? __ldg(P.grad_scale) : 1.f;
  stage_map_table(P, s_desc, tid, DBW_BWD_NT);
  const bool want_alpha = ALPHA && P.g_faces_alpha != nullptr;
  const bool alpha_in_smem = want_alpha && P.n_alpha <= DBW_ALPHA_SMEM_MAX;       // few opacity entries: hot addresses
  if (alpha_in_smem) for (int i = tid; i < P.n_alpha; i += DBW_BWD_NT) s_galpha[i] = 0.f;
  const bool want_dist = P.sigma > 0.f && P.g_tri != nullptr;
  // d loss / d alpha of the pixel feeds only the suffix pass; without it a zero alpha gradient changes no result (a pixel
  // whose only non-zero gradient is alpha's contributes zeros), and the plane is not read -- a loss epilogue may not write it
  const bool want_ga = want_alpha || want_dist;
  const size_t slot_base = (size_t)view * 2 * P.F;
  __syncthreads();

  // Every warp walks ITS 8x4 patch of the strip's tiles on its own: no barrier between tiles, and the first-level loads of
  // the next patch -- gradient pixel, fragment count, first record pair -- are issued before the current patch is processed,
  // so that their DRAM latency is covered by work instead of by the other (few) resident warps.
  struct First { float g0, g1, g2, g3; int n; float4 rec, rgb; };
  auto load_first = [&](int t, First& f) {
    f.g0 = f.g1 = f.g2 = f.g3 = 0.f; f.n = 0; f.rec = make_float4(0.f, 0.f, 0.f, 0.f); f.rgb = f.rec;
    const int y = (strip * DBW_BWD_TILES + t) * TH + (warp >> 1) * 4 + (lane >> 3);
    if (t < DBW_BWD_TILES && xi < P.W && y < P.H && y >= row_lo && y < row_hi) {
      const size_t px = (size_t)y * P.W + xi;
      const float* go = P.grad_rgba + (size_t)view * 4 * plane + px;
      f.g0 = go[0]; f.g1 = go[plane]; f.g2 = go[2 * plane];
      if (want_ga) f.g3 = go[3 * plane];
      f.n = (int)P.nfrag[(size_t)view * plane + px];
      f.rec = P.frag[(size_t)view * P.K * plane + px];          // speculative: a valid workspace address whether or not a
      if (P.frag_rgb) f.rgb = P.frag_rgb[(size_t)view * P.K * plane + px];      // fragment exists (no colours: see keeps_colours)
    }
  };
  First first_next;
  load_first(0, first_next);
  bool need_bary = false;       // K1 && DETACH: this thread saw a fragment that raster_bary_backward_kernel must visit
  for (int t = 0; t < DBW_BWD_TILES; ++t) {
  const First first = first_next;
  load_first(t + 1, first_next);
  const int yi = (strip * DBW_BWD_TILES + t) * TH + (warp >> 1) * 4 + (lane >> 3);
  const bool live = xi < P.W && yi < P.H && yi >= row_lo && yi < row_hi;
  const size_t pix = live ? (size_t)yi * P.W + xi : 0;
  const float4* frag = P.frag + (size_t)view * P.K * plane + pix;
  const float4* frag_rgb = P.frag_rgb + (size_t)view * P.K * plane + pix;
  const float gr = first.g0 * gs, gg = first.g1 * gs, gb = first.g2 * gs, ga = first.g3 * gs;
  const bool any_grad = live && ((gr != 0.f) || (gg != 0.f) || (gb != 0.f) || (ga != 0.f));
  const int n_px = any_grad ? first.n : 0;
  float4 rec_cur = first.rec, rgb_cur = first.rgb, rec_nxt = make_float4(0.f, 0.f, 0.f, 0.f), rgb_nxt = rec_nxt;
  if (!K1 && n_px > 1) { rec_nxt = frag[plane]; rgb_nxt = frag_rgb[plane]; }
  const f2 p = {pix_to_ndc(P.W - 1 - xi, P.W, P.H), pix_to_ndc(P.H - 1 - yi, P.H, P.W)};

  // fragments are walked front to back until every lane of the warp has run out (warp-uniform trip count); the records of
  // layers k+1 and k+2 are in flight while layer k is processed
  int n_warp = n_px;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_warp = max(n_warp, __shfl_xor_sync(0xffffffffu, n_warp, o));
  int n = 0;
  float occ = 1.f;
  for (int k = 0; k < n_warp; ++k) {
    const float4 fr = rec_cur, fc = rgb_cur;
    if (!K1) {
      rec_cur = rec_nxt; rgb_cur = rgb_nxt;
      if (k + 2 < n_px) { rec_nxt = frag[(size_t)(k + 2) * plane]; rgb_nxt = frag_rgb[(size_t)(k + 2) * plane]; }
    }
    const bool have = k < n_px && occ != 0.f;      // everything behind a fully opaque fragment has zero weight and zero gradient
    int key = -1, ckey = -1, tkey = -1, t01 = -1, t10 = -1, t11 = -1;
    bool tcells = false;
    float gv9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float gc9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float tg[3] = {0.f, 0.f, 0.f}, tw[4] = {0.f, 0.f, 0.f, 0.f};      // texture gradient = tg x tw (colour x tap weights)
    if (have) {
      n = k + 1;
      const int bits = __float_as_int(fr.x), slot = bits & DBW_FRAG_SLOT_MASK;
      const int face = slot >= P.F ? slot - P.F : slot;
      const float d = fr.w;
      Texel4 tx;
      Shade s;
      const bool bary_path = !DETACH && face >= P.n_static_faces;
      const int4 desc = s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT];
      if (bary_path) {              // the gradient through (u, v) needs the four texels and the face's geometry again
        shade_geometry(P, view, slot, p, s);
        fetch_color(P, s.u, s.v, desc, tx);
      } else {                      // texture / opacity / distance gradients: the saved colour and tap addresses suffice
        tap_only(fr.y, fr.z, desc, tx);
        tx.color = {fc.x, fc.y, fc.z};
      }
      const float e = frag_alpha(d, P.sigma, P.clip_inside);
      const float fa = ALPHA ? __ldg(&P.faces_alpha[alpha_index(P, view, face)]) : 1.f;
      const float a = e * fa;
      const float cdot = tx.color.x * gr + tx.color.y * gg + tx.color.z * gb;
      s_q[k * DBW_BWD_NT] = make_float4(a, cdot, e, occ);
      s_bits[k * DBW_BWD_NT] = bits;
      const float w = occ * a;                 // d RGB / d colour_k
      if (w != 0.f) {
        const float gcx = w * gr, gcy = w * gg, gcz = w * gb;
        if (P.g_maps4) {
          tkey = tx.tap.i00; t01 = tx.tap.i01; t10 = tx.tap.i10; t11 = tx.tap.i11; tcells = desc.w != 0;
          tg[0] = gcx; tg[1] = gcy; tg[2] = gcz;
          tw[0] = tx.tap.w00; tw[1] = tx.tap.w01; tw[2] = tx.tap.w10; tw[3] = tx.tap.w11;
        }
        if (bary_path && P.g_tri) {
          key = slot;
          if (bary_frag_backward(P, slot_base + slot, p, s, tx, gcx, gcy, gcz, gv9, gc9)) ckey = slot;
        }
      }
      if (K1 && DETACH && face >= P.n_static_faces && w != 0.f) need_bary = true;
      occ *= (1.f - a);
    }
    if (P.g_maps4) warp_tex_scatter<K1>(P, tkey, t01, t10, t11, tcells, tg, tw, lane, warp);
    if (!DETACH) {
      if (__ballot_sync(0xffffffffu, key >= 0)) warp_agg_add<9>(P.g_tri + slot_base * 9, 9, key, gv9, lane);
      if (__ballot_sync(0xffffffffu, ckey >= 0)) warp_agg_add<9>(P.g_conv + slot_base * 9, 9, ckey, gc9, lane);
    }
  }

  // pass 2: suffix recurrence on the stored per-fragment scalars
  suffix_backward(P, s_q, s_bits, DBW_BWD_NT, n, n_warp, p, gr, gg, gb, ga, view, slot_base, want_alpha, alpha_in_smem, s_galpha,
                  want_dist, lane);
  }   // tiles of the strip
  if (alpha_in_smem) {               // one global atomic per (CTA, opacity entry) instead of one per (warp, layer, entry)
    __syncthreads();
    for (int i = tid; i < P.n_alpha; i += DBW_BWD_NT) {
      const float v = s_galpha[i];
      if (v != 0.f) atomicAdd(&P.g_faces_alpha[(size_t)view * P.alpha_stride + i], v);
    }
  }
  if (K1 && DETACH && P.bary_flags) {
    if (__syncthreads_or(need_bary) && tid == 0) P.bary_flags[((size_t)view * gridDim.y + blockIdx.y) * gridDim.z + strip] = 1;
  }
}

// depth_backward_kernel (dbw_render_backward_depth): raster_backward_kernel with the gradients of the depth outputs too -- a
// copy of its walk with the DEPTH branches, rather than DEPTH branches in it: routing raster_backward_kernel through a shared
// body changes its instruction schedule.  d D / d w_k = z_k joins the colour's
// d RGB / d w_k in cdot, so it takes the same opacity / distance chain through the suffix pass; each fragment's own depth
// gets g_z = g_D w_k + g_zbuf_k, which depth_frag_backward takes to the slot's vertices -- with DETACH too (only the
// barycentrics of the colour are detached).  The fragment's geometry is re-derived for its z.  Every recorded layer is visited,
// also those behind a fully opaque one (the DEPTH forward records them: their zbuf has a gradient, their weight none).
template <bool DETACH, bool ALPHA, bool K1>
__global__ void __launch_bounds__(DBW_BWD_NT, DBW_BWD_BARY_MINB) depth_backward_kernel(const RasterParams P, const DepthIO Dz) {
  constexpr bool DEPTH = true;
  extern __shared__ float4 s_dyn[];             // [k][tid] (alpha, cdot, e, occ), [k][tid] record bits, the map table, opacity sums
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = blockIdx.x;
  constexpr int DBW_BWD_TILES = K1 ? DBW_BWD_TILES_K1 : DBW_BWD_TILES_KN;
  const int strip = centre_out(blockIdx.z, gridDim.z);          // DBW_BWD_TILES vertically adjacent 16 x 8 tiles per CTA
  const int xi = blockIdx.y * TILE_W + (warp & 1) * 8 + (lane & 7);
  int row_lo = 0, row_hi = P.H;
  if (P.view_rows) { row_lo = P.view_rows[view * 2]; row_hi = P.view_rows[view * 2 + 1]; }
  constexpr int TH = DBW_BWD_NT / 16;
  if (strip * DBW_BWD_TILES * TH >= row_hi || (strip + 1) * DBW_BWD_TILES * TH <= row_lo) return;
  const size_t plane = (size_t)P.H * P.W;
  float4* const s_q = s_dyn + tid;
  int* const s_bits = reinterpret_cast<int*>(s_dyn + (size_t)P.K * DBW_BWD_NT) + tid;
  int4* const s_desc = reinterpret_cast<int4*>(reinterpret_cast<int*>(s_dyn + (size_t)P.K * DBW_BWD_NT) + (size_t)P.K * DBW_BWD_NT);
  float* const s_galpha = reinterpret_cast<float*>(s_desc + P.M);
  const float gs = P.grad_scale ? __ldg(P.grad_scale) : 1.f;
  stage_map_table(P, s_desc, tid, DBW_BWD_NT);
  const bool want_alpha = ALPHA && P.g_faces_alpha != nullptr;
  const bool alpha_in_smem = want_alpha && P.n_alpha <= DBW_ALPHA_SMEM_MAX;       // few opacity entries: hot addresses
  if (alpha_in_smem) for (int i = tid; i < P.n_alpha; i += DBW_BWD_NT) s_galpha[i] = 0.f;
  const bool want_dist = P.sigma > 0.f && P.g_tri != nullptr;
  // d loss / d alpha of the pixel feeds only the suffix pass; without it a zero alpha gradient changes no result (a pixel
  // whose only non-zero gradient is alpha's contributes zeros), and the plane is not read -- a loss epilogue may not write it
  const bool want_ga = want_alpha || want_dist;
  const size_t slot_base = (size_t)view * 2 * P.F;
  __syncthreads();

  // Every warp walks ITS 8x4 patch of the strip's tiles on its own: no barrier between tiles, and the first-level loads of
  // the next patch -- gradient pixel, fragment count, first record pair -- are issued before the current patch is processed,
  // so that their DRAM latency is covered by work instead of by the other (few) resident warps.
  struct First { float g0, g1, g2, g3; int n; float4 rec, rgb; };
  auto load_first = [&](int t, First& f) {
    f.g0 = f.g1 = f.g2 = f.g3 = 0.f; f.n = 0; f.rec = make_float4(0.f, 0.f, 0.f, 0.f); f.rgb = f.rec;
    const int y = (strip * DBW_BWD_TILES + t) * TH + (warp >> 1) * 4 + (lane >> 3);
    if (t < DBW_BWD_TILES && xi < P.W && y < P.H && y >= row_lo && y < row_hi) {
      const size_t px = (size_t)y * P.W + xi;
      const float* go = P.grad_rgba + (size_t)view * 4 * plane + px;
      f.g0 = go[0]; f.g1 = go[plane]; f.g2 = go[2 * plane];
      if (want_ga) f.g3 = go[3 * plane];
      f.n = (int)P.nfrag[(size_t)view * plane + px];
      f.rec = P.frag[(size_t)view * P.K * plane + px];          // speculative: a valid workspace address whether or not a
      if (P.frag_rgb) f.rgb = P.frag_rgb[(size_t)view * P.K * plane + px];      // fragment exists (no colours: see keeps_colours)
    }
  };
  First first_next;
  load_first(0, first_next);
  // DEPTH: the pixel's depth gradient, loaded one patch ahead as well
  auto load_gd = [&](int t) -> float {
    const int y = (strip * DBW_BWD_TILES + t) * TH + (warp >> 1) * 4 + (lane >> 3);
    if (!DEPTH || !Dz.g_depth || t >= DBW_BWD_TILES || xi >= P.W || y >= P.H || y < row_lo || y >= row_hi) return 0.f;
    return Dz.g_depth[(size_t)view * plane + (size_t)y * P.W + xi];
  };
  float gd_next = DEPTH ? load_gd(0) : 0.f;
  bool need_bary = false;       // K1 && DETACH: this thread saw a fragment that raster_bary_backward_kernel must visit
  for (int t = 0; t < DBW_BWD_TILES; ++t) {
  const First first = first_next;
  load_first(t + 1, first_next);
  const float gd = gd_next * gs;
  if (DEPTH) gd_next = load_gd(t + 1);
  const int yi = (strip * DBW_BWD_TILES + t) * TH + (warp >> 1) * 4 + (lane >> 3);
  const bool live = xi < P.W && yi < P.H && yi >= row_lo && yi < row_hi;
  const size_t pix = live ? (size_t)yi * P.W + xi : 0;
  const float4* frag = P.frag + (size_t)view * P.K * plane + pix;
  const float4* frag_rgb = P.frag_rgb + (size_t)view * P.K * plane + pix;
  const float gr = first.g0 * gs, gg = first.g1 * gs, gb = first.g2 * gs, ga = first.g3 * gs;
  const bool any_grad = live && ((gr != 0.f) || (gg != 0.f) || (gb != 0.f) || (ga != 0.f) || (DEPTH && (gd != 0.f || Dz.g_zbuf)));
  const int n_px = any_grad ? first.n : 0;
  float4 rec_cur = first.rec, rgb_cur = first.rgb, rec_nxt = make_float4(0.f, 0.f, 0.f, 0.f), rgb_nxt = rec_nxt;
  if (!K1 && n_px > 1) { rec_nxt = frag[plane]; rgb_nxt = frag_rgb[plane]; }
  const f2 p = {pix_to_ndc(P.W - 1 - xi, P.W, P.H), pix_to_ndc(P.H - 1 - yi, P.H, P.W)};

  // fragments are walked front to back until every lane of the warp has run out (warp-uniform trip count); the records of
  // layers k+1 and k+2 are in flight while layer k is processed
  int n_warp = n_px;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_warp = max(n_warp, __shfl_xor_sync(0xffffffffu, n_warp, o));
  int n = 0;
  float occ = 1.f;
  for (int k = 0; k < n_warp; ++k) {
    const float4 fr = rec_cur, fc = rgb_cur;
    if (!K1) {
      rec_cur = rec_nxt; rgb_cur = rgb_nxt;
      if (k + 2 < n_px) { rec_nxt = frag[(size_t)(k + 2) * plane]; rgb_nxt = frag_rgb[(size_t)(k + 2) * plane]; }
    }
    // everything behind a fully opaque fragment has zero weight and zero gradient (but for DEPTH, that of its zbuf)
    const bool have = k < n_px && (DEPTH || occ != 0.f);
    int key = -1, ckey = -1, tkey = -1, t01 = -1, t10 = -1, t11 = -1;
    bool tcells = false;
    float gv9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float gc9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float tg[3] = {0.f, 0.f, 0.f}, tw[4] = {0.f, 0.f, 0.f, 0.f};      // texture gradient = tg x tw (colour x tap weights)
    if (have) {
      n = k + 1;
      const int bits = __float_as_int(fr.x), slot = bits & DBW_FRAG_SLOT_MASK;
      const int face = slot >= P.F ? slot - P.F : slot;
      const float d = fr.w;
      Texel4 tx;
      Shade s;
      const bool bary_path = !DETACH && face >= P.n_static_faces;
      const int4 desc = s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT];
      if (bary_path) {              // the gradient through (u, v) needs the four texels and the face's geometry again
        shade_geometry(P, view, slot, p, s);
        fetch_color(P, s.u, s.v, desc, tx);
      } else {                      // texture / opacity / distance gradients: the saved colour and tap addresses suffice
        if (DEPTH) shade_geometry(P, view, slot, p, s);          // (but not the fragment's depth)
        tap_only(fr.y, fr.z, desc, tx);
        tx.color = {fc.x, fc.y, fc.z};
      }
      const float e = frag_alpha(d, P.sigma, P.clip_inside);
      const float fa = ALPHA ? __ldg(&P.faces_alpha[alpha_index(P, view, face)]) : 1.f;
      const float a = e * fa;
      float cdot = tx.color.x * gr + tx.color.y * gg + tx.color.z * gb;
      if (DEPTH) cdot += s.b.pz * gd;          // the depth is a fourth colour channel with background 0
      s_q[k * DBW_BWD_NT] = make_float4(a, cdot, e, occ);
      s_bits[k * DBW_BWD_NT] = bits;
      const float w = occ * a;                 // d RGB / d colour_k
      if (w != 0.f) {
        const float gcx = w * gr, gcy = w * gg, gcz = w * gb;
        if (P.g_maps4) {
          tkey = tx.tap.i00; t01 = tx.tap.i01; t10 = tx.tap.i10; t11 = tx.tap.i11; tcells = desc.w != 0;
          tg[0] = gcx; tg[1] = gcy; tg[2] = gcz;
          tw[0] = tx.tap.w00; tw[1] = tx.tap.w01; tw[2] = tx.tap.w10; tw[3] = tx.tap.w11;
        }
        if (bary_path && P.g_tri) {
          key = slot;
          if (bary_frag_backward(P, slot_base + slot, p, s, tx, gcx, gcy, gcz, gv9, gc9)) ckey = slot;
        }
      }
      if (DEPTH && P.g_tri && face >= P.n_static_faces) {
        const float g_pz = gd * w + (Dz.g_zbuf ? Dz.g_zbuf[((size_t)view * P.K + k) * plane + pix] * gs : 0.f);
        if (g_pz != 0.f) { key = slot; depth_frag_backward(p, s.t, s.b, P.persp, P.clipb, g_pz, gv9); }
      }
      if (K1 && DETACH && face >= P.n_static_faces && w != 0.f) need_bary = true;
      occ *= (1.f - a);
    }
    if (P.g_maps4) warp_tex_scatter<K1>(P, tkey, t01, t10, t11, tcells, tg, tw, lane, warp);
    if (!DETACH || DEPTH) {
      if (__ballot_sync(0xffffffffu, key >= 0)) warp_agg_add<9>(P.g_tri + slot_base * 9, 9, key, gv9, lane);
    }
    if (!DETACH) {
      if (__ballot_sync(0xffffffffu, ckey >= 0)) warp_agg_add<9>(P.g_conv + slot_base * 9, 9, ckey, gc9, lane);
    }
  }

  // pass 2: suffix recurrence on the stored per-fragment scalars
  suffix_backward(P, s_q, s_bits, DBW_BWD_NT, n, n_warp, p, gr, gg, gb, ga, view, slot_base, want_alpha, alpha_in_smem, s_galpha,
                  want_dist, lane);
  }   // tiles of the strip
  if (alpha_in_smem) {               // one global atomic per (CTA, opacity entry) instead of one per (warp, layer, entry)
    __syncthreads();
    for (int i = tid; i < P.n_alpha; i += DBW_BWD_NT) {
      const float v = s_galpha[i];
      if (v != 0.f) atomicAdd(&P.g_faces_alpha[(size_t)view * P.alpha_stride + i], v);
    }
  }
  if (K1 && DETACH && P.bary_flags) {
    if (__syncthreads_or(need_bary) && tid == 0) P.bary_flags[((size_t)view * gridDim.y + blockIdx.y) * gridDim.z + strip] = 1;
  }
}

// Barycentric-path vertex gradient of a single-layer pass that is not detached (the environment pass: the ground's pose
// gets gradient only through its barycentrics).  It runs after raster_backward_kernel<true, *, true>, which scatters the
// texture gradients and the opacity / distance gradients of every pixel and flags the strips holding a fragment of a face
// >= n_static_faces; this kernel has the same grid and leaves the unflagged strips at once.  Per pixel it re-derives the
// fragment's geometry and its four texels for d(colour)/d(uv), and aggregates the slot gradients -- no texture scatter,
// so the geometry has the register file to itself.
template <bool ALPHA>
__global__ void __launch_bounds__(DBW_BWD_NT, DBW_BWD_GEOM_MINB) raster_bary_backward_kernel(const RasterParams P) {
  extern __shared__ int4 s_desc[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = blockIdx.x;
  const int strip = centre_out(blockIdx.z, gridDim.z);
  const int xi = blockIdx.y * TILE_W + (warp & 1) * 8 + (lane & 7);
  int row_lo = 0, row_hi = P.H;
  if (P.view_rows) { row_lo = P.view_rows[view * 2]; row_hi = P.view_rows[view * 2 + 1]; }
  constexpr int TH = DBW_BWD_NT / 16;
  if (strip * DBW_BWD_TILES_K1 * TH >= row_hi || (strip + 1) * DBW_BWD_TILES_K1 * TH <= row_lo) return;
  if (!P.bary_flags[((size_t)view * gridDim.y + blockIdx.y) * gridDim.z + strip]) return;
  stage_map_table(P, s_desc, tid, DBW_BWD_NT);
  const size_t plane = (size_t)P.H * P.W;
  const float gs = P.grad_scale ? __ldg(P.grad_scale) : 1.f;
  const size_t slot_base = (size_t)view * 2 * P.F;
  __syncthreads();
  // As in raster_backward_kernel<K1>: each warp walks its patches on its own, and the next patch's fragment count, record and
  // RGB gradient are in flight while the current one is processed.  The record is loaded whether or not a fragment exists
  // (a valid workspace address either way), so that the three loads do not wait on each other.
  struct First { bool n; float4 rec; float g0, g1, g2; };
  auto load_first = [&](int t, First& f) {
    f.n = false; f.rec = make_float4(0.f, 0.f, 0.f, 0.f); f.g0 = f.g1 = f.g2 = 0.f;
    const int y = (strip * DBW_BWD_TILES_K1 + t) * TH + (warp >> 1) * 4 + (lane >> 3);
    if (t < DBW_BWD_TILES_K1 && xi < P.W && y < P.H && y >= row_lo && y < row_hi) {
      const size_t px = (size_t)y * P.W + xi;
      f.n = P.nfrag[(size_t)view * plane + px] != 0;
      f.rec = P.frag[(size_t)view * plane + px];
      const float* go = P.grad_rgba + (size_t)view * 4 * plane + px;
      f.g0 = go[0]; f.g1 = go[plane]; f.g2 = go[2 * plane];
    }
  };
  First first_next;
  load_first(0, first_next);
  for (int t = 0; t < DBW_BWD_TILES_K1; ++t) {
    const First first = first_next;
    load_first(t + 1, first_next);
    const int yi = (strip * DBW_BWD_TILES_K1 + t) * TH + (warp >> 1) * 4 + (lane >> 3);
    int key = -1, ckey = -1;
    float gv9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float gc9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (first.n) {                  // only a pixel of the call's rows has one (load_first)
      const float4 fr = first.rec;
      const int bits = __float_as_int(fr.x), slot = bits & DBW_FRAG_SLOT_MASK;
      const int face = slot >= P.F ? slot - P.F : slot;
      if (face >= P.n_static_faces) {
        const float gr = first.g0 * gs, gg = first.g1 * gs, gb = first.g2 * gs;
        const float fa = ALPHA ? __ldg(&P.faces_alpha[alpha_index(P, view, face)]) : 1.f;
        const float w = frag_alpha(fr.w, P.sigma, P.clip_inside) * fa;        // the only layer: occlusion 1
        if (w != 0.f && (gr != 0.f || gg != 0.f || gb != 0.f)) {
          const f2 p = {pix_to_ndc(P.W - 1 - xi, P.W, P.H), pix_to_ndc(P.H - 1 - yi, P.H, P.W)};
          Shade s;
          Texel4 tx;
          shade_geometry(P, view, slot, p, s);
          fetch_color(P, s.u, s.v, s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT], tx);
          key = slot;
          if (bary_frag_backward(P, slot_base + slot, p, s, tx, w * gr, w * gg, w * gb, gv9, gc9)) ckey = slot;
        }
      }
    }
    if (__ballot_sync(0xffffffffu, key >= 0)) warp_agg_add<9>(P.g_tri + slot_base * 9, 9, key, gv9, lane);
    if (__ballot_sync(0xffffffffu, ckey >= 0)) warp_agg_add<9>(P.g_conv + slot_base * 9, 9, ckey, gc9, lane);
  }
}

// per (view, face): fold the gradients of the (clipped) triangle slots back onto the face's 3 projected vertices
__device__ __forceinline__ void lerp_clip_backward(const float* p1, const float* p2, float w, bool persp, const float* gp4,
                                                   float* gp1, float* gp2, float& gw) {
  if (persp) {
    const float q1x = p1[0] * p1[2], q1y = p1[1] * p1[2], q2x = p2[0] * p2[2], q2y = p2[1] * p2[2];
    const float Px = q1x * (1.f - w) + q2x * w, Py = q1y * (1.f - w) + q2y * w, Pz = p1[2] * (1.f - w) + p2[2] * w;
    const float gPx = gp4[0] / Pz, gPy = gp4[1] / Pz;
    const float gPz = gp4[2] - (gp4[0] * Px + gp4[1] * Py) / (Pz * Pz);
    gw += gPx * (q2x - q1x) + gPy * (q2y - q1y) + gPz * (p2[2] - p1[2]);
    const float a = 1.f - w;
    // q = (x z, y z, z)
    gp1[0] += gPx * a * p1[2]; gp1[1] += gPy * a * p1[2]; gp1[2] += gPx * a * p1[0] + gPy * a * p1[1] + gPz * a;
    gp2[0] += gPx * w * p2[2]; gp2[1] += gPy * w * p2[2]; gp2[2] += gPx * w * p2[0] + gPy * w * p2[1] + gPz * w;
  } else {
    const float a = 1.f - w;
#pragma unroll
    for (int i = 0; i < 3; ++i) { gp1[i] += gp4[i] * a; gp2[i] += gp4[i] * w; gw += gp4[i] * (p2[i] - p1[i]); }
  }
}

__global__ void face_setup_backward_kernel(const float* __restrict__ verts_ndc, const int* __restrict__ faces, int B, int V, int F,
                                           float z_clip, int persp, const float* __restrict__ g_tri, const float* __restrict__ g_conv,
                                           const float* __restrict__ scale, float* __restrict__ g_verts_ndc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * F) return;
  const float sc = scale ? __ldg(scale) : 1.f;       // g_tri and g_conv are multiplied by *scale (NULL = 1)
  const int b = i / F, f = i - b * F;
  const size_t s0 = (size_t)b * 2 * F + f, s1 = s0 + F;
  float a[3][3]; int vid[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    vid[j] = faces[f * 3 + j];
    const float* v = verts_ndc + ((size_t)b * V + vid[j]) * 3;
    a[j][0] = v[0]; a[j][1] = v[1]; a[j][2] = v[2];
  }
  int nb = 0, behind[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) { behind[j] = (z_clip >= 0.f) && (a[j][2] < z_clip); nb += behind[j]; }
  if (nb == 3) return;
  float ga[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  const float* gt0 = g_tri + s0 * 9;
  if (nb == 0) {
#pragma unroll
    for (int j = 0; j < 3; ++j) { ga[j][0] = gt0[j * 3]; ga[j][1] = gt0[j * 3 + 1]; ga[j][2] = gt0[j * 3 + 2]; }
  } else {
    int i1 = 0;
    if (nb == 2) { for (int j = 0; j < 3; ++j) if (!behind[j]) i1 = j; }
    else         { for (int j = 0; j < 3; ++j) if (behind[j]) i1 = j; }
    const int i2 = (i1 + 1) % 3, i3 = (i1 + 2) % 3;
    const float* p1 = a[i1]; const float* p2 = a[i2]; const float* p3 = a[i3];
    const float den2 = p1[2] - p2[2], den3 = p1[2] - p3[2];
    const float w2 = (p1[2] - z_clip) / den2, w3 = (p1[2] - z_clip) / den3;
    float gp1[3] = {0, 0, 0}, gp2[3] = {0, 0, 0}, gp3[3] = {0, 0, 0}, gp4[3] = {0, 0, 0}, gp5[3] = {0, 0, 0};
    float gb4[3] = {0, 0, 0}, gb5[3] = {0, 0, 0};
    const float* gc0 = g_conv + s0 * 9;
    if (nb == 2) {      // slot0 = (p4, p5, p1), conv rows (b4, b5, b1)
#pragma unroll
      for (int c = 0; c < 3; ++c) { gp4[c] += gt0[c]; gp5[c] += gt0[3 + c]; gp1[c] += gt0[6 + c]; gb4[c] += gc0[c]; gb5[c] += gc0[3 + c]; }
    } else {            // slot0 = (p4, p2, p5) ; slot1 = (p5, p2, p3)
      const float* gt1 = g_tri + s1 * 9; const float* gc1 = g_conv + s1 * 9;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        gp4[c] += gt0[c]; gp2[c] += gt0[3 + c] + gt1[3 + c]; gp5[c] += gt0[6 + c] + gt1[c]; gp3[c] += gt1[6 + c];
        gb4[c] += gc0[c]; gb5[c] += gc0[6 + c] + gc1[c];
      }
    }
    float gw2 = 0.f, gw3 = 0.f;
    // b4 = e_i1 (1-w2) + e_i2 w2 ; b5 = e_i1 (1-w3) + e_i3 w3
    gw2 += gb4[i2] - gb4[i1];
    gw3 += gb5[i3] - gb5[i1];
    lerp_clip_backward(p1, p2, w2, persp != 0, gp4, gp1, gp2, gw2);
    lerp_clip_backward(p1, p3, w3, persp != 0, gp5, gp1, gp3, gw3);
    // w = (z1 - zc) / (z1 - z_other)
    gp1[2] += gw2 * (z_clip - p2[2]) / (den2 * den2) + gw3 * (z_clip - p3[2]) / (den3 * den3);
    gp2[2] += gw2 * (p1[2] - z_clip) / (den2 * den2);
    gp3[2] += gw3 * (p1[2] - z_clip) / (den3 * den3);
#pragma unroll
    for (int c = 0; c < 3; ++c) { ga[i1][c] = gp1[c]; ga[i2][c] = gp2[c]; ga[i3][c] = gp3[c]; }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float* g = g_verts_ndc + ((size_t)b * V + vid[j]) * 3;
    if (ga[j][0] != 0.f) atomicAdd(g, sc * ga[j][0]);
    if (ga[j][1] != 0.f) atomicAdd(g + 1, sc * ga[j][1]);
    if (ga[j][2] != 0.f) atomicAdd(g + 2, sc * ga[j][2]);
  }
}

// ------------------------------------------------------------------------------------------------ compositing + MSE (dbw.py:223, 366-367)
__global__ void composite_mse_kernel(int n_px_total, int plane, const float* __restrict__ fg, const float* __restrict__ env,
                                     const float* __restrict__ imgs, float inv_count, float* __restrict__ rec,
                                     float* __restrict__ loss_sum, float* __restrict__ g_fg, float* __restrict__ g_env) {
  float local = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_px_total; i += gridDim.x * blockDim.x) {
    const int b = i / plane, px = i - b * plane;
    const float* f = fg + (size_t)b * 4 * plane + px;
    const float* e = env + (size_t)b * 4 * plane + px;
    const float* im = imgs + (size_t)b * 3 * plane + px;
    const float m = f[3 * (size_t)plane];
    float gm = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float fc = f[(size_t)c * plane], ec = e[(size_t)c * plane];
      const float r = fc * m + (1.f - m) * ec;
      const float diff = r - im[(size_t)c * plane];
      local += diff * diff;
      if (rec) rec[(size_t)b * 3 * plane + (size_t)c * plane + px] = r;
      const float gr = 2.f * diff * inv_count;
      if (g_fg) g_fg[(size_t)b * 4 * plane + (size_t)c * plane + px] = gr * m;
      if (g_env) g_env[(size_t)b * 4 * plane + (size_t)c * plane + px] = gr * (1.f - m);
      gm += gr * (fc - ec);
    }
    if (g_fg) g_fg[(size_t)b * 4 * plane + 3 * (size_t)plane + px] = gm;
    if (g_env) g_env[(size_t)b * 4 * plane + 3 * (size_t)plane + px] = 0.f;
  }
  // block reduction -> one atomic per block
  __shared__ float red[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) atomicAdd(loss_sum, v * inv_count);
  }
}

// gradient of (g_loss * loss + <g_rec, rec>) w.r.t. fg and env, straight from the inputs: no saved gradient buffers and
// no elementwise rescaling kernels
__global__ void composite_backward_kernel(int n_px_total, int plane, const float* __restrict__ fg, const float* __restrict__ env,
                                          const float* __restrict__ imgs, float inv_count, const float* __restrict__ g_loss,
                                          const float* __restrict__ g_rec, float* __restrict__ g_fg, float* __restrict__ g_env) {
  const float gl = g_loss ? __ldg(g_loss) : 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_px_total; i += gridDim.x * blockDim.x) {
    const int b = i / plane, px = i - b * plane;
    const float* f = fg + (size_t)b * 4 * plane + px;
    const float* e = env + (size_t)b * 4 * plane + px;
    const float m = f[3 * (size_t)plane];
    float gm = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float fc = f[(size_t)c * plane], ec = e[(size_t)c * plane];
      const float r = fc * m + (1.f - m) * ec;
      float gr = 2.f * (r - imgs[(size_t)b * 3 * plane + (size_t)c * plane + px]) * inv_count * gl;
      if (g_rec) gr += g_rec[(size_t)b * 3 * plane + (size_t)c * plane + px];
      g_fg[(size_t)b * 4 * plane + (size_t)c * plane + px] = gr * m;
      g_env[(size_t)b * 4 * plane + (size_t)c * plane + px] = gr * (1.f - m);
      gm += gr * (fc - ec);
    }
    g_fg[(size_t)b * 4 * plane + 3 * (size_t)plane + px] = gm;
    g_env[(size_t)b * 4 * plane + 3 * (size_t)plane + px] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ host side
static RasterParams make_params(const DbwRenderSettings& s, const Workspace& w, const float* faces_alpha) {
  RasterParams P;
  memset(&P, 0, sizeof(P));
  P.B = s.n_views; P.H = s.height; P.W = s.width; P.K = s.faces_per_pixel; P.V = s.n_verts; P.F = s.n_faces; P.M = s.n_maps;
  P.alpha_stride = s.alpha_view_stride; P.inv_alpha_group = 1.f / (float)(s.alpha_group > 0 ? s.alpha_group : 1);
  P.n_static_faces = s.n_static_faces; P.view_rows = s.view_rows;
  P.n_alpha = s.n_faces / (s.alpha_group > 0 ? s.alpha_group : 1);
  P.sigma = s.sigma; P.blur = s.blur_radius; P.sqrt_blur = sqrtf(s.blur_radius); P.bg0 = s.background[0]; P.bg1 = s.background[1]; P.bg2 = s.background[2];
  P.clip_inside = s.clip_inside; P.persp = s.perspective_correct; P.clipb = s.clip_barycentric; P.detach_bary = s.detach_bary;
  P.bbox = w.bbox; P.rec = w.rec; P.rec2 = w.rec2; P.conv = w.conv; P.view_flags = w.view_flags; P.view_bbox = w.view_bbox;
  P.view_nvis = w.view_nvis; P.vis_list = w.vis_list;
  P.cbin_count = w.cbin_count; P.cbin_list = w.cbin_list; P.cbin_nx = w.cbin_nx; P.cbin_ny = w.cbin_ny;
  P.maps4 = w.maps4; P.faces_alpha = faces_alpha;
  P.frag = s.save_fragment_state ? w.frag : nullptr; P.nfrag = s.save_fragment_state ? w.nfrag : nullptr;
  P.frag_rgb = s.save_fragment_state ? w.frag_rgb : nullptr;
  return P;
}

// backward grid: (view, 16-px tile column, strip of DBW_BWD_TILES_K1 / _KN tiles)
static dim3 bwd_grid(const DbwRenderSettings& s) {
  const int strip_rows = (s.faces_per_pixel == 1 ? DBW_BWD_TILES_K1 : DBW_BWD_TILES_KN) * (DBW_BWD_NT / 16);
  return dim3(s.n_views, (s.width + TILE_W - 1) / TILE_W, (s.height + strip_rows - 1) / strip_rows);
}
// one flag per backward CTA of a single-layer pass that is not detached (see raster_bary_backward_kernel)
static size_t bary_flag_count(const DbwRenderSettings& s) {
  if (s.faces_per_pixel != 1 || s.detach_bary) return 0;
  const dim3 g = bwd_grid(s);
  return (size_t)g.x * g.y * g.z;
}

// dynamic shared memory of the raster kernels: K list entries (forward) / K saved scalars (backward) of 20 B per thread, the
// map table, and `alpha_tables` arrays of n_alpha floats (the opacity sums, then the opacity table) when they fit
static size_t frag_smem_bytes(int K, int NT, int M, int n_alpha = 0, int alpha_tables = 1) {
  return (size_t)K * NT * (sizeof(float4) + sizeof(float)) + (size_t)M * sizeof(int4) +
         (n_alpha <= DBW_ALPHA_SMEM_MAX ? (size_t)alpha_tables * n_alpha * sizeof(float) : 0);
}

// BLOCKS: blocks_loss_kernel, whose dispatch guarantees ep_grad and n_alpha <= DBW_ALPHA_SMEM_MAX; DEPTH: depth_forward_kernel
template <int NT, bool BLOCKS = false, bool DEPTH = false>
static cudaError_t launch_forward(const RasterParams& P, cudaStream_t st, const DepthIO* depth = nullptr) {
  static_assert(!BLOCKS || NT == 128, "blocks_loss_kernel runs 128 threads");
  const dim3 grid(P.B, (P.W + TILE_W - 1) / TILE_W, (P.H + NT / 16 - 1) / (NT / 16));       // see centre_out()
  const size_t smem = BLOCKS ? frag_smem_bytes(P.K, NT, P.M, P.faces_alpha ? P.n_alpha : 0, 2)
                             : frag_smem_bytes(P.K, NT, P.M, P.ep_grad && P.faces_alpha && P.g_faces_alpha ? P.n_alpha : 0);
  auto go = [&](auto kern) -> cudaError_t {
    if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
    kern<<<grid, NT, smem, st>>>(P);
    return cudaSuccess;
  };
  if (BLOCKS) return go(blocks_loss_kernel);
  if (DEPTH) {
    if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(depth_forward_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
    depth_forward_kernel<NT><<<grid, NT, smem, st>>>(P, *depth);
    return cudaSuccess;
  }
  return P.ep_target ? go(raster_forward_kernel<NT, true>) : go(raster_forward_kernel<NT, false>);
}

// the backward scratch and the gradients a loss-epilogue forward computes itself (dbw_render_forward_loss_grad)
struct EpilogueGrad { void* scratch; size_t scratch_bytes; int32_t mask; };
// viz: the resolving hard render of dbw_render_forward_viz (its frames replace out_rgba)
static int render_forward_impl(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                               const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                               const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                               size_t workspace_bytes, const float* face_shade, float* out_dists, const DbwLossEpilogue* ep,
                               void* stream, const EpilogueGrad* eg = nullptr, const VizOut* viz = nullptr,
                               const PhongIn* phong = nullptr, const DepthIO* depth = nullptr);

extern "C" int dbw_render_forward(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                  const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                  const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                                  size_t workspace_bytes, const float* face_shade, float* out_dists, void* stream) {
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_rgba, topk_ids,
                             workspace, workspace_bytes, face_shade, out_dists, nullptr, stream);
}

// the epilogue arguments both loss-epilogue forwards require; `who` names the entry point in the error message
static int check_epilogue(const DbwLossEpilogue* ep, const char* who) {
  const char* why = !ep ? "null epilogue"
                  : (!ep->env_rgba || !ep->target || !ep->g_env || !ep->loss_partials) ? "env_rgba, target, g_env and loss_partials are required"
                  : (ep->n_partials < 1 || (ep->n_partials & (ep->n_partials - 1))) ? "n_partials must be a power of two"
                  : nullptr;
  if (!why) return 0;
  char msg[160];
  snprintf(msg, sizeof(msg), "%s: %s", who, why);
  return fail(msg);
}

extern "C" int dbw_render_forward_loss(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                       const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                       const float* T, const float* faces_alpha, float* out_g_rgba, int32_t* topk_ids,
                                       void* workspace, size_t workspace_bytes, const DbwLossEpilogue* ep, void* stream) {
  if (check_epilogue(ep, "dbw_render_forward_loss")) return -1;
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_g_rgba, topk_ids,
                             workspace, workspace_bytes, nullptr, nullptr, ep, stream);
}

extern "C" int dbw_render_forward_loss_grad(const DbwRenderSettings* s, const float* verts, const int32_t* faces,
                                            const float* faces_uvs, const int32_t* face_map, const float* maps,
                                            const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                                            void* workspace, size_t workspace_bytes, const DbwLossEpilogue* ep, int32_t grad_mask,
                                            void* bwd_scratch, size_t bwd_scratch_bytes, void* stream) {
  if (check_epilogue(ep, "dbw_render_forward_loss_grad")) return -1;
  if (validate(s)) return -1;
  if (!s->detach_bary) return fail("dbw_render_forward_loss_grad: the pass must be detach_bary");
  if (s->maps_are_texels4 != 2) return fail("dbw_render_forward_loss_grad: the maps must be float4 cell maps (maps_are_texels4 = 2)");
  if (grad_mask & ~(DBW_GRAD_VERTS | DBW_GRAD_MAPS | DBW_GRAD_ALPHA)) return fail("dbw_render_forward_loss_grad: unknown grad_mask bits");
  if (s->save_fragment_state) return fail("dbw_render_forward_loss_grad: no fragment records are written (save_fragment_state must be 0)");
  if (!bwd_scratch) return fail("dbw_render_forward_loss_grad: null backward scratch");
  const EpilogueGrad eg = {bwd_scratch, bwd_scratch_bytes, grad_mask};
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, nullptr, nullptr,
                             workspace, workspace_bytes, nullptr, nullptr, ep, stream, &eg);
}

static int render_forward_impl(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                               const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                               const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                               size_t workspace_bytes, const float* face_shade, float* out_dists, const DbwLossEpilogue* ep,
                               void* stream, const EpilogueGrad* eg, const VizOut* viz, const PhongIn* phong,
                               const DepthIO* depth) {
  if (validate(s)) return -1;
  if (!verts || !faces || !faces_uvs || !face_map || !maps || !map_table || (!out_rgba && !eg && !viz) || !workspace)
    return fail("dbw_render_forward: null pointer argument");
  if (!s->verts_are_ndc && (!R || !T)) return fail("dbw_render_forward: R and T are required unless verts_are_ndc");
  if (s->save_fragment_state == 2 && faces_alpha) return fail("dbw_render_forward: save_fragment_state = 2 declares a pass without faces_alpha");
  Workspace w = carve(*s, workspace, !viz);
  if (workspace_bytes < w.total) return fail("dbw_render_forward: workspace too small (see dbw_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s->n_views, V = s->n_verts, F = s->n_faces;
  const float* verts_ndc = verts;
  if (!s->verts_are_ndc) {
    const int n_thr = B * (V > 4 ? V : 4);          // the kernel also resets the per-view bbox / flags (4 ints per view)
    project_verts_kernel<<<(n_thr + 255) / 256, 256, 0, st>>>(verts, R, T, s->fx, s->fy, s->px, s->py, s->proj_eps, B, V, w.verts_ndc,
                                                              w.view_bbox, w.view_flags, w.view_nvis);
    LAUNCH_CK("project_verts_kernel");
    verts_ndc = w.verts_ndc;
  } else {
    init_view_bbox_kernel<<<(B * 4 + 127) / 128, 128, 0, st>>>(w.view_bbox, w.view_flags, w.view_nvis, B);
    LAUNCH_CK("init_view_bbox_kernel");
  }
  face_setup_kernel<<<(B * F + 127) / 128, 128, 0, st>>>(verts_ndc, faces, B, V, F, s->z_clip, s->perspective_correct,
                                                         sqrtf(s->blur_radius), faces_uvs, face_map, map_table, w.bbox, w.rec,
                                                         w.rec2, w.conv, w.view_flags, w.view_bbox, w.view_nvis, w.vis_list,
                                                         s->width > s->height ? (float)s->width / s->height : 1.f,
                                                         s->height > s->width ? (float)s->height / s->width : 1.f);
  LAUNCH_CK("face_setup_kernel");
  if (!s->maps_are_texels4) {
    const int n_texels = s->n_map_floats / 3;
    const int blocks = stride_grid(n_texels, 8);
    if (blocks < 0) return fail("maps_to_float4_kernel: SM count", cudaGetLastError());
    maps_to_float4_kernel<<<blocks, 256, 0, st>>>(maps, w.maps4, n_texels);
    LAUNCH_CK("maps_to_float4_kernel");
  }
  RasterParams P = make_params(*s, w, faces_alpha);
  if (s->maps_are_texels4) P.maps4 = (const float4*)maps;
  P.map_table = map_table;
  P.out_rgba = out_rgba; P.topk = topk_ids; P.face_shade = face_shade; P.out_dists = out_dists;
  if (ep) {
    CK(cudaMemsetAsync(ep->loss_partials, 0, (size_t)ep->n_partials * sizeof(float), st));
    P.ep_env = ep->env_rgba; P.ep_target = ep->target; P.ep_g_env = ep->g_env; P.ep_rec = ep->rec;
    P.ep_partials = ep->loss_partials; P.ep_inv_count = ep->inv_count; P.ep_part_mask = ep->n_partials - 1;
    P.ep_skip_env_alpha = ep->env_alpha_unread && !g_keep_unread;
  }
  if (eg) {           // the scratch dbw_render_backward_deferred folds: zero-filled here, accumulated by the forward kernel
    const BwdScratch g = carve_bwd(*s, eg->scratch);
    if (eg->scratch_bytes < g.total) return fail("dbw_render_forward_loss_grad: backward scratch too small (see dbw_workspace_bytes)");
    CK(cudaMemsetAsync(eg->scratch, 0, g.total, st));
    P.ep_grad = 1;
    if (eg->mask & DBW_GRAD_VERTS) { P.g_tri = g.g_tri; P.g_conv = g.g_conv; }
    // cell_grad_copy picks the CTA's copy of g_cells; g_maps4 only says that a texture gradient is wanted
    if (eg->mask & DBW_GRAD_MAPS) { P.g_cells = g.g_cells; P.n_cells = s->n_map_floats / 3; P.g_maps4 = g.g_cells; }
    if ((eg->mask & DBW_GRAD_ALPHA) && faces_alpha) P.g_faces_alpha = g.g_alpha;
  }
  const int K = s->faces_per_pixel;
  {
    ScopedTimer timer(0, K, st);
    // a hard single-layer render without distances has its own kernel (dbw_debug_generic_kernel_only(1): the generic one)
    const bool hard = viz || phong || (K == 1 && s->sigma == 0.f && s->blur_radius == 0.f && !out_dists && !ep && !g_no_hard_kernel);
    if (!hard && w.cbin_list) {
      coarse_bin_kernel<<<dim3(B, w.cbin_nx * w.cbin_ny), 256, 0, st>>>(w.bbox, w.view_flags, F, s->height, s->width, w.cbin_nx,
                                                                        w.cbin_ny, w.cbin_count, w.cbin_list);
      ++g_launches;
    } else {
      P.cbin_list = nullptr; P.cbin_count = nullptr;
    }
    if (hard) {
      const dim3 grid(P.B, (P.W + 15) / 16, (P.H + 15) / 16);
      if (phong && viz) phong_resolve_hard_viz_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P, *viz, *phong);
      else if (phong) phong_hard_forward_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P, *phong);
      else if (viz) resolve_hard_viz_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P, *viz);
      else if (depth) depth_hard_forward_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P, *depth);
      else raster_hard_forward_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P);
    } else {
      // the coarse phase's blocks loss pass (K > 4) has a kernel of its own; anything it does not serve takes the generic one
      const bool blocks_loss = eg && K > 4 && !g_generic_blocks_loss && (!faces_alpha || P.n_alpha <= DBW_ALPHA_SMEM_MAX) &&
                               !P.out_rgba && !P.topk && !P.face_shade && !P.out_dists && !P.frag && !P.nfrag;
      cudaError_t e;
      if (blocks_loss) {
        ScopedTimer bl_timer(2, K, st);
        e = launch_forward<128, true>(P, st);
      } else if (depth) {
        e = K <= 4 ? launch_forward<DBW_FWD_NT_SMALLK, false, true>(P, st, depth) : launch_forward<DBW_FWD_NT, false, true>(P, st, depth);
      } else {
        e = K <= 4 ? launch_forward<DBW_FWD_NT_SMALLK>(P, st) : launch_forward<DBW_FWD_NT>(P, st);
      }
      if (e != cudaSuccess) return fail("raster_forward_kernel attribute", e);
    }
  }
  LAUNCH_CK("raster_forward_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ depth
// what the depth entry points leave to dbw_render_forward / dbw_render_backward (NULL: nothing)
static const char* depth_unsupported(const DbwRenderSettings& s) {
  if (s.view_rows) return "row bands (view_rows) are not supported";
  return nullptr;
}

extern "C" int dbw_render_forward_depth(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                        const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                        const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids,
                                        void* workspace, size_t workspace_bytes, const float* face_shade, float* out_dists,
                                        float* out_zbuf, float* out_depth, void* stream) {
  if (validate(s)) return -1;
  const char* why = depth_unsupported(*s);
  if (!why && face_shade) why = "lit renders (face_shade) are not supported";
  if (why) { char msg[192]; snprintf(msg, sizeof(msg), "dbw_render_forward_depth: %s", why); return fail(msg); }
  const DepthIO depth = {out_zbuf, out_depth, nullptr, nullptr};
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_rgba, topk_ids,
                             workspace, workspace_bytes, nullptr, out_dists, nullptr, stream, nullptr, nullptr, nullptr, &depth);
}

// ------------------------------------------------------------------------------------------------ resolving hard render
// settings that dbw_render_forward_viz cannot serve (NULL: none); the settings describe the factor x factor sample grid
static const char* viz_unsupported(const DbwRenderSettings& s, int32_t factor) {
  if (factor != 4) return "factor must be 4 (the supersampling of the reference's VizMeshRenderer)";
  if (s.faces_per_pixel != 1 || s.sigma != 0.f || s.blur_radius != 0.f) return "a hard render needs faces_per_pixel = 1, sigma = 0, blur_radius = 0";
  if (s.height % factor || s.width % factor) return "height and width (of the sample grid) must be multiples of factor";
  if (s.view_rows) return "view_rows is not supported";
  if (s.save_fragment_state) return "no fragment records are written (save_fragment_state must be 0)";
  return nullptr;
}

extern "C" int dbw_viz_workspace_bytes(const DbwRenderSettings* s, int32_t factor, size_t* bytes) {
  if (validate(s)) return -1;
  if (const char* why = viz_unsupported(*s, factor)) { char msg[192]; snprintf(msg, sizeof(msg), "dbw_viz_workspace_bytes: %s", why); return fail(msg); }
  if (!bytes) return fail("dbw_viz_workspace_bytes: null output");
  *bytes = carve(*s, nullptr, false).total;
  return 0;
}

extern "C" int dbw_render_forward_viz(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                      const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                      const float* T, const float* faces_alpha, const float* face_shade, int32_t factor,
                                      const float* bkg, int32_t bkg_views, float* out_rgba, uint8_t* out_rgb8, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  if (validate(s)) return -1;
  const char* why = viz_unsupported(*s, factor);
  if (!why && !out_rgba && !out_rgb8) why = "out_rgba and out_rgb8 are both NULL";
  if (!why && bkg && bkg_views != 1 && bkg_views != s->n_views) why = "bkg_views must be 1 or n_views";
  if (why) { char msg[192]; snprintf(msg, sizeof(msg), "dbw_render_forward_viz: %s", why); return fail(msg); }
  const size_t plane = (size_t)(s->height / factor) * (s->width / factor);
  if (3 * plane > (size_t)INT32_MAX) return fail("dbw_render_forward_viz: frame too large");
  const VizOut viz = {bkg, bkg && bkg_views > 1 ? (int)(3 * plane) : 0, out_rgba, out_rgb8};
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, nullptr, nullptr,
                             workspace, workspace_bytes, face_shade, nullptr, nullptr, stream, nullptr, &viz);
}

// ------------------------------------------------------------------------------------------------ phong hard render
extern "C" int dbw_render_forward_phong(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                        const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                        const float* T, const float* faces_alpha, const float* verts_world, const float* normals,
                                        const DbwPhongShading* shading, int32_t factor, const float* bkg, int32_t bkg_views,
                                        float* out_rgba, uint8_t* out_rgb8, void* workspace, size_t workspace_bytes, void* stream) {
  if (validate(s)) return -1;
  const char* why = nullptr;
  if (factor == 1) {
    if (s->faces_per_pixel != 1 || s->sigma != 0.f || s->blur_radius != 0.f) why = "a hard render needs faces_per_pixel = 1, sigma = 0, blur_radius = 0";
    else if (s->save_fragment_state) why = "no fragment records are written (save_fragment_state must be 0)";
    else if (bkg || out_rgb8) why = "bkg and out_rgb8 belong to factor 4";
    else if (!out_rgba) why = "null out_rgba";
  } else {
    why = viz_unsupported(*s, factor);
    if (!why && !out_rgba && !out_rgb8) why = "out_rgba and out_rgb8 are both NULL";
    if (!why && bkg && bkg_views != 1 && bkg_views != s->n_views) why = "bkg_views must be 1 or n_views";
  }
  if (!why && !shading) why = "null shading";
  if (!why && (shading->light < DBW_LIGHT_AMBIENT || shading->light > DBW_LIGHT_POINT)) why = "unknown light type";
  if (!why && (!verts_world || !normals || !R || !T)) why = "verts_world, normals, R and T are required";
  if (why) { char msg[192]; snprintf(msg, sizeof(msg), "dbw_render_forward_phong: %s", why); return fail(msg); }
  const PhongIn phong = {verts_world, normals, faces, R, T, *shading};
  if (factor == 1)
    return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_rgba, nullptr,
                               workspace, workspace_bytes, nullptr, nullptr, nullptr, stream, nullptr, nullptr, &phong);
  const size_t plane = (size_t)(s->height / factor) * (s->width / factor);
  if (3 * plane > (size_t)INT32_MAX) return fail("dbw_render_forward_phong: frame too large");
  const VizOut viz = {bkg, bkg && bkg_views > 1 ? (int)(3 * plane) : 0, out_rgba, out_rgb8};
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, nullptr, nullptr,
                             workspace, workspace_bytes, nullptr, nullptr, nullptr, stream, nullptr, &viz, &phong);
}

// adds the cell-gradient copies of the backward scratch into g_maps, times *scale (NULL = 1)
static int fold_gcells(const DbwRenderSettings& s, const BwdScratch& g, float* g_maps, const float* scale, cudaStream_t st) {
  const int n_entries = s.n_map_floats / 3;
  const int blocks = stride_grid(n_entries, 8);
  if (blocks < 0) return fail("fold_gcells_kernel: SM count", cudaGetLastError());
  fold_gcells_kernel<<<blocks, 256, 0, st>>>(g.g_cells, (float4*)g_maps, n_entries, scale);
  LAUNCH_CK("fold_gcells_kernel");
  return 0;
}

// the vertex and camera end of a backward: the triangle-slot gradients of the scratch, times *scale (NULL = 1), through the
// face setup backward onto the NDC vertices, then through the projection into g_verts and reduced per view into g_R / g_T.
// Nothing to do when no vertex or camera gradient is wanted.
static int geometry_backward(const DbwRenderSettings& s, const Workspace& w, const BwdScratch& g, const float* verts,
                             const int32_t* faces, const float* R, const float* T, const float* scale, float* g_verts,
                             float* g_R, float* g_T, cudaStream_t st) {
  if (!g_verts && !g_R && !g_T) return 0;
  const int B = s.n_views, V = s.n_verts, F = s.n_faces;
  const float* verts_ndc = s.verts_are_ndc ? verts : w.verts_ndc;
  float* g_ndc = s.verts_are_ndc ? g_verts : g.g_verts_ndc;
  face_setup_backward_kernel<<<(B * F + 127) / 128, 128, 0, st>>>(verts_ndc, faces, B, V, F, s.z_clip, s.perspective_correct,
                                                                  g.g_tri, g.g_conv, scale, g_ndc);
  LAUNCH_CK("face_setup_backward_kernel");
  if (!s.verts_are_ndc && g_verts) {
    project_verts_backward_kernel<<<(V * 32 + 127) / 128, 128, 0, st>>>(verts, R, T, s.fx, s.fy, s.px, s.py, s.proj_eps, B, V,
                                                                   g.g_verts_ndc, g_verts);
    LAUNCH_CK("project_verts_backward_kernel");
  }
  if (g_R || g_T) {
    camera_grad_kernel<<<B, DBW_CAM_NT, 0, st>>>(verts, R, T, s.fx, s.fy, s.px, s.py, s.proj_eps, V, g.g_verts_ndc, g_R, g_T);
    LAUNCH_CK("camera_grad_kernel");
  }
  return 0;
}

// g_zbuf / g_depth: the gradients of dbw_render_forward_depth's outputs (both NULL: the plain backward)
static int render_backward_impl(const DbwRenderSettings* s_in, const float* verts, const int32_t* faces, const float* faces_uvs,
                                const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                const float* T, const float* faces_alpha, const void* workspace, size_t workspace_bytes,
                                const float* grad_rgba, const float* grad_scale, float* g_verts, float* g_faces_alpha,
                                float* g_maps, float* g_R, float* g_T, void* bwd_scratch, size_t bwd_scratch_bytes,
                                void* stream, const float* g_zbuf = nullptr, const float* g_depth = nullptr,
                                const char* who = "dbw_render_backward");

extern "C" int dbw_render_backward(const DbwRenderSettings* s_in, const float* verts, const int32_t* faces, const float* faces_uvs,
                                   const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                   const float* T, const float* faces_alpha, const void* workspace, size_t workspace_bytes,
                                   const float* grad_rgba, const float* grad_scale, float* g_verts, float* g_faces_alpha,
                                   float* g_maps, float* g_R, float* g_T, void* bwd_scratch, size_t bwd_scratch_bytes,
                                   void* stream) {
  return render_backward_impl(s_in, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, workspace,
                              workspace_bytes, grad_rgba, grad_scale, g_verts, g_faces_alpha, g_maps, g_R, g_T, bwd_scratch,
                              bwd_scratch_bytes, stream);
}

extern "C" int dbw_render_backward_depth(const DbwRenderSettings* s, const float* verts, const int32_t* faces,
                                         const float* faces_uvs, const int32_t* face_map, const float* maps,
                                         const DbwMapDesc* map_table, const float* R, const float* T, const float* faces_alpha,
                                         const void* workspace, size_t workspace_bytes, const float* grad_rgba,
                                         const float* grad_scale, const float* g_zbuf, const float* g_depth, float* g_verts,
                                         float* g_faces_alpha, float* g_maps, float* g_R, float* g_T, void* bwd_scratch,
                                         size_t bwd_scratch_bytes, void* stream) {
  if (validate(s)) return -1;
  if (const char* why = depth_unsupported(*s)) { char msg[192]; snprintf(msg, sizeof(msg), "dbw_render_backward_depth: %s", why); return fail(msg); }
  return render_backward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, workspace,
                              workspace_bytes, grad_rgba, grad_scale, g_verts, g_faces_alpha, g_maps, g_R, g_T, bwd_scratch,
                              bwd_scratch_bytes, stream, g_zbuf, g_depth, "dbw_render_backward_depth");
}

static int render_backward_impl(const DbwRenderSettings* s_in, const float* verts, const int32_t* faces, const float* faces_uvs,
                                const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                const float* T, const float* faces_alpha, const void* workspace, size_t workspace_bytes,
                                const float* grad_rgba, const float* grad_scale, float* g_verts, float* g_faces_alpha,
                                float* g_maps, float* g_R, float* g_T, void* bwd_scratch, size_t bwd_scratch_bytes,
                                void* stream, const float* g_zbuf, const float* g_depth, const char* who) {
  char msg[256];                 // error messages name the entry point (`who`)
  if (validate(s_in)) return -1;
  if (!verts || !faces || !faces_uvs || !face_map || !maps || !map_table || !workspace || !grad_rgba || !bwd_scratch)
    { snprintf(msg, sizeof(msg), "%s: null pointer argument", who); return fail(msg); }
  if (!s_in->save_fragment_state) { snprintf(msg, sizeof(msg), "%s: the forward must run with save_fragment_state = 1 or 2", who); return fail(msg); }
  if (s_in->save_fragment_state == 2 && faces_alpha) { snprintf(msg, sizeof(msg), "%s: save_fragment_state = 2 declares a pass without faces_alpha", who); return fail(msg); }
  const bool cams = g_R != nullptr || g_T != nullptr;
  if (cams && s_in->verts_are_ndc) { snprintf(msg, sizeof(msg), "%s: no camera gradient when verts_are_ndc (R and T are not used)", who); return fail(msg); }
  if ((cams || (g_verts && !s_in->verts_are_ndc)) && (!R || !T)) { snprintf(msg, sizeof(msg), "%s: R and T are required unless verts_are_ndc", who); return fail(msg); }
  // every face moves in the image when the camera moves: a call with camera gradients differentiates the static faces too
  DbwRenderSettings s_local = *s_in;
  if (cams) s_local.n_static_faces = 0;
  const DbwRenderSettings* s = &s_local;
  Workspace w = carve(*s, (void*)workspace);
  BwdScratch g = carve_bwd(*s, bwd_scratch);
  if (workspace_bytes < w.total || bwd_scratch_bytes < g.total) { snprintf(msg, sizeof(msg), "%s: workspace too small", who); return fail(msg); }
  cudaStream_t st = (cudaStream_t)stream;
  const bool need_geom = g_verts != nullptr || cams;     // both are reductions of the per-view NDC vertex gradient
  CK(cudaMemsetAsync(bwd_scratch, 0, g.total, st));
  RasterParams P = make_params(*s, w, faces_alpha);
  if (s->maps_are_texels4) P.maps4 = (const float4*)maps;
  P.map_table = map_table;
  P.grad_rgba = grad_rgba; P.grad_scale = grad_scale; P.g_tri = need_geom ? g.g_tri : nullptr; P.g_conv = g.g_conv;
  P.g_faces_alpha = g_faces_alpha; P.g_maps4 = g_maps ? (s->maps_are_texels4 ? (float4*)g_maps : g.g_maps4) : nullptr;
  const DepthIO dz = {nullptr, nullptr, g_zbuf, g_depth};
  const bool dep = g_zbuf != nullptr || g_depth != nullptr;
  const int n_entries = s->n_map_floats / 3;
  if (g_maps && s->maps_are_texels4 == 2) { P.g_cells = g.g_cells; P.n_cells = n_entries; }
  const dim3 grid = bwd_grid(*s);        // see centre_out()
  const size_t smem = frag_smem_bytes(s->faces_per_pixel, DBW_BWD_NT, s->n_maps, P.n_alpha);
  {
    ScopedTimer timer(1, s->faces_per_pixel, st);       // both launches of a split single-layer pass
    auto launch = [&](auto kern) -> cudaError_t {
      if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
      kern<<<grid, DBW_BWD_NT, smem, st>>>(P);
      return cudaSuccess;
    };
    auto launch_depth = [&](auto kern) -> cudaError_t {
      if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
      kern<<<grid, DBW_BWD_NT, smem, st>>>(P, dz);
      return cudaSuccess;
    };
    const bool det = s->detach_bary != 0, al = faces_alpha != nullptr, k1 = s->faces_per_pixel == 1;
    // A single-layer pass that is not detached runs as the detached kernel (texture, opacity and distance gradients of
    // every pixel) plus raster_bary_backward_kernel over the strips that hold faces with vertex gradients
    const bool split = k1 && !det && need_geom;
    if (split) P.bary_flags = g.bary_flags;
    cudaError_t e;
    if (!dep)
      e = k1  ? (al ? launch(raster_backward_kernel<true, true, true>) : launch(raster_backward_kernel<true, false, true>))
        : det ? (al ? launch(raster_backward_kernel<true, true, false>) : launch(raster_backward_kernel<true, false, false>))
              : (al ? launch(raster_backward_kernel<false, true, false>) : launch(raster_backward_kernel<false, false, false>));
    else        // the same dispatch; the split single-layer pass keeps raster_bary_backward_kernel for the colour's barycentrics
      e = k1  ? (al ? launch_depth(depth_backward_kernel<true, true, true>) : launch_depth(depth_backward_kernel<true, false, true>))
        : det ? (al ? launch_depth(depth_backward_kernel<true, true, false>) : launch_depth(depth_backward_kernel<true, false, false>))
              : (al ? launch_depth(depth_backward_kernel<false, true, false>) : launch_depth(depth_backward_kernel<false, false, false>));
    if (e != cudaSuccess) return fail("raster_backward_kernel attribute", e);
    LAUNCH_CK("raster_backward_kernel");
    if (split) {
      const size_t gsmem = (size_t)s->n_maps * sizeof(int4);
      auto launch_bary = [&](auto kern) -> cudaError_t {
        if (gsmem > 40 * 1024) { cudaError_t e2 = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsmem); if (e2 != cudaSuccess) return e2; }
        kern<<<grid, DBW_BWD_NT, gsmem, st>>>(P);
        return cudaSuccess;
      };
      e = al ? launch_bary(raster_bary_backward_kernel<true>) : launch_bary(raster_bary_backward_kernel<false>);
      if (e != cudaSuccess) return fail("raster_bary_backward_kernel attribute", e);
      LAUNCH_CK("raster_bary_backward_kernel");
    }
  }
  if (P.g_cells && fold_gcells(*s, g, g_maps, nullptr, st)) return -1;
  if (g_maps && !s->maps_are_texels4) {
    const int n_texels = s->n_map_floats / 3;
    const int blocks = stride_grid(n_texels, 8);
    if (blocks < 0) return fail("fold_gmaps_kernel: SM count", cudaGetLastError());
    fold_gmaps_kernel<<<blocks, 256, 0, st>>>(g.g_maps4, g_maps, n_texels);
    LAUNCH_CK("fold_gmaps_kernel");
  }
  return geometry_backward(*s, w, g, verts, faces, R, T, nullptr, g_verts, g_R, g_T, st);
}

extern "C" int dbw_render_backward_deferred(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* R,
                                            const float* T, const void* workspace, size_t workspace_bytes, const float* grad_scale,
                                            float* g_verts, float* g_faces_alpha, float* g_maps, float* g_R, float* g_T,
                                            void* bwd_scratch, size_t bwd_scratch_bytes, void* stream) {
  if (validate(s)) return -1;
  if (!verts || !faces || !workspace || !grad_scale || !bwd_scratch) return fail("dbw_render_backward_deferred: null pointer argument");
  if (s->maps_are_texels4 != 2) return fail("dbw_render_backward_deferred: the maps must be float4 cell maps (maps_are_texels4 = 2)");
  const bool cams = g_R != nullptr || g_T != nullptr;
  if (cams && s->verts_are_ndc) return fail("dbw_render_backward_deferred: no camera gradient when verts_are_ndc (R and T are not used)");
  if ((cams || (g_verts && !s->verts_are_ndc)) && (!R || !T)) return fail("dbw_render_backward_deferred: R and T are required");
  const Workspace w = carve(*s, (void*)workspace);
  const BwdScratch g = carve_bwd(*s, bwd_scratch);
  if (workspace_bytes < w.total || bwd_scratch_bytes < g.total) return fail("dbw_render_backward_deferred: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  // the differentiation itself ran inside raster_forward_kernel<NT, true>: this is the blocks backward a caller times
  ScopedTimer timer(1, s->faces_per_pixel, st);
  if (g_maps && fold_gcells(*s, g, g_maps, grad_scale, st)) return -1;
  if (g_faces_alpha) {
    const int n_alpha = s->n_faces / (s->alpha_group > 0 ? s->alpha_group : 1);
    const int n = s->alpha_view_stride ? s->n_views * n_alpha : n_alpha;
    scale_add_kernel<<<(n + 255) / 256, 256, 0, st>>>(g_faces_alpha, g.g_alpha, n, grad_scale);
    LAUNCH_CK("scale_add_kernel");
  }
  return geometry_backward(*s, w, g, verts, faces, R, T, grad_scale, g_verts, g_R, g_T, st);
}

extern "C" int dbw_composite_mse(int32_t n_views, int32_t height, int32_t width, const float* fg, const float* env,
                                 const float* imgs, float inv_count, float* rec, float* loss_sum, float* g_fg, float* g_env,
                                 void* stream) {
  if (!fg || !env || !imgs || !loss_sum) return fail("dbw_composite_mse: null pointer argument");
  if (n_views <= 0 || height <= 0 || width <= 0) return fail("dbw_composite_mse: bad sizes");
  const int plane = height * width;
  const long long total = (long long)n_views * plane;
  if (total > 0x7fffffffLL) return fail("dbw_composite_mse: too many pixels for one call");
  const int blocks = stride_grid(total, 16);
  if (blocks < 0) return fail("composite_mse_kernel: SM count", cudaGetLastError());
  composite_mse_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((int)total, plane, fg, env, imgs, inv_count, rec, loss_sum, g_fg, g_env);
  LAUNCH_CK("composite_mse_kernel");
  return 0;
}

extern "C" int dbw_composite_mse_backward(int32_t n_views, int32_t height, int32_t width, const float* fg, const float* env,
                                          const float* imgs, float inv_count, const float* g_loss, const float* g_rec,
                                          float* g_fg, float* g_env, void* stream) {
  if (!fg || !env || !imgs || !g_fg || !g_env) return fail("dbw_composite_mse_backward: null pointer argument");
  if (n_views <= 0 || height <= 0 || width <= 0) return fail("dbw_composite_mse_backward: bad sizes");
  const int plane = height * width;
  const long long total = (long long)n_views * plane;
  if (total > 0x7fffffffLL) return fail("dbw_composite_mse_backward: too many pixels for one call");
  const int blocks = stride_grid(total, 16);
  if (blocks < 0) return fail("composite_backward_kernel: SM count", cudaGetLastError());
  composite_backward_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((int)total, plane, fg, env, imgs, inv_count, g_loss, g_rec, g_fg, g_env);
  LAUNCH_CK("composite_backward_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ host-buffer entry point
static struct { char* base; size_t cap; } g_arena = {nullptr, 0};

static int arena_reserve(size_t bytes) {
  if (bytes <= g_arena.cap) return 0;
  if (g_arena.base) cudaFree(g_arena.base);
  g_arena.base = nullptr; g_arena.cap = 0;
  CK(cudaMalloc((void**)&g_arena.base, bytes));
  g_arena.cap = bytes;
  return 0;
}
extern "C" void dbw_host_arena_release(void) {
  if (g_arena.base) cudaFree(g_arena.base);
  g_arena.base = nullptr; g_arena.cap = 0;
}

extern "C" int dbw_render_forward_host(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                       const int32_t* face_map, const float* maps, size_t maps_floats, const DbwMapDesc* map_table,
                                       const float* R, const float* T, const float* faces_alpha, float* out_rgba, void* stream) {
  if (validate(s)) return -1;
  if (!verts || !faces || !faces_uvs || !face_map || !maps || !map_table || !out_rgba) return fail("dbw_render_forward_host: null pointer argument");
  const size_t B = s->n_views, V = s->n_verts, F = s->n_faces, M = s->n_maps, HW = (size_t)s->height * s->width, K = s->faces_per_pixel;
  size_t fwd = 0; dbw_workspace_bytes(s, &fwd, nullptr);
  const size_t n_verts_f = (s->verts_are_ndc ? B : 1) * V * 3;
  const size_t n_alpha = faces_alpha ? (s->alpha_view_stride ? B * F : F) : 0;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
  const size_t o_verts = take(n_verts_f * 4), o_faces = take(F * 3 * 4), o_fuv = take(F * 6 * 4), o_fmap = take(F * 4);
  const size_t o_maps = take(maps_floats * 4), o_tab = take(M * sizeof(DbwMapDesc)), o_R = take(B * 9 * 4), o_T = take(B * 3 * 4);
  const size_t o_alpha = take(n_alpha * 4 + 4), o_out = take(B * 4 * HW * 4), o_ids = take(B * K * HW * 4), o_ws = take(fwd);
  if (arena_reserve(off)) return -1;
  char* d = g_arena.base;
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(d + o_verts, verts, n_verts_f * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_faces, faces, F * 3 * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_fuv, faces_uvs, F * 6 * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_fmap, face_map, F * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_maps, maps, maps_floats * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_tab, map_table, M * sizeof(DbwMapDesc), cudaMemcpyHostToDevice, st));
  if (R) CK(cudaMemcpyAsync(d + o_R, R, B * 9 * 4, cudaMemcpyHostToDevice, st));
  if (T) CK(cudaMemcpyAsync(d + o_T, T, B * 3 * 4, cudaMemcpyHostToDevice, st));
  if (faces_alpha) CK(cudaMemcpyAsync(d + o_alpha, faces_alpha, n_alpha * 4, cudaMemcpyHostToDevice, st));
  const int rc = dbw_render_forward(s, (float*)(d + o_verts), (int32_t*)(d + o_faces), (float*)(d + o_fuv), (int32_t*)(d + o_fmap),
                                    (float*)(d + o_maps), (DbwMapDesc*)(d + o_tab), R ? (float*)(d + o_R) : nullptr,
                                    T ? (float*)(d + o_T) : nullptr, faces_alpha ? (float*)(d + o_alpha) : nullptr,
                                    (float*)(d + o_out), (int32_t*)(d + o_ids), d + o_ws, fwd, nullptr, nullptr, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out_rgba, d + o_out, B * 4 * HW * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}
