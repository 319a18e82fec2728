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
static Workspace carve(const DbwRenderSettings& s, void* base) {
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
  const bool use_bins = B * nb * S * sizeof(int) <= ((size_t)1 << 30) && nb > 1;
  w.cbin_count = use_bins ? (int*)(p + off) : nullptr;  off += use_bins ? align_up(B * nb * sizeof(int)) : 0;
  w.cbin_list = use_bins ? (int*)(p + off) : nullptr;   off += use_bins ? align_up(B * nb * S * sizeof(int)) : 0;
  w.maps4 = (float4*)(p + off);    off += s.maps_are_texels4 ? 0 : align_up((size_t)(s.n_map_floats / 3) * sizeof(float4));
  const size_t npx = B * (size_t)s.height * s.width;
  w.frag = (float4*)(p + off);     off += s.save_fragment_state ? align_up(npx * (size_t)s.faces_per_pixel * sizeof(float4)) : 0;
  w.frag_rgb = (float4*)(p + off); off += s.save_fragment_state ? align_up(npx * (size_t)s.faces_per_pixel * sizeof(float4)) : 0;
  w.nfrag = (unsigned char*)(p + off); off += s.save_fragment_state ? align_up(npx) : 0;
  w.total = off; return w;
}
struct BwdScratch { float* g_tri; float* g_conv; float* g_verts_ndc; float4* g_maps4; size_t total; };
static BwdScratch carve_bwd(const DbwRenderSettings& s, void* base) {
  BwdScratch w; char* p = (char*)base; size_t off = 0;
  const size_t B = s.n_views, V = s.n_verts, S = 2 * (size_t)s.n_faces;
  w.g_tri = (float*)(p + off);        off += align_up(B * S * 9 * sizeof(float));
  w.g_conv = (float*)(p + off);       off += align_up(B * S * 9 * sizeof(float));
  w.g_verts_ndc = (float*)(p + off);  off += align_up(B * V * 3 * sizeof(float));
  w.g_maps4 = (float4*)(p + off);     off += s.maps_are_texels4 ? 0 : align_up((size_t)(s.n_map_floats / 3) * sizeof(float4));
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
  if (2 * (long long)s->n_faces > DBW_FRAG_SLOT_MASK) return fail("too many faces: triangle slots are stored in 20 bits");
  if (s->n_maps > DBW_FRAG_MAX_MAPS) return fail("too many texture maps: a fragment's map is stored in 9 bits");
  if (s->sigma < 0.f || s->blur_radius < 0.f) return fail("sigma and blur_radius must be >= 0");
  if (s->n_map_floats <= 0 || s->n_map_floats % 3 != 0) return fail("n_map_floats must be a positive multiple of 3");
  return 0;
}

// ------------------------------------------------------------------------------------------------ texel repack
__global__ void maps_to_float4_kernel(const float* __restrict__ maps, float4* __restrict__ maps4, int n_texels) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_texels; i += gridDim.x * blockDim.x)
    maps4[i] = make_float4(maps[3 * i], maps[3 * i + 1], maps[3 * i + 2], 0.f);
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
    const float xv = X * r[0] + Y * r[3] + Z * r[6] + t[0];
    const float yv = X * r[1] + Y * r[4] + Z * r[7] + t[1];
    const float zv = X * r[2] + Y * r[5] + Z * r[8] + t[2];
    const float sgn = (zv > 0.f) ? 1.f : ((zv < 0.f) ? -1.f : 1.f);
    const bool clamped = fabsf(zv) < eps;
    const float den = sgn * fmaxf(fabsf(zv), eps);
    const float* g = g_ndc + ((size_t)b * V + v) * 3;
    const float gx = g[0], gy = g[1], gz = g[2];
    const float nx = fx * xv + px * zv, ny = fy * yv + py * zv;
    const float gxv = gx * fx / den, gyv = gy * fy / den;
    float gzv = gz + (gx * px + gy * py) / den;
    if (!clamped) gzv -= (gx * nx + gy * ny) / (den * den);
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
// per-tile scan of all 8000 slots was half of the forward's instructions.
__global__ void coarse_bin_kernel(const float4* __restrict__ bbox, const int* __restrict__ view_flags, int F, int H, int W,
                                  int nbx, int nby, int* __restrict__ cbin_count, int* __restrict__ cbin_list) {
  __shared__ int s_n;
  const int view = blockIdx.x, bin = blockIdx.y, bx = bin % nbx, by = bin / nbx;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) s_n = 0;
  __syncthreads();
  const int x0 = bx * DBW_CBIN, x1 = min(x0 + DBW_CBIN, W) - 1, y0 = by * DBW_CBIN, y1 = min(y0 + DBW_CBIN, H) - 1;
  // NDC extents of the bin's pixel centres (+X is left, +Y is up: the last column / row has the smallest coordinate)
  const float xmin = pix_to_ndc(W - 1 - x1, W, H), xmax = pix_to_ndc(W - 1 - x0, W, H);
  const float ymin = pix_to_ndc(H - 1 - y1, H, W), ymax = pix_to_ndc(H - 1 - y0, H, W);
  const int nslots = (view_flags[view] & 1) ? 2 * F : F;
  const float4* bb = bbox + (size_t)view * 2 * F;
  int* list = cbin_list + ((size_t)view * gridDim.y + bin) * 2 * F;
  for (int base = 0; base < nslots; base += blockDim.x) {
    const int sl = base + tid;
    bool hit = false;
    if (sl < nslots) { const float4 b = __ldg(&bb[sl]); hit = !(b.x > xmax || b.y < xmin || b.z > ymax || b.w < ymin); }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m == 0u) continue;
    int wbase = 0;
    if (lane == 0) wbase = atomicAdd(&s_n, __popc(m));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (hit) list[wbase + __popc(m & ((1u << lane) - 1u))] = sl;
  }
  __syncthreads();
  if (tid == 0) cbin_count[(size_t)view * gridDim.y + bin] = s_n;
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
  // backward only
  const float* grad_rgba; float* g_tri; float* g_conv; float* g_faces_alpha; float4* g_maps4;
  const float* grad_scale;   // device scalar multiplied into grad_rgba (the upstream gradient of a fused loss) or NULL
  // fused compositing + MSE epilogue of the forward (DbwLossEpilogue); ep_target == NULL: plain render
  const float* ep_env; const float* ep_target; float* ep_g_env; float* ep_rec; float* ep_partials;
  float ep_inv_count; int ep_part_mask;
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
// the map table in shared memory: (first texel, H, W, -) per map, staged once per CTA -- a fragment's tap addresses then
// depend on no global load
__device__ __forceinline__ void stage_map_table(const RasterParams& P, int4* s_desc, int tid, int nthreads) {
  for (int m = tid; m < P.M; m += nthreads) {
    const DbwMapDesc d = P.map_table[m];
    s_desc[m] = make_int4(d.offset / 3, d.height, d.width, 0);
  }
}
__device__ __forceinline__ void tap_only(float u, float v, int4 d, Texel4& s) { s.tap = tex_tap(u, v, d.x, d.y, d.z); }
__device__ __forceinline__ void fetch_color(const RasterParams& P, float u, float v, int4 d, Texel4& s) {
  s.tap = tex_tap(u, v, d.x, d.y, d.z);
  s.c00 = ld_texel(P.maps4, s.tap.i00); s.c01 = ld_texel(P.maps4, s.tap.i01);
  s.c10 = ld_texel(P.maps4, s.tap.i10); s.c11 = ld_texel(P.maps4, s.tap.i11);
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

// CTA -> (view, tile) mapping of the raster kernels.  CTAs are dispatched in linear grid order, so the grid is laid out as
// (view, tile column, tile row RANK) with the rows ranked centre-out: every view's central rows -- where the blocks are and the
// CTAs run longest -- are dispatched first, the cheap border rows last.  With the few waves a view-sharded rank has (8750 CTAs
// at 8 GPUs = 8 waves), the last wave otherwise holds the heavy tiles of the last view while most SMs idle.
__device__ __forceinline__ int centre_out(int rank, int n) {
  const int c = n >> 1;
  return (rank & 1) ? c - ((rank + 1) >> 1) : c + (rank >> 1);
}

// One kernel for every K: the per-pixel list of the K nearest fragments lives in (dynamic) shared memory (dbw_fraglist.cuh).
// EP: with the compositing + MSE loss epilogue (DbwLossEpilogue); a template flag so that plain renders carry none of it
template <int NT, bool EP>
__global__ void __launch_bounds__(NT, NT <= 128 ? DBW_FWD_MINB : DBW_FWD_SMALLK_MINB) raster_forward_kernel(const RasterParams P) {
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
  DbwMapDesc my_desc = {0, 0, 0, 0};
  if (tid < P.M) my_desc = P.map_table[tid];
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
  const bool dist_inside = (!P.clip_inside && P.sigma > 0.f) || P.out_dists != nullptr;

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
  auto scan_hit = [&](int& s, float4& bb) -> bool {
    if (s >= nslots) return false;
    if (clist) s = __ldg(clist + s);
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
  if (tid < P.M) s_desc[tid] = make_int4(my_desc.offset / 3, my_desc.height, my_desc.width, 0);
  for (int m = tid + NT; m < P.M; m += NT) { const DbwMapDesc d = P.map_table[m]; s_desc[m] = make_int4(d.offset / 3, d.height, d.width, 0); }
  __syncthreads();
  const int total = s_count;
  if (total <= CAP) {
    if (total > 0) raster_list(total);
  } else {
    // chunked path (more than CAP faces touch this tile): re-scan, flushing the list whenever it may overflow
    __syncthreads();
    if (tid == 0) s_count = 0;
    __syncthreads();
    constexpr int BS = NT < CAP ? NT : CAP;          // slots scanned per batch: a batch never overflows an empty list
    for (int base = 0; base < nslots; base += BS) {
      float4 bb = make_float4(0, 0, 0, 0);
      int sl = base + tid;
      const bool hit = tid < BS && scan_hit(sl, bb);
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      int wbase = 0;
      if (lane == 0 && m) wbase = atomicAdd(&s_count, __popc(m));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      if (hit) {
        const int pos = wbase + __popc(m & ((1u << lane) - 1u));
        s_slot[pos] = sl; s_bbox[pos] = bb;
      }
      __syncthreads();
      const int cnt = s_count;
      const bool last = base + BS >= nslots;
      if (cnt > CAP - BS || last) {
        raster_list(cnt);
        __syncthreads();              // every warp is done with the list before it is reset and refilled
        if (tid == 0) s_count = 0;
        __syncthreads();
      }
    }
  }

  float ep_sq = 0.f;          // this pixel's squared error (fused loss epilogue)
  if (live) {
  // ---- shade + blend the sorted fragments front to back (layered_rgb_blend, Appendix B)
  float occ = 1.f, r = 0.f, g = 0.f, bl = 0.f;
  const size_t plane = (size_t)P.H * P.W;
  const size_t pix = (size_t)yi * P.W + xi;
  int n_saved = 0;
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
    const float4 e = lA[k * NT];
    const int bits = __float_as_int(e.y), slot = bits & DBW_FRAG_SLOT_MASK;
    const float d0 = e.z;
    if (P.topk) P.topk[((size_t)view * K + k) * plane + pix] = slot;
    if (P.out_dists) P.out_dists[((size_t)view * K + k) * plane + pix] = d0;
    if (occ == 0.f) continue;     // behind a fully opaque fragment (fine phase: alpha = 1 inside a face): contributes exactly 0
    const float v = lV[k * NT];
    const int face = slot >= P.F ? slot - P.F : slot;
    Texel4 tx;
    fetch_color(P, e.w, v, s_desc[(unsigned)bits >> DBW_FRAG_MAP_SHIFT], tx);
    float a = frag_alpha(d0, P.sigma, P.clip_inside);
    if (P.faces_alpha) a *= __ldg(&P.faces_alpha[alpha_index(P, view, face)]);
    if (P.face_shade) {          // flat shading: colour = texel * (ambient + diffuse * relu(n . l)) per (view, face)
      const float* m = P.face_shade + ((size_t)view * P.F + face) * 3;
      tx.color.x *= __ldg(m); tx.color.y *= __ldg(m + 1); tx.color.z *= __ldg(m + 2);
    }
    if (P.frag) {                 // what the backward streams instead of re-deriving geometry and texels: two 16 B records
      const size_t fi = ((size_t)view * K + k) * plane + pix;
      P.frag[fi] = make_float4(e.y, e.w, v, d0);
      P.frag_rgb[fi] = make_float4(tx.color.x, tx.color.y, tx.color.z, 0.f);
      n_saved = k + 1;
    }
    const float w = occ * a;
    r += w * tx.color.x; g += w * tx.color.y; bl += w * tx.color.z;
    occ *= (1.f - a);
  }
  if (P.nfrag) P.nfrag[(size_t)view * plane + pix] = (unsigned char)n_saved;
  for (int k = n; k < K; ++k) {
    if (P.topk) P.topk[((size_t)view * K + k) * plane + pix] = -1;
    if (P.out_dists) P.out_dists[((size_t)view * K + k) * plane + pix] = -1.f;
  }
  float* o = P.out_rgba + (size_t)view * 4 * plane + pix;
  const float fc[3] = {r + occ * P.bg0, g + occ * P.bg1, bl + occ * P.bg2};
  const float m = 1.f - occ;
  if (!EP) {
    o[0] = fc[0]; o[plane] = fc[1]; o[2 * plane] = fc[2]; o[3 * plane] = m;
  } else {
    // fused epilogue (same arithmetic as composite_mse_kernel): composite over the environment render, squared error
    // against the target, and the gradients of the MSE w.r.t. both layers -- out_rgba receives d loss / d (this render)
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
      o[(size_t)c * plane] = gr * m;
      ge[(size_t)c * plane] = gr * (1.f - m);
      gm += gr * (fc[c] - ec);
    }
    o[3 * plane] = gm;
    ge[3 * plane] = 0.f;
  }
  }   // live
  if (EP) {
    // one atomic per warp into a strip of partial sums (the caller adds them up): no single hot address
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ep_sq += __shfl_xor_sync(0xffffffffu, ep_sq, off);
    if (lane == 0 && ep_sq != 0.f) {
      const unsigned cta = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;      // any spread over the strip will do
      atomicAdd(&P.ep_partials[(cta * (NT / 32) + warp) & P.ep_part_mask], ep_sq * P.ep_inv_count);
    }
  }
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
__global__ void __launch_bounds__(HARD_NT, 5) raster_hard_forward_kernel(const RasterParams P) {
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
  for (int m = tid; m < P.M; m += HARD_NT) { const DbwMapDesc d = P.map_table[m]; s_desc[m] = make_int4(d.offset / 3, d.height, d.width, 0); }
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
  if (!live) return;
  const size_t plane = (size_t)P.H * P.W;
  const size_t pix = (size_t)yi * P.W + xi;
  float* o = P.out_rgba + (size_t)view * 4 * plane + pix;
  if (best_j < 0) {
    o[0] = P.bg0; o[plane] = P.bg1; o[2 * plane] = P.bg2; o[3 * plane] = 0.f;
    if (P.nfrag) P.nfrag[(size_t)view * plane + pix] = 0;
    if (P.topk) P.topk[(size_t)view * plane + pix] = -1;
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
    P.frag_rgb[fi] = make_float4(tx.color.x, tx.color.y, tx.color.z, 0.f);
    P.nfrag[fi] = 1;
  }
  if (P.topk) P.topk[(size_t)view * plane + pix] = best_slot;
  const float occ = 1.f - a;
  o[0] = a * tx.color.x + occ * P.bg0; o[plane] = a * tx.color.y + occ * P.bg1; o[2 * plane] = a * tx.color.z + occ * P.bg2;
  o[3 * plane] = a;
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
#pragma unroll
      for (int j = 0; j < c; ++j) {
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

// Group sums through the integer reduction unit (REDUX, sm_80+): the members of a group (`grp`, all executing this) scale
// their N values by a common power of two derived from the group's largest magnitude, round to int32 (|x| < 2^25, so 32
// addends cannot overflow), add them with one REDUX.SUM per value and scale back.  Quantisation: 2^-25 of the group's largest
// magnitude per addend -- the size of fp32 summation rounding -- and the sum itself is exact and order-independent.
// One instruction per value instead of a shuffle butterfly.  Returns the sums to every member.
template <int N>
__device__ __forceinline__ void group_sum_redux(unsigned grp, const float (&v)[N], float (&out)[N]) {
  float mx = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) mx = fmaxf(mx, fabsf(v[i]));
  const unsigned gmax = __reduce_max_sync(grp, __float_as_uint(mx));        // non-negative floats order like their bit patterns
  int ex = (int)(gmax >> 23) - 127;
  ex = ex < -100 ? -100 : ex;
  const float scale = __int_as_float((127 + 24 - ex) << 23), inv = __int_as_float((127 - 24 + ex) << 23);
#pragma unroll
  for (int i = 0; i < N; ++i) out[i] = (float)__reduce_add_sync(grp, __float2int_rn(v[i] * scale)) * inv;
}

template <int N>
__device__ __forceinline__ void warp_agg_add(float* __restrict__ dst, int stride, int key, const float (&v)[N], int lane) {
#ifdef DBW_AGG_REDUX
  unsigned todo_r = __ballot_sync(0xffffffffu, key >= 0);
  while (todo_r) {
    const int leader = __ffs(todo_r) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = (key == lk);
    const unsigned grp = __ballot_sync(0xffffffffu, mine);
    if (mine) {
      float r[N];
      group_sum_redux<N>(grp, v, r);
      if (lane == leader) {
#pragma unroll
        for (int i = 0; i < N; ++i) if (r[i] != 0.f) atomicAdd(dst + (size_t)lk * stride + i, r[i]);
      }
    }
    todo_r &= ~grp;
  }
  return;
#endif
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

// Texture-gradient scatter of one fragment: 4 bilinear taps x RGB.  Under magnification (the environment maps seen
// through a narrow field of view: hundreds of pixels per texel) whole warps hit the same 2x2 texel footprint, so
// lanes that share the footprint with >= 8 others are reduced (16-wide spread reduction: total i lands in lane 2i and
// is added to channel i % 3 of tap i / 3); the rest issue plain vector reds.
// Coherence is probed from the first pending lane only (no match.any): an incoherent warp pays two ballots.
__device__ __forceinline__ void warp_tex_scatter(float4* __restrict__ gm, int key, int i01, int i10, int i11,
                                                 const float (&v)[12], int lane) {
  unsigned todo = __ballot_sync(0xffffffffu, key >= 0);
  bool done = key < 0;
  while (todo) {
    const int leader = __ffs(todo) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = !done && key == lk;
    const unsigned grp = __ballot_sync(0xffffffffu, mine);
    if (__popc(grp) < 8) break;
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = (i < 12 && mine) ? v[i] : 0.f;
    const float r = warp_sum_spread<16>(x, lane);
    // the footprint (i00 = key, i01, i10, i11) is the same for every lane of the group: fetch it from the leader
    const int l01 = __shfl_sync(0xffffffffu, i01, leader), l10 = __shfl_sync(0xffffffffu, i10, leader);
    const int l11 = __shfl_sync(0xffffffffu, i11, leader);
    const int idx = lane >> 1, tap = idx / 3, ch = idx - tap * 3;
    const int texel = tap == 0 ? lk : (tap == 1 ? l01 : (tap == 2 ? l10 : l11));
    if ((lane & 1) == 0 && idx < 12 && texel >= 0 && r != 0.f) atomicAdd(reinterpret_cast<float*>(gm + texel) + ch, r);
    done = done || mine;
    todo &= ~grp;
  }
  if (!done) {
    red_add_v4(gm + key, v[0], v[1], v[2]);
    if (i01 >= 0) red_add_v4(gm + i01, v[3], v[4], v[5]);
    if (i10 >= 0) red_add_v4(gm + i10, v[6], v[7], v[8]);
    if (i11 >= 0) red_add_v4(gm + i11, v[9], v[10], v[11]);
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
// vertices.  4-wide spread reduction (5 shuffles): total i lands in lane 8 i and goes to float off[i] of the slot's 9.
__device__ __forceinline__ void warp_agg_add_edge(float* __restrict__ g_tri, int key, const float (&v)[4], int lane) {
  unsigned todo = __ballot_sync(0xffffffffu, key >= 0);
  while (todo) {
    const int leader = __ffs(todo) - 1;
    const int lk = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = (key == lk);
    const unsigned grp = __ballot_sync(0xffffffffu, mine);
    const int edge = lk & 3;
    // vertex pair of the edge: 0 = (v0, v1), 1 = (v0, v2), 2 = (v1, v2); vertex j's (x, y) live at floats 3j, 3j+1
    const int ia = edge == 2 ? 3 : 0, ib = edge == 0 ? 3 : 6;
    float* d = g_tri + (size_t)(lk >> 2) * 9;
#ifdef DBW_AGG_REDUX
    if (mine) {
      float r[4];
      group_sum_redux<4>(grp, v, r);
      if (lane == leader) {
        if (r[0] != 0.f) atomicAdd(d + ia, r[0]);
        if (r[1] != 0.f) atomicAdd(d + ia + 1, r[1]);
        if (r[2] != 0.f) atomicAdd(d + ib, r[2]);
        if (r[3] != 0.f) atomicAdd(d + ib + 1, r[3]);
      }
    }
    todo &= ~grp;
    continue;
#endif
    if (__popc(grp) <= DBW_AGG_MIN) {
      if (mine) {
        if (v[0] != 0.f) atomicAdd(d + ia, v[0]);
        if (v[1] != 0.f) atomicAdd(d + ia + 1, v[1]);
        if (v[2] != 0.f) atomicAdd(d + ib, v[2]);
        if (v[3] != 0.f) atomicAdd(d + ib + 1, v[3]);
      }
    } else {
      float x[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] = mine ? v[i] : 0.f;
      const float r = warp_sum_spread<4>(x, lane);
      const int idx = lane >> 3;
      if ((lane & 7) == 0 && r != 0.f) atomicAdd(d + (idx < 2 ? ia + idx : ib + idx - 2), r);
    }
    todo &= ~grp;
  }
}

// One thread per pixel.  Pass 1 streams the pixel's saved fragment records {slot, u, v, signed distance} front to back,
// re-fetches the four texels of each (the float4 atlas is L2-resident), scatters the texture gradient and -- unless
// detach_bary -- re-derives the geometry for the barycentric-path vertex gradient (skipped for faces whose vertices are
// constants); pass 2 walks back to front with the division-free suffix recurrence of SURVEY Appendix B for d/d(alpha_k)
// -> opacity and distance -> vertex gradients.  Loops are warp-uniform (trip count = warp max) so that the aggregation
// helpers run converged.
#define DBW_ALPHA_SMEM_MAX 512      // opacity entries per view that a CTA may pre-accumulate in shared memory
// 16 x 8 tiles a backward CTA walks (each warp its own patch of every tile, no barrier between, the next patch's first-level
// loads in flight).  A single-layer pass is a chain of DRAM latencies per pixel and gains from 8 tiles; the K = 10 blocks
// pass walks one (more tiles make longer CTAs and worse tails)
#define DBW_BWD_TILES_K1 8
#define DBW_BWD_TILES_KN 1

// K1: faces_per_pixel == 1 (the environment pass): no record prefetch registers, at most one trip through the loops
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
      f.g0 = go[0]; f.g1 = go[plane]; f.g2 = go[2 * plane]; f.g3 = go[3 * plane];
      f.n = (int)P.nfrag[(size_t)view * plane + px];
      f.rec = P.frag[(size_t)view * P.K * plane + px];          // speculative: a valid workspace address whether or not a
      f.rgb = P.frag_rgb[(size_t)view * P.K * plane + px];      // fragment exists
    }
  };
  First first_next;
  load_first(0, first_next);
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
    float gv9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float gc9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float tv[12] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
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
          tkey = tx.tap.i00; t01 = tx.tap.i01; t10 = tx.tap.i10; t11 = tx.tap.i11;
          tv[0] = gcx * tx.tap.w00; tv[1] = gcy * tx.tap.w00; tv[2] = gcz * tx.tap.w00;
          tv[3] = gcx * tx.tap.w01; tv[4] = gcy * tx.tap.w01; tv[5] = gcz * tx.tap.w01;
          tv[6] = gcx * tx.tap.w10; tv[7] = gcy * tx.tap.w10; tv[8] = gcz * tx.tap.w10;
          tv[9] = gcx * tx.tap.w11; tv[10] = gcy * tx.tap.w11; tv[11] = gcz * tx.tap.w11;
        }
        if (bary_path && P.g_tri) {
          // colour -> (ix, iy) -> (u, v) -> barycentrics -> vertices  (grid_sample backward + A6)
          const float fx0 = (float)tx.tap.x0, fy0 = (float)tx.tap.y0;
          const float ex = fx0 + 1.f - tx.tap.ix, wx = tx.tap.ix - fx0, ey = fy0 + 1.f - tx.tap.iy, wy = tx.tap.iy - fy0;
          const float d00 = tx.c00.x * gcx + tx.c00.y * gcy + tx.c00.z * gcz, d01 = tx.c01.x * gcx + tx.c01.y * gcy + tx.c01.z * gcz;
          const float d10 = tx.c10.x * gcx + tx.c10.y * gcy + tx.c10.z * gcz, d11 = tx.c11.x * gcx + tx.c11.y * gcy + tx.c11.z * gcz;
          const float gix = (d01 - d00) * ey + (d11 - d10) * wy;
          const float giy = (d10 - d00) * ex + (d11 - d01) * wx;
          const float gu = gix * tx.tap.mx, gv = giy * tx.tap.my;
          f3 gbu = {gu * s.uv01.x + gv * s.uv01.y, gu * s.uv01.z + gv * s.uv01.w, gu * s.u2 + gv * s.v2};
          const size_t gsl = slot_base + slot;
          f3 gbc = gbu;
          if (s.t.flags & 1) {
            // z-clipped face (the ground plane under the camera is one): bu = bc @ conv, so the conversion matrix gets
            // gradient too; it is accumulated per slot with the same warp aggregation as the vertex gradient below
            const float* cv = P.conv + gsl * 9;
            gbc.x = cv[0] * gbu.x + cv[1] * gbu.y + cv[2] * gbu.z;
            gbc.y = cv[3] * gbu.x + cv[4] * gbu.y + cv[5] * gbu.z;
            gbc.z = cv[6] * gbu.x + cv[7] * gbu.y + cv[8] * gbu.z;
            ckey = slot;
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
          key = slot;
          gv9[0] = g0.x; gv9[1] = g0.y; gv9[2] = gz0; gv9[3] = g1.x; gv9[4] = g1.y; gv9[5] = gz1; gv9[6] = g2.x; gv9[7] = g2.y; gv9[8] = gz2;
        }
      }
      occ *= (1.f - a);
    }
    if (P.g_maps4) warp_tex_scatter(P.g_maps4, tkey, t01, t10, t11, tv, lane);
    if (!DETACH) {
      if (__ballot_sync(0xffffffffu, key >= 0)) warp_agg_add<9>(P.g_tri + slot_base * 9, 9, key, gv9, lane);
      if (__ballot_sync(0xffffffffu, ckey >= 0)) warp_agg_add<9>(P.g_conv + slot_base * 9, 9, ckey, gc9, lane);
    }
  }

  // pass 2: suffix recurrence on the stored per-fragment scalars -- no division (alpha may be exactly 1)
  float Tacc = P.bg0 * gr + P.bg1 * gg + P.bg2 * gb - ga;
  if (want_alpha || want_dist) {
    // the edge geometry of a halo fragment (2 vertices + 1 / |edge|^2, from the face record) is loaded one layer ahead
    struct EdgeGeom { float4 r0; float2 r1; float4 r3; };
    auto load_edge = [&](int kk, EdgeGeom& g) {
      g.r0 = make_float4(0.f, 0.f, 0.f, 0.f); g.r1 = make_float2(0.f, 0.f); g.r3 = g.r0;
      if (!want_dist || kk < 0 || kk >= n) return;
      const int bits = s_bits[kk * DBW_BWD_NT];
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
        const float4 q = s_q[k * DBW_BWD_NT];      // (alpha, cdot, e, occ)
        const float g_alpha = q.w * (q.y - Tacc);
        Tacc = q.x * q.y + (1.f - q.x) * Tacc;
        if (g_alpha != 0.f) {
          const int bits = s_bits[k * DBW_BWD_NT], slot = bits & DBW_FRAG_SLOT_MASK;
          const int face = slot >= P.F ? slot - P.F : slot;
          if (want_alpha) { akey = alpha_index(P, alpha_in_smem ? 0 : view, face); aval = g_alpha * q.z; }
          if (want_dist) {
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
  }   // tiles of the strip
  if (alpha_in_smem) {               // one global atomic per (CTA, opacity entry) instead of one per (warp, layer, entry)
    __syncthreads();
    for (int i = tid; i < P.n_alpha; i += DBW_BWD_NT) {
      const float v = s_galpha[i];
      if (v != 0.f) atomicAdd(&P.g_faces_alpha[(size_t)view * P.alpha_stride + i], v);
    }
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
                                           float* __restrict__ g_verts_ndc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * F) return;
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
    if (ga[j][0] != 0.f) atomicAdd(g, ga[j][0]);
    if (ga[j][1] != 0.f) atomicAdd(g + 1, ga[j][1]);
    if (ga[j][2] != 0.f) atomicAdd(g + 2, ga[j][2]);
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

// dynamic shared memory of the raster kernels: K list entries (forward) / K saved scalars (backward) of 20 B per thread
static size_t frag_smem_bytes(int K, int NT, int M, int n_alpha = 0) {
  return (size_t)K * NT * (sizeof(float4) + sizeof(float)) + (size_t)M * sizeof(int4) + (n_alpha <= 512 ? (size_t)n_alpha * sizeof(float) : 0);
}

template <int NT>
static cudaError_t launch_forward(const RasterParams& P, cudaStream_t st) {
  const dim3 grid(P.B, (P.W + TILE_W - 1) / TILE_W, (P.H + NT / 16 - 1) / (NT / 16));       // see centre_out()
  const size_t smem = frag_smem_bytes(P.K, NT, P.M);
  auto go = [&](auto kern) -> cudaError_t {
    if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
    kern<<<grid, NT, smem, st>>>(P);
    return cudaSuccess;
  };
  return P.ep_target ? go(raster_forward_kernel<NT, true>) : go(raster_forward_kernel<NT, false>);
}

extern "C" int dbw_render_forward(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                  const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                  const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return dbw_render_forward_ex(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_rgba, topk_ids,
                               workspace, workspace_bytes, nullptr, nullptr, stream);
}

static int render_forward_impl(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                               const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                               const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                               size_t workspace_bytes, const float* face_shade, float* out_dists, const DbwLossEpilogue* ep,
                               void* stream);

extern "C" int dbw_render_forward_ex(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                     const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                     const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                                     size_t workspace_bytes, const float* face_shade, float* out_dists, void* stream) {
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_rgba, topk_ids,
                             workspace, workspace_bytes, face_shade, out_dists, nullptr, stream);
}

extern "C" int dbw_render_forward_loss(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                       const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                       const float* T, const float* faces_alpha, float* out_g_rgba, int32_t* topk_ids,
                                       void* workspace, size_t workspace_bytes, const DbwLossEpilogue* ep, void* stream) {
  if (!ep) return fail("dbw_render_forward_loss: null epilogue");
  if (!ep->env_rgba || !ep->target || !ep->g_env || !ep->loss_partials)
    return fail("dbw_render_forward_loss: env_rgba, target, g_env and loss_partials are required");
  if (ep->n_partials < 1 || (ep->n_partials & (ep->n_partials - 1))) return fail("dbw_render_forward_loss: n_partials must be a power of two");
  return render_forward_impl(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, out_g_rgba, topk_ids,
                             workspace, workspace_bytes, nullptr, nullptr, ep, stream);
}

static int render_forward_impl(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                               const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                               const float* T, const float* faces_alpha, float* out_rgba, int32_t* topk_ids, void* workspace,
                               size_t workspace_bytes, const float* face_shade, float* out_dists, const DbwLossEpilogue* ep,
                               void* stream) {
  if (validate(s)) return -1;
  if (!verts || !faces || !faces_uvs || !face_map || !maps || !map_table || !out_rgba || !workspace)
    return fail("dbw_render_forward: null pointer argument");
  if (!s->verts_are_ndc && (!R || !T)) return fail("dbw_render_forward: R and T are required unless verts_are_ndc");
  Workspace w = carve(*s, workspace);
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
  }
  const int K = s->faces_per_pixel;
  {
    ScopedTimer timer(0, K, st);
    // a hard single-layer render without distances has its own kernel (dbw_debug_generic_kernel_only(1): the generic one)
    const bool hard = K == 1 && s->sigma == 0.f && s->blur_radius == 0.f && !out_dists && !ep && !g_no_hard_kernel;
    if (!hard && w.cbin_list) {
      coarse_bin_kernel<<<dim3(B, w.cbin_nx * w.cbin_ny), 256, 0, st>>>(w.bbox, w.view_flags, F, s->height, s->width, w.cbin_nx,
                                                                        w.cbin_ny, w.cbin_count, w.cbin_list);
      ++g_launches;
    } else {
      P.cbin_list = nullptr; P.cbin_count = nullptr;
    }
    if (hard) {
      const dim3 grid(P.B, (P.W + 15) / 16, (P.H + 15) / 16);
      raster_hard_forward_kernel<<<grid, HARD_NT, (size_t)P.M * sizeof(int4), st>>>(P);
    } else {
      const cudaError_t e = K <= 4 ? launch_forward<DBW_FWD_NT_SMALLK>(P, st) : launch_forward<DBW_FWD_NT>(P, st);
      if (e != cudaSuccess) return fail("raster_forward_kernel attribute", e);
    }
  }
  LAUNCH_CK("raster_forward_kernel");
  return 0;
}

extern "C" int dbw_render_backward(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                   const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                   const float* T, const float* faces_alpha, const int32_t* topk_ids, const void* workspace,
                                   size_t workspace_bytes, const float* grad_rgba, float* g_verts, float* g_faces_alpha,
                                   float* g_maps, void* bwd_scratch, size_t bwd_scratch_bytes, void* stream) {
  return dbw_render_backward_scaled(s, verts, faces, faces_uvs, face_map, maps, map_table, R, T, faces_alpha, topk_ids, workspace,
                                    workspace_bytes, grad_rgba, nullptr, g_verts, g_faces_alpha, g_maps, bwd_scratch,
                                    bwd_scratch_bytes, stream);
}

extern "C" int dbw_render_backward_scaled(const DbwRenderSettings* s, const float* verts, const int32_t* faces, const float* faces_uvs,
                                          const int32_t* face_map, const float* maps, const DbwMapDesc* map_table, const float* R,
                                          const float* T, const float* faces_alpha, const int32_t* topk_ids, const void* workspace,
                                          size_t workspace_bytes, const float* grad_rgba, const float* grad_scale, float* g_verts,
                                          float* g_faces_alpha, float* g_maps, void* bwd_scratch, size_t bwd_scratch_bytes,
                                          void* stream) {
  if (validate(s)) return -1;
  (void)topk_ids;          // kept in the signature for ABI continuity: the backward streams the workspace's fragment records
  if (!verts || !faces || !faces_uvs || !face_map || !maps || !map_table || !workspace || !grad_rgba || !bwd_scratch)
    return fail("dbw_render_backward: null pointer argument");
  if (!s->save_fragment_state) return fail("dbw_render_backward: the forward must run with save_fragment_state = 1");
  Workspace w = carve(*s, (void*)workspace);
  BwdScratch g = carve_bwd(*s, bwd_scratch);
  if (workspace_bytes < w.total || bwd_scratch_bytes < g.total) return fail("dbw_render_backward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s->n_views, V = s->n_verts, F = s->n_faces;
  const bool need_geom = g_verts != nullptr;
  CK(cudaMemsetAsync(bwd_scratch, 0, g.total, st));
  RasterParams P = make_params(*s, w, faces_alpha);
  if (s->maps_are_texels4) P.maps4 = (const float4*)maps;
  P.map_table = map_table;
  P.grad_rgba = grad_rgba; P.grad_scale = grad_scale; P.g_tri = need_geom ? g.g_tri : nullptr; P.g_conv = g.g_conv;
  P.g_faces_alpha = g_faces_alpha; P.g_maps4 = g_maps ? (s->maps_are_texels4 ? (float4*)g_maps : g.g_maps4) : nullptr;
  const int strip_rows = (s->faces_per_pixel == 1 ? DBW_BWD_TILES_K1 : DBW_BWD_TILES_KN) * (DBW_BWD_NT / 16);
  dim3 grid(B, (s->width + TILE_W - 1) / TILE_W, (s->height + strip_rows - 1) / strip_rows);       // see centre_out()
  const size_t smem = frag_smem_bytes(s->faces_per_pixel, DBW_BWD_NT, s->n_maps, P.n_alpha);
  {
    auto launch = [&](auto kern) -> cudaError_t {
      if (smem > 40 * 1024) { cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e; }
      ScopedTimer timer(1, s->faces_per_pixel, st);
      kern<<<grid, DBW_BWD_NT, smem, st>>>(P);
      return cudaSuccess;
    };
    const bool det = s->detach_bary != 0, al = faces_alpha != nullptr, k1 = s->faces_per_pixel == 1;
    cudaError_t e = k1  ? (det ? (al ? launch(raster_backward_kernel<true, true, true>) : launch(raster_backward_kernel<true, false, true>))
                               : (al ? launch(raster_backward_kernel<false, true, true>) : launch(raster_backward_kernel<false, false, true>)))
                  : det ? (al ? launch(raster_backward_kernel<true, true, false>) : launch(raster_backward_kernel<true, false, false>))
                        : (al ? launch(raster_backward_kernel<false, true, false>) : launch(raster_backward_kernel<false, false, false>));
    if (e != cudaSuccess) return fail("raster_backward_kernel attribute", e);
  }
  LAUNCH_CK("raster_backward_kernel");
  if (g_maps && !s->maps_are_texels4) {
    const int n_texels = s->n_map_floats / 3;
    const int blocks = stride_grid(n_texels, 8);
    if (blocks < 0) return fail("fold_gmaps_kernel: SM count", cudaGetLastError());
    fold_gmaps_kernel<<<blocks, 256, 0, st>>>(g.g_maps4, g_maps, n_texels);
    LAUNCH_CK("fold_gmaps_kernel");
  }
  if (need_geom) {
    const float* verts_ndc = s->verts_are_ndc ? verts : w.verts_ndc;
    float* g_ndc = s->verts_are_ndc ? g_verts : g.g_verts_ndc;
    face_setup_backward_kernel<<<(B * F + 127) / 128, 128, 0, st>>>(verts_ndc, faces, B, V, F, s->z_clip, s->perspective_correct,
                                                                    g.g_tri, g.g_conv, g_ndc);
    LAUNCH_CK("face_setup_backward_kernel");
    if (!s->verts_are_ndc) {
      if (!R || !T) return fail("dbw_render_backward: R and T are required unless verts_are_ndc");
      project_verts_backward_kernel<<<(V * 32 + 127) / 128, 128, 0, st>>>(verts, R, T, s->fx, s->fy, s->px, s->py, s->proj_eps, B, V,
                                                                     g.g_verts_ndc, g_verts);
      LAUNCH_CK("project_verts_backward_kernel");
    }
  }
  return 0;
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
                                    (float*)(d + o_out), (int32_t*)(d + o_ids), d + o_ws, fwd, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out_rgba, d + o_out, B * 4 * HW * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}
