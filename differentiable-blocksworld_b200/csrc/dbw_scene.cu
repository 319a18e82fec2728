// dbw_scene.cu -- fused scene construction of the DBW render hot path (include/dbw_render.h, "scene" entry points).
//
// Replaces the ~200 small eager kernels per step of the reference's build_blocks / build_ground / build_bkg
// (src/model/dbw.py:267-352) and their autograd:
//   * superquadric mesh build: sq_eps -> parametric superquadric (src/utils/superquadric.py:10-14) -> * ratio * (exp(S)+s_min)
//     -> @ rot6d(R_6d) + T -> world transform (dbw.py:311,344), for the N blocks AND the ground plane, ONE launch;
//     backward: one CTA per primitive reduces its vertices' gradients into (sq_eps, S, R_6d, T) without atomics;
//   * texture prep: sigmoid -> optional 8x8 box decimation (avg_pool + nearest upsample, dbw.py:331-334) -> circular u
//     padding (dbw.py:339-341) written straight into the float4 texel atlas the rasterizer samples; backward folds the
//     atlas gradient through padding, decimation and the sigmoid.
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);
#define SCENE_LAUNCH_CK(name) do { dbw_count_launch_(); cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return dbw_fail_(name, _e); } while (0)

// ------------------------------------------------------------------------------------------------ geometry
#include "dbw_scene_math.cuh"

// out: (n_static + Vg + N*Vb, 3) world-space vertices: the static environment vertices (copied; there may be none), the
// ground, then the blocks
__global__ void scene_geometry_forward_kernel(const GeomParams P, float* __restrict__ out, const float* __restrict__ env_static,
                                              int n_static) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int nb = P.n_blocks * P.verts_per_block;
  if (i < n_static * 3) out[i] = env_static[i];
  if (i >= nb + P.n_ground_verts) return;
  out += (ptrdiff_t)(n_static + (i < nb ? P.n_ground_verts : -nb)) * 3;      // blocks move behind the ground
  const int prim = i < nb ? i / P.verts_per_block : P.n_blocks;
  const int v = i < nb ? i - prim * P.verts_per_block : i - nb;
  float u[3], aux[6], R[9], sc[3] = {1.f, 1.f, 1.f};
  local_vertex(P, prim, v, u, aux);
  const float* T;
  if (prim < P.n_blocks) {
    rot6d(P.R6 + prim * 6, R);
#pragma unroll
    for (int c = 0; c < 3; ++c) sc[c] = expf(P.S[prim * 3 + c]) + P.scale_min;
    T = P.T + prim * 3;
  } else { rot6d(P.R6g, R); T = P.Tg; }
  const float x = u[0] * sc[0], y = u[1] * sc[1], z = u[2] * sc[2];
  // row vector times matrix (dbw.py:311), then the world transform (dbw.py:344)
  const float px = (x * R[0] + y * R[3] + z * R[6] + T[0]) * P.S_world;
  const float py = (x * R[1] + y * R[4] + z * R[7] + T[1]) * P.S_world;
  const float pz = (x * R[2] + y * R[5] + z * R[8] + T[2]) * P.S_world;
  const float* W = P.R_world.m;
  out[i * 3 + 0] = px * W[0] + py * W[3] + pz * W[6] + P.T_world[0];
  out[i * 3 + 1] = px * W[1] + py * W[4] + pz * W[7] + P.T_world[1];
  out[i * 3 + 2] = px * W[2] + py * W[5] + pz * W[8] + P.T_world[2];
}

// one CTA (64 threads) per primitive; outputs are WRITTEN (not accumulated)
__global__ void __launch_bounds__(64) scene_geometry_backward_kernel(const GeomParams P, const float* __restrict__ g_blocks,
                                                                     const float* __restrict__ g_ground,
                                                                     float* __restrict__ g_sq_eps, float* __restrict__ g_S,
                                                                     float* __restrict__ g_R6, float* __restrict__ g_T,
                                                                     float* __restrict__ g_R6g, float* __restrict__ g_Tg) {
  const int prim = blockIdx.x, v = threadIdx.x;
  const bool is_block = prim < P.n_blocks;
  const int nv = is_block ? P.verts_per_block : P.n_ground_verts;
  float R[9], sc[3] = {1.f, 1.f, 1.f};
  rot6d(is_block ? P.R6 + prim * 6 : P.R6g, R);
  if (is_block) for (int c = 0; c < 3; ++c) sc[c] = expf(P.S[prim * 3 + c]) + P.scale_min;
  // per-thread partial sums: gT(3) gR(9) gS(3) ge(2)
  float acc[17];
#pragma unroll
  for (int k = 0; k < 17; ++k) acc[k] = 0.f;
  for (int vv = v; vv < nv; vv += 64) {
    float u[3], aux[6] = {0, 0, 0, 0, 1, 1};
    local_vertex(P, prim, vv, u, aux);
    const float* g_v = is_block ? g_blocks + (size_t)(prim * P.verts_per_block + vv) * 3 : g_ground + (size_t)vv * 3;
    const float gx = g_v[0], gy = g_v[1], gz = g_v[2];
    const float* W = P.R_world.m;
    // world transform backward: g_p = S_world * (g @ R_world^T)
    const float gp[3] = {(gx * W[0] + gy * W[1] + gz * W[2]) * P.S_world, (gx * W[3] + gy * W[4] + gz * W[5]) * P.S_world,
                         (gx * W[6] + gy * W[7] + gz * W[8]) * P.S_world};
    const float xs[3] = {u[0] * sc[0], u[1] * sc[1], u[2] * sc[2]};
    acc[0] += gp[0]; acc[1] += gp[1]; acc[2] += gp[2];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[3 + a * 3 + b] += xs[a] * gp[b];
    if (is_block) {
      // g wrt the scaled vertex, then scale and superquadric exponents
      const float gxs[3] = {R[0] * gp[0] + R[1] * gp[1] + R[2] * gp[2], R[3] * gp[0] + R[4] * gp[1] + R[5] * gp[2],
                            R[6] * gp[0] + R[7] * gp[1] + R[8] * gp[2]};
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[12 + c] += gxs[c] * u[c] * (sc[c] - P.scale_min);       // d exp(S) = exp(S)
      const float gu[3] = {gxs[0] * sc[0] * P.ratio, gxs[1] * sc[1] * P.ratio, gxs[2] * sc[2] * P.ratio};
      const float ce = aux[0], se = aux[1], co = aux[2], so = aux[3];
      const float g_ce = gu[0] * so + gu[2] * co, g_so = gu[0] * ce, g_se = gu[1], g_co = gu[2] * ce;
      const float eta = P.sq_eta[prim * P.verts_per_block + vv], om = P.sq_omega[prim * P.verts_per_block + vv];
      const float ace = fabsf(cosf(eta)), ase = fabsf(sinf(eta)), aco = fabsf(cosf(om)), aso = fabsf(sinf(om));
      // d/de sign(x)|x|^e = sign(x)|x|^e ln|x|, with torch's convention 0 where |x| == 0
      acc[15] += (ace > 0.f ? g_ce * ce * logf(ace) : 0.f) + (ase > 0.f ? g_se * se * logf(ase) : 0.f);
      acc[16] += (aco > 0.f ? g_co * co * logf(aco) : 0.f) + (aso > 0.f ? g_so * so * logf(aso) : 0.f);
    }
  }
  __shared__ float red[2][17];
#pragma unroll
  for (int k = 0; k < 17; ++k) {
    float x = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t[17];
#pragma unroll
    for (int k = 0; k < 17; ++k) t[k] = red[0][k] + red[1][k];
    float gd6[6];
    rot6d_backward(is_block ? P.R6 + prim * 6 : P.R6g, t + 3, gd6);
    if (is_block) {
      for (int c = 0; c < 3; ++c) { g_T[prim * 3 + c] = t[c]; g_S[prim * 3 + c] = t[12 + c]; }
      for (int c = 0; c < 6; ++c) g_R6[prim * 6 + c] = gd6[c];
      for (int c = 0; c < 2; ++c) {
        const float sg = 1.f / (1.f + expf(-P.sq_eps[prim * 2 + c]));
        g_sq_eps[prim * 2 + c] = t[15 + c] * 1.8f * sg * (1.f - sg);
      }
    } else {
      for (int c = 0; c < 3; ++c) g_Tg[c] = t[c];
      for (int c = 0; c < 6; ++c) g_R6g[c] = gd6[c];
    }
  }
}

static GeomParams make_geom(const DbwSceneGeometry* g) {
  GeomParams P;
  P.n_blocks = g->n_blocks; P.verts_per_block = g->verts_per_block; P.n_ground_verts = g->n_ground_verts;
  P.sq_eta = g->sq_eta; P.sq_omega = g->sq_omega; P.sq_eps = g->sq_eps; P.S = g->S; P.R6 = g->R_6d; P.T = g->T;
  P.ground_verts = g->ground_verts; P.R6g = g->R_6d_ground; P.Tg = g->T_ground;
  P.ratio = g->ratio_block_scene; P.scale_min = g->scale_min; P.S_world = g->S_world;
  for (int i = 0; i < 9; ++i) P.R_world.m[i] = g->R_world[i];
  for (int i = 0; i < 3; ++i) P.T_world[i] = g->T_world[i];
  return P;
}

extern "C" int dbw_scene_geometry_forward(const DbwSceneGeometry* g, const float* env_static_verts, int32_t n_env_static,
                                          float* verts_out, void* stream) {
  if (!g || !verts_out || (n_env_static > 0 && !env_static_verts)) return dbw_fail_("dbw_scene_geometry_forward: null pointer argument", cudaSuccess);
  if (g->n_blocks < 0 || g->verts_per_block <= 0 || g->n_ground_verts < 0 || g->verts_per_block > 4096 || n_env_static < 0)
    return dbw_fail_("dbw_scene_geometry_forward: bad sizes", cudaSuccess);
  const int n = g->n_blocks * g->verts_per_block + g->n_ground_verts;
  const int threads = n > n_env_static * 3 ? n : n_env_static * 3;
  if (threads == 0) return 0;
  scene_geometry_forward_kernel<<<(threads + 127) / 128, 128, 0, (cudaStream_t)stream>>>(make_geom(g), verts_out, env_static_verts,
                                                                                         n_env_static);
  SCENE_LAUNCH_CK("scene_geometry_forward_kernel");
  return 0;
}

extern "C" int dbw_scene_geometry_backward(const DbwSceneGeometry* g, const float* g_block_verts, const float* g_ground_verts,
                                           float* g_sq_eps, float* g_S, float* g_R_6d, float* g_T, float* g_R_6d_ground,
                                           float* g_T_ground, void* stream) {
  if (!g || (g->n_blocks > 0 && !g_block_verts) || (g->n_ground_verts > 0 && !g_ground_verts))
    return dbw_fail_("dbw_scene_geometry_backward: null pointer argument", cudaSuccess);
  const int prims = g->n_blocks + (g->n_ground_verts > 0 ? 1 : 0);
  if (prims == 0) return 0;
  scene_geometry_backward_kernel<<<prims, 64, 0, (cudaStream_t)stream>>>(make_geom(g), g_block_verts, g_ground_verts, g_sq_eps, g_S,
                                                                         g_R_6d, g_T, g_R_6d_ground, g_T_ground);
  SCENE_LAUNCH_CK("scene_geometry_backward_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ opacities
// src/model/dbw.py:300-316 with static shapes, one launch: alpha = sigmoid(logit + noise_scale * noise); blocks whose NOISE-FREE
// opacity is not above keep_threshold are disabled through the face map (-1) and zeroed in alpha_kept.
__global__ void opacity_forward_kernel(const float* __restrict__ logit, const float* __restrict__ noise, float noise_scale,
                                       float keep_threshold, const int* __restrict__ face_map_in, int n_blocks, int faces_per_block,
                                       float* __restrict__ alpha, float* __restrict__ alpha_kept, int* __restrict__ face_map_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_blocks * faces_per_block) return;
  const int k = i / faces_per_block;
  const float l = logit[k];
  const bool keep = keep_threshold < 0.f || 1.f / (1.f + expf(-l)) > keep_threshold;
  if (face_map_out) face_map_out[i] = keep ? face_map_in[i] : -1;
  if (i == k * faces_per_block) {
    const float a = 1.f / (1.f + expf(-(noise ? l + noise_scale * noise[k] : l)));
    alpha[k] = a;
    if (alpha_kept) alpha_kept[k] = keep ? a : 0.f;
  }
}

__global__ void opacity_backward_kernel(const float* __restrict__ logit, const float* __restrict__ noise, float noise_scale,
                                        float keep_threshold, const float* __restrict__ g_alpha, const float* __restrict__ g_alpha_kept,
                                        int n_blocks, float* __restrict__ g_logit) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_blocks) return;
  const float l = logit[k];
  const bool keep = keep_threshold < 0.f || 1.f / (1.f + expf(-l)) > keep_threshold;
  const float a = 1.f / (1.f + expf(-(noise ? l + noise_scale * noise[k] : l)));
  float g = g_alpha ? g_alpha[k] : 0.f;
  if (g_alpha_kept && keep) g += g_alpha_kept[k];
  g_logit[k] = g * a * (1.f - a);
}

extern "C" int dbw_opacity_forward(const float* alpha_logit, const float* noise, float noise_scale, float keep_threshold,
                                   const int32_t* face_map_in, int32_t n_blocks, int32_t faces_per_block, float* alpha,
                                   float* alpha_kept, int32_t* face_map_out, void* stream) {
  if (!alpha_logit || !alpha || (face_map_out && !face_map_in)) return dbw_fail_("dbw_opacity_forward: null pointer argument", cudaSuccess);
  if (n_blocks < 0 || faces_per_block <= 0) return dbw_fail_("dbw_opacity_forward: bad sizes", cudaSuccess);
  if (n_blocks == 0) return 0;
  const int n = n_blocks * faces_per_block;
  opacity_forward_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(alpha_logit, noise, noise_scale, keep_threshold, face_map_in,
                                                                            n_blocks, faces_per_block, alpha, alpha_kept, face_map_out);
  SCENE_LAUNCH_CK("opacity_forward_kernel");
  return 0;
}

extern "C" int dbw_opacity_backward(const float* alpha_logit, const float* noise, float noise_scale, float keep_threshold,
                                    const float* g_alpha, const float* g_alpha_kept, int32_t n_blocks, float* g_alpha_logit,
                                    void* stream) {
  if (!alpha_logit || !g_alpha_logit) return dbw_fail_("dbw_opacity_backward: null pointer argument", cudaSuccess);
  if (n_blocks <= 0) return n_blocks == 0 ? 0 : dbw_fail_("dbw_opacity_backward: bad sizes", cudaSuccess);
  opacity_backward_kernel<<<(n_blocks + 127) / 128, 128, 0, (cudaStream_t)stream>>>(alpha_logit, noise, noise_scale, keep_threshold,
                                                                                    g_alpha, g_alpha_kept, n_blocks, g_alpha_logit);
  SCENE_LAUNCH_CK("opacity_backward_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------ textures
// one thread per SOURCE texel (m, y, x); decimation cells are f x f (f = 1: none) and never straddle a warp row segment:
// with f = 8 each run of 8 lanes shares a cell column, rows are combined through shared memory.
// up to DBW_MAX_TEX_JOBS texture stacks per launch (background, ground, blocks: ONE launch each way per step instead of three,
// and the two environment maps land in one atlas without a concatenation)
struct TexJobs { DbwTexJob j[DBW_MAX_TEX_JOBS]; int n; int zoff[DBW_MAX_TEX_JOBS + 1]; };

__global__ void texture_prep_forward_kernel(const TexJobs J) {
  // block = (32, 8): 32 texels along x, 8 rows -> with f = 8 a block holds 4 complete cells
  int job = 0;
  while (job + 1 < J.n && (int)blockIdx.z >= J.zoff[job + 1]) ++job;
  const DbwTexJob& jb = J.j[job];
  const float* __restrict__ tex = jb.textures;
  float4* __restrict__ atlas = reinterpret_cast<float4*>(jb.atlas);
  const int TS = jb.txt_size, p_left = jb.p_left, p_right = jb.p_right, f = jb.decimate, stage = jb.stage;
  if ((int)blockIdx.x * 32 >= TS || (int)blockIdx.y * 8 >= TS) return;          // the grid is sized for the largest stack
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, m = blockIdx.z - J.zoff[job];
  __shared__ float s_sum[8][32][3];
  float s[3] = {0.f, 0.f, 0.f};
  const bool ok = x < TS && y < TS;
  const int CS = TS / f;                                                         // cells per side
  const size_t cell = (((size_t)m * CS + y / f) * CS + x / f) * 3;
  if (ok) {
    if (stage == DBW_TEX_STAGE_EXPAND) {                                         // `textures` holds the cell colours
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] = tex[cell + c];
    } else {
      const float* t = tex + (((size_t)m * TS + y) * TS + x) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] = 1.f / (1.f + expf(-t[c]));
    }
  }
  if (f == 8 && stage != DBW_TEX_STAGE_EXPAND) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = s[c];
      v += __shfl_xor_sync(0xffffffffu, v, 1); v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 4);
      s_sum[threadIdx.y][threadIdx.x][c] = v;          // sum over the 8 lanes of this row segment
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) v += s_sum[r][threadIdx.x][c];
      s[c] = v * (1.f / 64.f);
    }
  }
  if (!ok) return;
  if (stage == DBW_TEX_STAGE_CELLS) {                                            // `atlas` receives the (n_maps, CS, CS, 3) cell colours
    if (x % f == 0 && y % f == 0) {
      float* out = jb.atlas + cell;
      out[0] = s[0]; out[1] = s[1]; out[2] = s[2];
    }
    return;
  }
  if (stage == DBW_TEX_STAGE_CELLS4) {                                           // (n_maps, CS, CS) float4 cells
    if (x % f == 0 && y % f == 0) atlas[cell / 3] = make_float4(s[0], s[1], s[2], 0.f);
    return;
  }
  const int Wp = TS + p_left + p_right;
  float4* row = atlas + ((size_t)m * TS + y) * Wp;
  const float4 val = make_float4(s[0], s[1], s[2], 0.f);
  row[x + p_left] = val;
  if (x < p_right) row[TS + p_left + x] = val;               // circular padding on the right: columns 0..p_right-1
  if (x >= TS - p_left) row[x - (TS - p_left)] = val;        // and on the left: the last p_left columns
}

__global__ void texture_prep_backward_kernel(const TexJobs J) {
  int job = 0;
  while (job + 1 < J.n && (int)blockIdx.z >= J.zoff[job + 1]) ++job;
  const DbwTexJob& jb = J.j[job];
  const float* __restrict__ tex = jb.textures;
  const float4* __restrict__ g_atlas = reinterpret_cast<const float4*>(jb.atlas);
  float* __restrict__ g_tex = jb.g_textures;
  const int TS = jb.txt_size, p_left = jb.p_left, p_right = jb.p_right, f = jb.decimate, stage = jb.stage;
  if ((int)blockIdx.x * 32 >= TS || (int)blockIdx.y * 8 >= TS) return;
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, m = blockIdx.z - J.zoff[job];
  __shared__ float s_sum[8][32][3];
  const bool ok = x < TS && y < TS;
  const int CS = TS / f;
  const size_t cell = (((size_t)m * CS + y / f) * CS + x / f) * 3;
  float g[3] = {0.f, 0.f, 0.f};
  if (stage == DBW_TEX_STAGE_CELLS || stage == DBW_TEX_STAGE_CELLS4) {
    // `atlas` holds the CELL gradient (n_maps, CS, CS, 3 or 4), already summed over the cell's texels (and over ranks); the
    // float4 one is read a float at a time: it may be a view of a gradient bucket at any 4-byte offset
    if (ok) {
      const float* gc = jb.atlas + (stage == DBW_TEX_STAGE_CELLS4 ? cell / 3 * 4 : cell);
      const size_t o = (((size_t)m * TS + y) * TS + x) * 3;
      const float scale = f == 8 ? 1.f / 64.f : 1.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float sg = 1.f / (1.f + expf(-tex[o + c]));
        g_tex[o + c] = gc[c] * scale * sg * (1.f - sg);
      }
    }
    return;
  }
  if (ok) {
    const int Wp = TS + p_left + p_right;
    const float4* row = g_atlas + ((size_t)m * TS + y) * Wp;
    float4 a = row[x + p_left];
    g[0] = a.x; g[1] = a.y; g[2] = a.z;
    if (x < p_right) { a = row[TS + p_left + x]; g[0] += a.x; g[1] += a.y; g[2] += a.z; }
    if (x >= TS - p_left) { a = row[x - (TS - p_left)]; g[0] += a.x; g[1] += a.y; g[2] += a.z; }
  }
  if (f == 8) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = g[c];
      v += __shfl_xor_sync(0xffffffffu, v, 1); v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 4);
      s_sum[threadIdx.y][threadIdx.x][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) v += s_sum[r][threadIdx.x][c];
      g[c] = stage == DBW_TEX_STAGE_EXPAND ? v : v * (1.f / 64.f);
    }
  }
  if (!ok) return;
  if (stage == DBW_TEX_STAGE_EXPAND) {                       // `g_textures` receives the cell gradient: the sum over the cell's texels
    if (x % f == 0 && y % f == 0) { g_tex[cell] = g[0]; g_tex[cell + 1] = g[1]; g_tex[cell + 2] = g[2]; }
    return;
  }
  const size_t o = (((size_t)m * TS + y) * TS + x) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float sg = 1.f / (1.f + expf(-tex[o + c]));
    g_tex[o + c] = g[c] * sg * (1.f - sg);
  }
}

static int check_tex(const char* who, int M, int TS, int p_left, int p_right, int f) {
  if (M <= 0 || TS <= 0 || p_left < 0 || p_right < 0 || p_left > TS || p_right > TS) return dbw_fail_(who, cudaSuccess);
  if (f != 1 && f != 8) return dbw_fail_("texture prep: decimate factor must be 1 or 8", cudaSuccess);
  if (f == 8 && TS % 8 != 0) return dbw_fail_("texture prep: txt_size must be a multiple of the decimation factor", cudaSuccess);
  return 0;
}

static int launch_tex(const DbwTexJob* jobs, int n_jobs, bool backward, void* stream) {
  const char* who = backward ? "dbw_texture_prep_backward_multi" : "dbw_texture_prep_forward_multi";
  if (!jobs || n_jobs < 1 || n_jobs > DBW_MAX_TEX_JOBS) return dbw_fail_("texture prep: 1 .. DBW_MAX_TEX_JOBS jobs", cudaSuccess);
  TexJobs J;
  memset(&J, 0, sizeof(J));
  J.n = n_jobs;
  int ts_max = 0;
  for (int i = 0; i < n_jobs; ++i) {
    const DbwTexJob& j = jobs[i];
    if (!j.textures || !j.atlas || (backward && !j.g_textures)) return dbw_fail_("texture prep: null pointer argument", cudaSuccess);
    if (j.stage < 0 || j.stage > 3) return dbw_fail_("texture prep: stage must be DBW_TEX_STAGE_FUSED, _CELLS, _EXPAND or _CELLS4", cudaSuccess);
    if (j.stage == DBW_TEX_STAGE_CELLS4 && !backward && (reinterpret_cast<uintptr_t>(j.atlas) & 15))
      return dbw_fail_("texture prep: float4 cells must be 16-byte aligned", cudaSuccess);
    if (check_tex(who, j.n_maps, j.txt_size, j.p_left, j.p_right, j.decimate)) return -1;
    J.j[i] = j; J.zoff[i + 1] = J.zoff[i] + j.n_maps;
    ts_max = j.txt_size > ts_max ? j.txt_size : ts_max;
  }
  dim3 grid((ts_max + 31) / 32, (ts_max + 7) / 8, J.zoff[n_jobs]), block(32, 8);
  if (backward) texture_prep_backward_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(J);
  else texture_prep_forward_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(J);
  SCENE_LAUNCH_CK(backward ? "texture_prep_backward_kernel" : "texture_prep_forward_kernel");
  return 0;
}

extern "C" int dbw_texture_prep_forward_multi(const DbwTexJob* jobs, int32_t n_jobs, void* stream) { return launch_tex(jobs, n_jobs, false, stream); }
extern "C" int dbw_texture_prep_backward_multi(const DbwTexJob* jobs, int32_t n_jobs, void* stream) { return launch_tex(jobs, n_jobs, true, stream); }
