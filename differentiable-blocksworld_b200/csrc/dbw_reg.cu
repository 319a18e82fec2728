// dbw_reg.cu -- sm_90a regularisers of the objective: parsimony, total variation and overlap with their gradients (see
// include/dbw_render.h, "Regularisers"; the per-element math is dbw_reg_math.cuh).
//
// Forward, two launches.  reg_forward_kernel's grid is the overlap CTAs (one sample point per thread) followed by the TV CTAs
// (REG_TV_TEXELS texels per thread over background | ground | blocks, read as logits: each texel's sigmoid is taken where it
// is read, no map is materialised).  Every CTA writes one double partial; reg_forward_finish_kernel sums them in a fixed
// order, adds the parsimony mean and writes the three weighted scalars.
//
// Backward, two launches.  reg_backward_kernel: the TV CTAs write each texel's logit gradient from its four neighbours; the
// overlap CTAs recompute their points' occupancies, then for every block form the 18 sums the block's gradient needs
// (block-frame rotation and scale pieces, e1, e2, alpha) and write them per CTA.  reg_backward_finish_kernel, one CTA per
// block, sums those rows in a fixed order and applies the chain rule to the leaves (exp, rot6d_backward, the sigmoid of the
// exponents) and the parsimony derivative.  No float atomics anywhere: two runs on the same inputs give the same bits.
//
// The overlap CTAs stage the blocks' records (R, T, S * ratio, e1, e2, alpha) in shared memory REG_OV_CHUNK blocks at a time.
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_reg_math.cuh"
#include "dbw_scene_math.cuh"

static_assert(DBW_REG_TV_NORM_L2 == DBW_REG_TV_L2 && DBW_REG_TV_NORM_L1 == DBW_REG_TV_L1 && DBW_REG_TV_NORM_L2SQ == DBW_REG_TV_L2SQ,
              "TV norm codes of the C-ABI and of dbw_reg_math.cuh");

constexpr int REG_THREADS = 256;
constexpr int REG_WARPS = REG_THREADS / 32;
constexpr int REG_TV_TEXELS = 4;                 // texels per thread in the forward
constexpr int REG_OV_CHUNK = 128;                // blocks staged in shared memory at a time
constexpr int REG_REC = 18;                      // R[9] T[3] S*ratio[3] e1 e2 alpha
constexpr int REG_GRADS = 18;                    // per-block sums: g_r[3] g_Sr[3] g_R[9] g_e1 g_e2 g_alpha

// what the host derives once per call
struct RegPlan {
  DbwRegularisers r;
  int n_ov_ctas, n_tv_fwd_ctas, n_tv_bwd_ctas;
  long long n_env_texels, n_blk_texels;          // per environment map, over all block maps
  float cv_env, cu_env, cv_ground, cu_ground, cv_blk, cu_blk;      // mean denominators and phase factors folded in
};

__device__ __forceinline__ float cta_sum(float v, float* red) {   // fixed-order CTA sum, result in thread 0
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < REG_WARPS; ++w) s += red[w];
  __syncthreads();
  return s;
}

// one block's record, from the leaves
__device__ __forceinline__ void block_record(const DbwRegularisers& r, int k, float* rec) {
  rot6d(r.R_6d + 6 * k, rec);
  for (int c = 0; c < 3; ++c) {
    rec[9 + c] = r.T[3 * k + c];
    rec[12 + c] = (expf(r.S[3 * k + c]) + r.scale_min) * r.ratio_block_scene;
  }
  rec[15] = reg_sq_eps(r.sq_eps[2 * k]);
  rec[16] = reg_sq_eps(r.sq_eps[2 * k + 1]);
  rec[17] = r.alpha_full[k];
}

// sample point j in the scene frame: ((2 u - 1) * ratio * S_b) @ R_b + T_b, b = j / n_points
__device__ __forceinline__ void sample_point(const DbwRegularisers& r, long long j, float* p) {
  const int b = (int)(j / r.n_points);
  float R[9], x[3];
  rot6d(r.R_6d + 6 * b, R);
  const float* u = r.unit_samples + 3 * j;
  for (int c = 0; c < 3; ++c) x[c] = (u[c] * 2.f - 1.f) * r.ratio_block_scene * (expf(r.S[3 * b + c]) + r.scale_min);
  for (int c = 0; c < 3; ++c) p[c] = x[0] * R[c] + x[1] * R[3 + c] + x[2] * R[6 + c] + r.T[3 * b + c];
}

// p in block frame `rec`: q = p - T, r_k = sum_m q_m R[k][m], local_k = r_k / (S_k ratio)
__device__ __forceinline__ void to_block_frame(const float* rec, const float* p, float* q, float* loc) {
  for (int c = 0; c < 3; ++c) q[c] = p[c] - rec[9 + c];
  for (int k = 0; k < 3; ++k)
    loc[k] = __fdiv_rn(q[0] * rec[3 * k] + q[1] * rec[3 * k + 1] + q[2] * rec[3 * k + 2], rec[12 + k]);
}

__device__ __forceinline__ void stage_chunk(const DbwRegularisers& r, int k0, float* s_rec) {
  __syncthreads();                               // the previous chunk is no longer read
  const int n = min(REG_OV_CHUNK, r.n_blocks - k0);
  for (int k = threadIdx.x; k < n; k += REG_THREADS) block_record(r, k0 + k, s_rec + REG_REC * k);
  __syncthreads();
}

// sum_k sigmoid(-sdf_k(p) / T) alpha_k over all blocks, in block order
__device__ float occupancy(const DbwRegularisers& r, const float* p, bool valid, float* s_rec, int* staged) {
  float occ = 0.f;
  for (int k0 = 0; k0 < r.n_blocks; k0 += REG_OV_CHUNK) {
    if (*staged != k0) { stage_chunk(r, k0, s_rec); *staged = k0; }
    const int n = min(REG_OV_CHUNK, r.n_blocks - k0);
    if (valid)
      for (int k = 0; k < n; ++k) {
        const float* rec = s_rec + REG_REC * k;
        float q[3], loc[3];
        to_block_frame(rec, p, q, loc);
        const float sdf = sq_implicit(loc, rec[15], rec[16]);
        occ += reg_sigmoid(__fdiv_rn(-sdf, DBW_REG_OVERLAP_TEMPERATURE)) * rec[17];
      }
  }
  return occ;
}

__device__ __forceinline__ int tv_segment(const RegPlan& P, long long t, long long* local) {
  if (t < P.n_env_texels) { *local = t; return 0; }
  if (t < 2 * P.n_env_texels) { *local = t - P.n_env_texels; return 1; }
  *local = t - 2 * P.n_env_texels; return 2;
}

__device__ __forceinline__ void load_sig(const float* base, long long texel, float* m) {
  for (int c = 0; c < 3; ++c) m[c] = reg_sigmoid(base[3 * texel + c]);
}

__global__ void __launch_bounds__(REG_THREADS) reg_forward_kernel(RegPlan P, double* __restrict__ partials) {
  __shared__ float s_rec[REG_OV_CHUNK * REG_REC];
  __shared__ float red[REG_WARPS];
  const DbwRegularisers& r = P.r;
  float acc = 0.f;
  if ((int)blockIdx.x < P.n_ov_ctas) {
    const long long j = (long long)blockIdx.x * REG_THREADS + threadIdx.x;
    const bool valid = j < (long long)r.n_blocks * r.n_points;
    float p[3] = {0.f, 0.f, 0.f};
    if (valid) sample_point(r, j, p);
    int staged = -1;
    const float occ = occupancy(r, p, valid, s_rec, &staged);
    if (valid) acc = fmaxf(occ - DBW_REG_OVERLAP_N_BLOCKS, 0.f);
  } else {
    const long long n_tv = 2 * P.n_env_texels + P.n_blk_texels;
    const long long t0 = (long long)(blockIdx.x - P.n_ov_ctas) * REG_THREADS * REG_TV_TEXELS + threadIdx.x;
    for (int i = 0; i < REG_TV_TEXELS; ++i) {
      const long long t = t0 + (long long)i * REG_THREADS;
      if (t >= n_tv) break;
      long long lt;
      const int seg = tv_segment(P, t, &lt);
      const int S = seg < 2 ? r.env_size : r.txt_size;
      const float* base = seg == 0 ? r.texture_bkg : (seg == 1 ? r.texture_ground : r.textures);
      const float cv = seg == 0 ? P.cv_env : (seg == 1 ? P.cv_ground : P.cv_blk);
      const float cu = seg == 0 ? P.cu_env : (seg == 1 ? P.cu_ground : P.cu_blk);
      const int u = (int)(lt % S), v = (int)((lt / S) % S);
      float m[3], n[3];
      load_sig(base, lt, m);
      if (v < S - 1) {
        load_sig(base, lt + S, n);
        acc += cv * tv_norm(r.tv_norm, n[0] - m[0], n[1] - m[1], n[2] - m[2]);
      }
      if (seg == 2 || u < S - 1) {
        load_sig(base, u < S - 1 ? lt + 1 : lt - (S - 1), n);          // the blocks' maps wrap in u
        acc += cu * tv_norm(r.tv_norm, n[0] - m[0], n[1] - m[1], n[2] - m[2]);
      }
    }
  }
  const float s = cta_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = (double)s;
}

__global__ void __launch_bounds__(REG_THREADS)
reg_forward_finish_kernel(RegPlan P, const double* __restrict__ partials, float* out_parsimony, float* out_tv, float* out_overlap) {
  __shared__ double red[3][REG_THREADS];
  const DbwRegularisers& r = P.r;
  const int tid = threadIdx.x;
  double ov = 0.0, tv = 0.0, par = 0.0;
  for (int i = tid; i < P.n_ov_ctas; i += REG_THREADS) ov += partials[i];
  for (int i = tid; i < P.n_tv_fwd_ctas; i += REG_THREADS) tv += partials[P.n_ov_ctas + i];
  if (r.terms & DBW_REG_PARSIMONY)
    for (int k = tid; k < r.n_blocks; k += REG_THREADS) par += (double)parsimony_value(r.alpha_full[k]);
  red[0][tid] = par; red[1][tid] = tv; red[2][tid] = ov;
  __syncthreads();
  for (int h = REG_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h)
      for (int c = 0; c < 3; ++c) red[c][tid] += red[c][tid + h];
    __syncthreads();
  }
  if (tid == 0) {
    if (r.terms & DBW_REG_PARSIMONY) *out_parsimony = r.w_parsimony * (float)(red[0][0] / r.n_blocks);
    if (r.terms & DBW_REG_TV) *out_tv = r.w_tv * (float)red[1][0];
    if (r.terms & DBW_REG_OVERLAP) *out_overlap = r.w_overlap * (float)(red[2][0] / ((double)r.n_blocks * r.n_points));
  }
}

__global__ void __launch_bounds__(REG_THREADS)
reg_backward_kernel(RegPlan P, const float* __restrict__ g_out_tv, const float* __restrict__ g_out_overlap,
                    float* g_texture_bkg, float* g_texture_ground, float* g_textures, float* __restrict__ partials) {
  __shared__ float s_rec[REG_OV_CHUNK * REG_REC];
  __shared__ float red[REG_WARPS][REG_GRADS];
  const DbwRegularisers& r = P.r;
  if ((int)blockIdx.x < P.n_ov_ctas) {
    const long long n_pts = (long long)r.n_blocks * r.n_points;
    const long long j = (long long)blockIdx.x * REG_THREADS + threadIdx.x;
    const bool valid = j < n_pts;
    float p[3] = {0.f, 0.f, 0.f};
    if (valid) sample_point(r, j, p);
    int staged = -1;
    const float occ = occupancy(r, p, valid, s_rec, &staged);
    // mean, then clamp(min=0): the gradient passes where the excess is >= 0
    const float g_pt = (valid && occ - DBW_REG_OVERLAP_N_BLOCKS >= 0.f)
                       ? __fdiv_rn(*g_out_overlap * r.w_overlap, (float)n_pts) : 0.f;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k0 = 0; k0 < r.n_blocks; k0 += REG_OV_CHUNK) {
      if (staged != k0) { stage_chunk(r, k0, s_rec); staged = k0; }
      const int n = min(REG_OV_CHUNK, r.n_blocks - k0);
      for (int k = 0; k < n; ++k) {
        const float* rec = s_rec + REG_REC * k;
        float g[REG_GRADS];
        for (int c = 0; c < REG_GRADS; ++c) g[c] = 0.f;
        if (valid) {
          float q[3], loc[3], gl[3], ge1, ge2;
          to_block_frame(rec, p, q, loc);
          const float sdf = sq_implicit(loc, rec[15], rec[16]);
          const float sg = reg_sigmoid(__fdiv_rn(-sdf, DBW_REG_OVERLAP_TEMPERATURE));
          // occ_k = sigmoid(-sdf / T) * alpha_k
          g[17] = g_pt * sg;
          const float g_sdf = -__fdiv_rn(g_pt * rec[17] * ((1.f - sg) * sg), DBW_REG_OVERLAP_TEMPERATURE);
          sq_implicit_backward(loc, rec[15], rec[16], g_sdf, gl, &ge1, &ge2);
          g[15] = ge1; g[16] = ge2;
          for (int a = 0; a < 3; ++a) {
            const float g_r = __fdiv_rn(gl[a], rec[12 + a]);           // local = r / (S ratio)
            g[a] = g_r;
            g[3 + a] = -g_r * loc[a];
            for (int m = 0; m < 3; ++m) g[6 + 3 * a + m] = g_r * q[m];
          }
        }
        for (int c = 0; c < REG_GRADS; ++c) {
          float v = g[c];
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) red[warp][c] = v;
        }
        __syncthreads();
        if (threadIdx.x < REG_GRADS) {
          float s = 0.f;
          for (int w = 0; w < REG_WARPS; ++w) s += red[w][threadIdx.x];
          partials[((long long)blockIdx.x * r.n_blocks + k0 + k) * REG_GRADS + threadIdx.x] = s;
        }
        __syncthreads();
      }
    }
    return;
  }
  // TV: one texel per thread, its logit gradient from the differences it enters
  const long long t = (long long)(blockIdx.x - P.n_ov_ctas) * REG_THREADS + threadIdx.x;
  if (t >= 2 * P.n_env_texels + P.n_blk_texels) return;
  long long lt;
  const int seg = tv_segment(P, t, &lt);
  float* out = seg == 0 ? g_texture_bkg : (seg == 1 ? g_texture_ground : g_textures);
  if (!out) return;
  const int S = seg < 2 ? r.env_size : r.txt_size;
  const float* base = seg == 0 ? r.texture_bkg : (seg == 1 ? r.texture_ground : r.textures);
  const float g_tv = *g_out_tv * r.w_tv;
  const float cv = g_tv * (seg == 0 ? P.cv_env : (seg == 1 ? P.cv_ground : P.cv_blk));
  const float cu = g_tv * (seg == 0 ? P.cu_env : (seg == 1 ? P.cu_ground : P.cu_blk));
  const int u = (int)(lt % S), v = (int)((lt / S) % S);
  const bool wrap = seg == 2;
  float m[3], n[3], gd[3], gm[3] = {0.f, 0.f, 0.f};
  load_sig(base, lt, m);
  if (v < S - 1) {                               // d = m[v+1] - m[v]
    load_sig(base, lt + S, n);
    tv_norm_backward(r.tv_norm, n[0] - m[0], n[1] - m[1], n[2] - m[2], cv, gd);
    for (int c = 0; c < 3; ++c) gm[c] -= gd[c];
  }
  if (v > 0) {                                   // d = m[v] - m[v-1]
    load_sig(base, lt - S, n);
    tv_norm_backward(r.tv_norm, m[0] - n[0], m[1] - n[1], m[2] - n[2], cv, gd);
    for (int c = 0; c < 3; ++c) gm[c] += gd[c];
  }
  if (wrap || u < S - 1) {                       // d = m[u+1] - m[u]
    load_sig(base, u < S - 1 ? lt + 1 : lt - (S - 1), n);
    tv_norm_backward(r.tv_norm, n[0] - m[0], n[1] - m[1], n[2] - m[2], cu, gd);
    for (int c = 0; c < 3; ++c) gm[c] -= gd[c];
  }
  if (wrap || u > 0) {                           // d = m[u] - m[u-1]
    load_sig(base, u > 0 ? lt - 1 : lt + (S - 1), n);
    tv_norm_backward(r.tv_norm, m[0] - n[0], m[1] - n[1], m[2] - n[2], cu, gd);
    for (int c = 0; c < 3; ++c) gm[c] += gd[c];
  }
  for (int c = 0; c < 3; ++c) out[3 * lt + c] = gm[c] * ((1.f - m[c]) * m[c]);
}

// one CTA per block: the fixed-order sum of the overlap CTAs' rows, then the chain rule to the leaves
__global__ void __launch_bounds__(REG_THREADS)
reg_backward_finish_kernel(RegPlan P, const float* __restrict__ partials, const float* __restrict__ g_out_parsimony,
                           float* g_S, float* g_R_6d, float* g_T, float* g_sq_eps, float* g_alpha_full) {
  __shared__ double red[REG_GRADS][REG_WARPS];
  const DbwRegularisers& r = P.r;
  const int k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool ov = (r.terms & DBW_REG_OVERLAP) != 0;
  if (ov) {
    double acc[REG_GRADS];
    for (int c = 0; c < REG_GRADS; ++c) acc[c] = 0.0;
    for (int i = tid; i < P.n_ov_ctas; i += REG_THREADS) {
      const float* row = partials + ((long long)i * r.n_blocks + k) * REG_GRADS;
      for (int c = 0; c < REG_GRADS; ++c) acc[c] += (double)row[c];
    }
    for (int c = 0; c < REG_GRADS; ++c) {
      double v = acc[c];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[c][warp] = v;
    }
    __syncthreads();
  }
  if (tid != 0) return;
  float g[REG_GRADS];
  for (int c = 0; c < REG_GRADS; ++c) {
    double s = 0.0;
    if (ov)
      for (int w = 0; w < REG_WARPS; ++w) s += red[c][w];
    g[c] = (float)s;
  }
  if (g_alpha_full) {
    float ga = g[17];
    if (r.terms & DBW_REG_PARSIMONY)
      ga += __fdiv_rn(*g_out_parsimony * r.w_parsimony, (float)r.n_blocks) * parsimony_grad(r.alpha_full[k]);
    g_alpha_full[k] = ga;
  }
  if (!ov) return;
  float R[9];
  rot6d(r.R_6d + 6 * k, R);
  if (g_T)                                       // q = p - T, r_a = sum_m q_m R[a][m]
    for (int m = 0; m < 3; ++m) g_T[3 * k + m] = -(g[0] * R[m] + g[1] * R[3 + m] + g[2] * R[6 + m]);
  if (g_S)                                       // S * ratio, S = exp(S) + scale_min
    for (int a = 0; a < 3; ++a) g_S[3 * k + a] = g[3 + a] * r.ratio_block_scene * expf(r.S[3 * k + a]);
  if (g_R_6d) rot6d_backward(r.R_6d + 6 * k, g + 6, g_R_6d + 6 * k);
  if (g_sq_eps)                                  // e = sigmoid(x) * 1.8 + 0.1
    for (int c = 0; c < 2; ++c) {
      const float s = reg_sigmoid(r.sq_eps[2 * k + c]);
      g_sq_eps[2 * k + c] = g[15 + c] * 1.8f * ((1.f - s) * s);
    }
}

static int make_plan(const DbwRegularisers* r, RegPlan* P) {
  if (!r) return dbw_fail_("dbw_regularisers: null argument", cudaSuccess);
  const int terms = r->terms;
  if (terms & ~(DBW_REG_PARSIMONY | DBW_REG_TV | DBW_REG_OVERLAP)) return dbw_fail_("dbw_regularisers: unknown bits in terms", cudaSuccess);
  if (r->n_blocks < 1) return dbw_fail_("dbw_regularisers: n_blocks < 1", cudaSuccess);
  if ((terms & (DBW_REG_PARSIMONY | DBW_REG_OVERLAP)) && !r->alpha_full) return dbw_fail_("dbw_regularisers: null alpha_full", cudaSuccess);
  if (terms & DBW_REG_TV) {
    if (r->env_size < 2 || r->txt_size < 2) return dbw_fail_("dbw_regularisers: env_size and txt_size must be >= 2", cudaSuccess);
    if (r->tv_norm < DBW_REG_TV_NORM_L2 || r->tv_norm > DBW_REG_TV_NORM_L2SQ) return dbw_fail_("dbw_regularisers: bad tv_norm", cudaSuccess);
    if (!r->texture_bkg || !r->texture_ground || !r->textures) return dbw_fail_("dbw_regularisers: null texture", cudaSuccess);
  }
  if (terms & DBW_REG_OVERLAP) {
    if (r->n_points < 1) return dbw_fail_("dbw_regularisers: n_points < 1", cudaSuccess);
    if (!r->S || !r->R_6d || !r->T || !r->sq_eps || !r->unit_samples) return dbw_fail_("dbw_regularisers: null block parameter", cudaSuccess);
  }
  P->r = *r;
  const long long n_pts = (terms & DBW_REG_OVERLAP) ? (long long)r->n_blocks * r->n_points : 0;
  P->n_ov_ctas = (int)((n_pts + REG_THREADS - 1) / REG_THREADS);
  const bool tv = (terms & DBW_REG_TV) != 0;
  P->n_env_texels = tv ? (long long)r->env_size * r->env_size : 0;
  P->n_blk_texels = tv ? (long long)r->n_blocks * r->txt_size * r->txt_size : 0;
  const long long n_tv = 2 * P->n_env_texels + P->n_blk_texels;
  P->n_tv_fwd_ctas = (int)((n_tv + REG_THREADS * REG_TV_TEXELS - 1) / (REG_THREADS * REG_TV_TEXELS));
  P->n_tv_bwd_ctas = (int)((n_tv + REG_THREADS - 1) / REG_THREADS);
  const double f = r->coarse ? 1.0 : 0.1, E = r->env_size, B = r->txt_size;
  P->cv_env = (float)(f / ((E - 1) * E)); P->cu_env = (float)(f / (E * (E - 1)));
  P->cv_ground = (float)(f * f / ((E - 1) * E)); P->cu_ground = (float)(f * f / (E * (E - 1)));
  P->cv_blk = (float)(f / ((B - 1) * B)); P->cu_blk = (float)(f / (B * B));
  return 0;
}

static size_t workspace_of(const RegPlan& P) {
  const size_t fwd = (size_t)(P.n_ov_ctas + P.n_tv_fwd_ctas) * sizeof(double);
  const size_t bwd = (size_t)P.n_ov_ctas * P.r.n_blocks * REG_GRADS * sizeof(float);
  return fwd > bwd ? fwd : bwd;
}

extern "C" int dbw_regularisers_workspace_bytes(const DbwRegularisers* r, size_t* bytes) {
  RegPlan P;
  if (int rc = make_plan(r, &P)) return rc;
  if (!bytes) return dbw_fail_("dbw_regularisers_workspace_bytes: null bytes", cudaSuccess);
  *bytes = workspace_of(P);
  return 0;
}

extern "C" int dbw_regularisers_forward(const DbwRegularisers* r, float* out_parsimony, float* out_tv, float* out_overlap,
                                        void* workspace, size_t workspace_bytes, void* stream) {
  RegPlan P;
  if (int rc = make_plan(r, &P)) return rc;
  if (((r->terms & DBW_REG_PARSIMONY) && !out_parsimony) || ((r->terms & DBW_REG_TV) && !out_tv) ||
      ((r->terms & DBW_REG_OVERLAP) && !out_overlap))
    return dbw_fail_("dbw_regularisers_forward: null output of a term that is on", cudaSuccess);
  if (!workspace || workspace_bytes < workspace_of(P)) return dbw_fail_("dbw_regularisers_forward: workspace too small", cudaSuccess);
  if (r->terms == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  double* partials = (double*)workspace;
  const int grid = P.n_ov_ctas + P.n_tv_fwd_ctas;
  if (grid > 0) {
    reg_forward_kernel<<<grid, REG_THREADS, 0, s>>>(P, partials);
    dbw_count_launch_();
  }
  reg_forward_finish_kernel<<<1, REG_THREADS, 0, s>>>(P, partials, out_parsimony, out_tv, out_overlap);
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("reg_forward_kernel", e);
}

extern "C" int dbw_regularisers_backward(const DbwRegularisers* r, const float* g_out_parsimony, const float* g_out_tv,
                                         const float* g_out_overlap, float* g_texture_bkg, float* g_texture_ground, float* g_textures,
                                         float* g_S, float* g_R_6d, float* g_T, float* g_sq_eps, float* g_alpha_full, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  RegPlan P;
  if (int rc = make_plan(r, &P)) return rc;
  if (((r->terms & DBW_REG_PARSIMONY) && !g_out_parsimony) || ((r->terms & DBW_REG_TV) && !g_out_tv) ||
      ((r->terms & DBW_REG_OVERLAP) && !g_out_overlap))
    return dbw_fail_("dbw_regularisers_backward: null upstream gradient of a term that is on", cudaSuccess);
  if (!workspace || workspace_bytes < workspace_of(P)) return dbw_fail_("dbw_regularisers_backward: workspace too small", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  float* partials = (float*)workspace;
  const int grid = P.n_ov_ctas + P.n_tv_bwd_ctas;
  if (grid > 0) {
    reg_backward_kernel<<<grid, REG_THREADS, 0, s>>>(P, g_out_tv, g_out_overlap, g_texture_bkg, g_texture_ground, g_textures, partials);
    dbw_count_launch_();
  }
  if (r->terms & (DBW_REG_PARSIMONY | DBW_REG_OVERLAP)) {
    reg_backward_finish_kernel<<<r->n_blocks, REG_THREADS, 0, s>>>(P, partials, g_out_parsimony, g_S, g_R_6d, g_T, g_sq_eps, g_alpha_full);
    dbw_count_launch_();
  }
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("reg_backward_kernel", e);
}
