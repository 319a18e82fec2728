// dbw_lpips.cu -- sm_90a LPIPS (VGG16, version 0.1) perceptual term: forward value and the gradient with respect to the
// second image (see include/dbw_render.h, "LPIPS").  Serves dbw_b200/perceptual.py.
//
// Activations are NHWC fp32.  Every 3x3 convolution with 64..512 channels on both sides (12 of the 13 layers, forward and
// input-gradient) is one implicit GEMM on the tensor cores: M = B*H*W pixels, N = output channels, K = 9*C_in ordered
// (ky, kx, ci).  Operands are TF32 (round to nearest, ties away from zero, at bit 13: the weights once in
// dbw_lpips_prepare_weights, the activations as they leave shared memory), products accumulate in fp32 (mma.sync
// m16n8k8).  A CTA computes a 128 x BN tile; the A tile of a K step is one (ky, kx) tap and 32 consecutive channels of
// 128 pixels, loaded by 16-byte cp.async with zero fill for the halo and the rows past M, in a 3-stage pipeline.  Shared
// rows are 32 floats with their 16-byte chunks XOR-swizzled by (row & 7), so the fragment loads are conflict-free.  The
// input-gradient pass of a layer runs through the same kernel with the weights transposed and flipped
// (W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx]) and multiplies by [activation > 0] of the layer below in its epilogue.
//
// The first layer (3 -> 64, reads the NCHW image and applies the input scaling) and the last input-gradient (64 -> 3,
// writes NCHW with the scaling's chain factor) are small fp32 CUDA-core kernels.  The heads (channel normalisation,
// squared difference, lin-layer dropout, 1x1 lin conv, spatial mean) are one warp per pixel; their per-CTA partials are
// summed in a fixed order, so the value does not depend on scheduling.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dbw_render.h"
#include "dbw_lpips_hash.cuh"
#include "dbw_lpips_cache.cuh"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);
#define LP_LAUNCH_CK(name) do { dbw_count_launch_(); cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return dbw_fail_(name, _e); } while (0)

namespace {

// ------------------------------------------------------------------------------------------------ network shape
constexpr int LP_LAYERS = 13;
constexpr int LP_CIN[LP_LAYERS] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int LP_COUT[LP_LAYERS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int LP_LEVEL[LP_LAYERS] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4};   // resolution level (pools before it)
constexpr int LP_TAP_LAYER[5] = {1, 3, 6, 9, 12};                              // relu1_2 .. relu5_3
constexpr int LP_TAP_C[5] = {64, 128, 256, 512, 512};
constexpr int HEAD_PIX = 64;                 // pixels per head CTA (8 warps x 8)
constexpr float LP_EPS = 1e-10f;

struct Dims { int64_t B; int H[5], W[5]; };

Dims dims_of(int64_t B, int H, int W) {
  Dims d; d.B = B; d.H[0] = H; d.W[0] = W;
  for (int l = 1; l < 5; ++l) { d.H[l] = d.H[l - 1] / 2; d.W[l] = d.W[l - 1] / 2; }
  return d;
}

int64_t align64(int64_t n) { return (n + 63) & ~int64_t(63); }        // floats: 256-byte aligned regions
int64_t head_chunks(int H, int W) { return ((int64_t)H * W + HEAD_PIX - 1) / HEAD_PIX; }

// levels: bit k requests level k (relu1_2 .. relu5_3); LPIPS requests all five
constexpr int ALL_LEVELS = 31;
bool wants(int levels, int k) { return (levels >> k) & 1; }
int deepest(int levels) { int L = 0; for (int k = 0; k < 5; ++k) if (wants(levels, k)) L = k; return L; }   // 0-based

// workspace layout, in floats (the contract is stated in include/dbw_render.h): rec's activations through the deepest
// requested level (only its requested taps when no backward follows), imgs' requested taps, two scratch tensors of
// B*H*W*64 (pool outputs and the intermediates not kept in the forward, the running gradient in the backward), the head
// partials of the requested levels, then a region of `tail_floats`: LPIPS's seed the forward used and the target cache's
// miss count, or the VGG term's constants
struct Layout {
  int64_t act[LP_LAYERS], tap0[5], s0, s1, partials, tail, total;
  int64_t chunks[5], part_off[5];
};

Layout layout_of(const Dims& d, int levels, bool save, int64_t tail_floats) {
  Layout L; int64_t o = 0;
  const int last = LP_TAP_LAYER[deepest(levels)];
  for (int l = 0; l < LP_LAYERS; ++l) {
    L.act[l] = -1;
    const int lv = LP_LEVEL[l];
    if (l > last || (!save && !(LP_TAP_LAYER[lv] == l && wants(levels, lv)))) continue;
    L.act[l] = o; o += align64(d.B * d.H[lv] * d.W[lv] * LP_COUT[l]);
  }
  for (int k = 0; k < 5; ++k) {
    L.tap0[k] = -1;
    if (wants(levels, k)) { L.tap0[k] = o; o += align64(d.B * d.H[k] * d.W[k] * LP_TAP_C[k]); }
  }
  const int64_t big = align64(d.B * d.H[0] * d.W[0] * 64);
  L.s0 = o; o += big;
  L.s1 = o; o += big;
  L.partials = o;
  int64_t p = 0;
  for (int k = 0; k < 5; ++k) {
    L.chunks[k] = wants(levels, k) ? head_chunks(d.H[k], d.W[k]) : 0;
    L.part_off[k] = p; p += d.B * L.chunks[k];
  }
  o += align64(p);
  L.tail = o; o += align64(tail_floats);
  L.total = o;
  return L;
}

// prepared weights, in floats: per layer 1..12 the forward copy [co][ky][kx][ci] then the input-gradient copy
// [ci][ky][kx][co], both TF32-rounded
int64_t wfwd_off(int l) { int64_t o = 0; for (int i = 1; i < l; ++i) o += 2 * (int64_t)9 * LP_CIN[i] * LP_COUT[i]; return o; }
int64_t wbwd_off(int l) { return wfwd_off(l) + (int64_t)9 * LP_CIN[l] * LP_COUT[l]; }
int64_t wprep_total() { return wfwd_off(LP_LAYERS); }

// ------------------------------------------------------------------------------------------------ TF32 rounding
// round to nearest, ties away from zero, at bit 13 (cvt.rna.tf32.f32 on finite values); the low 13 bits are cleared
__device__ __forceinline__ uint32_t tf32_rna(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }

// ------------------------------------------------------------------------------------------------ implicit-GEMM conv
constexpr int CV_BM = 128, CV_BK = 32, CV_STAGES = 3, CV_THREADS = 256;

template <int BN>
struct CvCfg {
  static constexpr int WARPS_N = BN == 128 ? 4 : 2;
  static constexpr int WARPS_M = 8 / WARPS_N;
  static constexpr int WM = CV_BM / WARPS_M, WN = BN / WARPS_N;
  static constexpr int MT = WM / 16, NT = WN / 8;
  static constexpr int A_FLOATS = CV_BM * CV_BK, B_FLOATS = BN * CV_BK;
  static constexpr int SMEM = CV_STAGES * (A_FLOATS + B_FLOATS) * 4;
};

__device__ __forceinline__ int swz(int r, int c) { return r * CV_BK + ((c ^ (r & 7)) << 2); }

__device__ __forceinline__ void cp_async16(float* s, const float* g, int src_bytes) {
  const uint32_t sa = (uint32_t)__cvta_generic_to_shared(s);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(g), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// out[m][n] = epilogue(sum_k A[m][k] wt[n][k]),  A[m][(ky*3+kx)*Cin + ci] = in[pixel m shifted by (ky-1, kx-1)][ci] (0 off
// the image); epilogue: + bias[n], ReLU, * [mask[m][n] > 0], each when requested.  M = B*H*W, Cin % 32 == 0, Cout % BN == 0.
// BOUNDED (the target cache's miss chain): only the first *count images are computed, M = min(M, *count H W); the CTAs
// past them exit at once.  An output row depends on its own image and the weights only, in a K order fixed by Cin, and the
// tile shape by Cout alone, so a row gives the same bits at any position in any batch.
template <int BN, bool BOUNDED>
__global__ void __launch_bounds__(CV_THREADS, 2) lpips_conv3x3_kernel(const float* __restrict__ in, const float* __restrict__ wt,
                                                                      const float* __restrict__ bias, const float* __restrict__ mask,
                                                                      float* __restrict__ out, int M, int H, int W, int Cin,
                                                                      int Cout, int relu, const int* __restrict__ count) {
  using C = CvCfg<BN>;
  if constexpr (BOUNDED) {
    M = min(M, *count * H * W);
    if ((int)blockIdx.x * CV_BM >= M) return;
  }
  extern __shared__ __align__(16) float smem[];
  float* sA = smem;
  float* sB = smem + CV_STAGES * C::A_FLOATS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / C::WARPS_N, wn = warp % C::WARPS_N, g = lane >> 2, t = lane & 3;
  const int m0 = blockIdx.x * CV_BM, n0 = blockIdx.y * BN;
  const int K = 9 * Cin, KT = K / CV_BK, cpt = Cin / CV_BK;
  const int chunk = tid & 7, row0 = tid >> 3;
  constexpr int AR = CV_BM / 32, BR = BN / 32;

  int ay[AR], ax[AR], am[AR];
#pragma unroll
  for (int i = 0; i < AR; ++i) {
    const int m = m0 + row0 + 32 * i;
    am[i] = m;
    if (m < M) {
      const int rem = m % (H * W);
      ay[i] = rem / W; ax[i] = rem - (rem / W) * W;
    } else {
      ay[i] = -4; ax[i] = -4;                          // fails the bounds test for every tap: zero rows
    }
  }

  auto load = [&](int kt, int slot) {
    const int tap = kt / cpt, ci = (kt - tap * cpt) * CV_BK + chunk * 4;
    const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
    float* a = sA + slot * C::A_FLOATS;
#pragma unroll
    for (int i = 0; i < AR; ++i) {
      const int y = ay[i] + dy, x = ax[i] + dx;
      const bool ok = (unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W;
      const float* src = ok ? in + (int64_t)(am[i] + dy * W + dx) * Cin + ci : in;
      cp_async16(a + swz(row0 + 32 * i, chunk), src, ok ? 16 : 0);
    }
    float* b = sB + slot * C::B_FLOATS;
#pragma unroll
    for (int i = 0; i < BR; ++i)
      cp_async16(b + swz(row0 + 32 * i, chunk), wt + (int64_t)(n0 + row0 + 32 * i) * K + kt * CV_BK + chunk * 4, 16);
  };

  float acc[C::MT][C::NT][4];
#pragma unroll
  for (int i = 0; i < C::MT; ++i)
#pragma unroll
    for (int j = 0; j < C::NT; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

#pragma unroll
  for (int s = 0; s < CV_STAGES - 1; ++s) {
    if (s < KT) load(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<CV_STAGES - 2>();
    __syncthreads();
    if (kt + CV_STAGES - 1 < KT) load(kt + CV_STAGES - 1, (kt + CV_STAGES - 1) % CV_STAGES);
    cp_async_commit();
    const float* a = sA + (kt % CV_STAGES) * C::A_FLOATS;
    const float* b = sB + (kt % CV_STAGES) * C::B_FLOATS;
#pragma unroll
    for (int ks = 0; ks < CV_BK / 8; ++ks) {
      uint32_t af[C::MT][4], bf[C::NT][2];
#pragma unroll
      for (int mt = 0; mt < C::MT; ++mt) {
        const int r = wm * C::WM + mt * 16 + g;
        af[mt][0] = tf32_rna(a[swz(r, 2 * ks) + t]);
        af[mt][1] = tf32_rna(a[swz(r + 8, 2 * ks) + t]);
        af[mt][2] = tf32_rna(a[swz(r, 2 * ks + 1) + t]);
        af[mt][3] = tf32_rna(a[swz(r + 8, 2 * ks + 1) + t]);
      }
#pragma unroll
      for (int nt = 0; nt < C::NT; ++nt) {
        const int n = wn * C::WN + nt * 8 + g;
        bf[nt][0] = __float_as_uint(b[swz(n, 2 * ks) + t]);
        bf[nt][1] = __float_as_uint(b[swz(n, 2 * ks + 1) + t]);
      }
#pragma unroll
      for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < C::NT; ++nt) mma_tf32(acc[mt][nt], af[mt], bf[nt]);
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm * C::WM + mt * 16 + g + 8 * h;
      if (m >= M) continue;
#pragma unroll
      for (int nt = 0; nt < C::NT; ++nt) {
        const int n = n0 + wn * C::WN + nt * 8 + 2 * t;
        float2 v = make_float2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
        if (bias) { v.x += bias[n]; v.y += bias[n + 1]; }
        if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
        const int64_t o = (int64_t)m * Cout + n;
        if (mask) {
          const float2 k = *reinterpret_cast<const float2*>(mask + o);
          v.x = k.x > 0.f ? v.x : 0.f; v.y = k.y > 0.f ? v.y : 0.f;
        }
        *reinterpret_cast<float2*>(out + o) = v;
      }
    }
}

// ------------------------------------------------------------------------------------------------ first layer (3 -> 64)
// 4 threads per pixel, 16 output channels each; fp32 FMA.  x' = normalize ? 2x - 1 : x, then (x' - shift) / scale; the
// zero padding is of the scaled image.  GATHER (the target cache's miss chain): output image s < *count reads image
// route[s][1] of x
template <bool GATHER>
__global__ void __launch_bounds__(256) lpips_conv_first_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, const float* __restrict__ shift,
                                                               const float* __restrict__ scale, int normalize,
                                                               float* __restrict__ out, int64_t M, int H, int W,
                                                               const int32_t* __restrict__ route, const int* __restrict__ count) {
  __shared__ float ws[27][64];       // [(ci*3+ky)*3+kx][co]
  __shared__ float bs[64];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) ws[i % 27][i / 27] = w[i];
  if (threadIdx.x < 64) bs[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if constexpr (GATHER) M = min(M, (int64_t)*count * H * W);
  if (q >= 4 * M) return;
  const int64_t m = q >> 2;
  const int cg = (int)(q & 3) * 16;
  const int64_t HW = (int64_t)H * W, b = m / HW;
  const int64_t bx = GATHER ? (int64_t)route[2 * b + 1] : b;
  const int rem = (int)(m - b * HW), y = rem / W, xx = rem - (rem / W) * W;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = bs[cg + j];
  for (int ci = 0; ci < 3; ++ci) {
    const float sh = shift[ci], sc = scale[ci];
    const float* plane = x + (bx * 3 + ci) * HW;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int yy = y + ky - 1, xs = xx + kx - 1;
        float v = 0.f;
        if ((unsigned)yy < (unsigned)H && (unsigned)xs < (unsigned)W) {
          float p = plane[(int64_t)yy * W + xs];
          if (normalize) p = __fsub_rn(__fmul_rn(2.f, p), 1.f);
          v = __fdiv_rn(__fsub_rn(p, sh), sc);
        }
        const float* wr = ws[(ci * 3 + ky) * 3 + kx] + cg;
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = fmaf(v, wr[j], acc[j]);
      }
  }
  float4* o = reinterpret_cast<float4*>(out + m * 64 + cg);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    o[j] = make_float4(fmaxf(acc[4 * j], 0.f), fmaxf(acc[4 * j + 1], 0.f), fmaxf(acc[4 * j + 2], 0.f), fmaxf(acc[4 * j + 3], 0.f));
}

// ------------------------------------------------------------------------------------------------ last input-gradient (64 -> 3)
// one thread per pixel: d x'[c] = sum_{co,ky,kx} W[co][c][ky][kx] g[pixel - (ky-1, kx-1)][co], then the chain of the
// scaling (and of 2x - 1): out (NCHW) = d x' * (normalize ? 2 : 1) / scale[c]
__global__ void __launch_bounds__(256) lpips_dgrad_last_kernel(const float* __restrict__ gz, const float* __restrict__ w,
                                                               const float* __restrict__ scale, int normalize,
                                                               float* __restrict__ out, int64_t M, int H, int W) {
  __shared__ float4 ws[9][64];       // [ky*3+kx][co] = (W[co][0..2][ky][kx], 0)
  for (int i = threadIdx.x; i < 9 * 64; i += blockDim.x) {
    const int tap = i / 64, co = i % 64;
    ws[tap][co] = make_float4(w[(co * 3 + 0) * 9 + tap], w[(co * 3 + 1) * 9 + tap], w[(co * 3 + 2) * 9 + tap], 0.f);
  }
  __syncthreads();
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int64_t HW = (int64_t)H * W, b = m / HW;
  const int rem = (int)(m - b * HW), y = rem / W, x = rem - (rem / W) * W;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int yy = y - ky + 1, xs = x - kx + 1;
      if ((unsigned)yy >= (unsigned)H || (unsigned)xs >= (unsigned)W) continue;
      const float4* gp = reinterpret_cast<const float4*>(gz + (b * HW + (int64_t)yy * W + xs) * 64);
      const float4* wr = ws[ky * 3 + kx];
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 gv = gp[c4];
        const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 wv = wr[4 * c4 + j];
          a0 = fmaf(gg[j], wv.x, a0); a1 = fmaf(gg[j], wv.y, a1); a2 = fmaf(gg[j], wv.z, a2);
        }
      }
    }
  const float f = normalize ? 2.f : 1.f;
  const float a[3] = {a0, a1, a2};
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(b * 3 + c) * HW + rem] = __fdiv_rn(__fmul_rn(a[c], f), scale[c]);
}

// ------------------------------------------------------------------------------------------------ max-pool 2x2, stride 2, floor
// BOUNDED: only the first *count images
template <bool BOUNDED>
__global__ void lpips_pool_kernel(const float4* __restrict__ in, float4* __restrict__ out, int64_t n_out, int H, int W, int C4,
                                  const int* __restrict__ count) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int OH = H / 2, OW = W / 2;
  if constexpr (BOUNDED) n_out = min(n_out, (int64_t)*count * OH * OW * C4);
  if (i >= n_out) return;
  const int c = (int)(i % C4);
  const int64_t p = i / C4;
  const int ox = (int)(p % OW), oy = (int)((p / OW) % OH);
  const int64_t b = p / ((int64_t)OW * OH);
  const float4* r = in + ((b * H + 2 * oy) * W + 2 * ox) * C4 + c;
  const float4 v0 = r[0], v1 = r[C4], v2 = r[(int64_t)W * C4], v3 = r[(int64_t)W * C4 + C4];
  out[i] = make_float4(fmaxf(fmaxf(v0.x, v1.x), fmaxf(v2.x, v3.x)), fmaxf(fmaxf(v0.y, v1.y), fmaxf(v2.y, v3.y)),
                       fmaxf(fmaxf(v0.z, v1.z), fmaxf(v2.z, v3.z)), fmaxf(fmaxf(v0.w, v1.w), fmaxf(v2.w, v3.w)));
}

// one thread per input element: the gradient of its window goes to the window's first maximum in (0,0), (0,1), (1,0),
// (1,1) order (as torch's max_pool2d); rows and columns the floor drops get 0
__device__ __forceinline__ float pool_pick(float v0, float v1, float v2, float v3, int k, float gv) {
  int a = 0; float best = v0;
  if (v1 > best) { a = 1; best = v1; }
  if (v2 > best) { a = 2; best = v2; }
  if (v3 > best) { a = 3; }
  return a == k ? gv : 0.f;
}

__global__ void lpips_pool_backward_kernel(const float4* __restrict__ in, const float4* __restrict__ gout, float4* __restrict__ gin,
                                           int64_t n_in, int H, int W, int C4) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_in) return;
  const int OH = H / 2, OW = W / 2;
  const int c = (int)(i % C4);
  const int64_t p = i / C4;
  const int x = (int)(p % W), y = (int)((p / W) % H);
  const int64_t b = p / ((int64_t)W * H);
  if (y >= 2 * OH || x >= 2 * OW) { gin[i] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
  const int oy = y >> 1, ox = x >> 1, k = (y & 1) * 2 + (x & 1);
  const float4* r = in + ((b * H + 2 * oy) * W + 2 * ox) * C4 + c;
  const float4 v0 = r[0], v1 = r[C4], v2 = r[(int64_t)W * C4], v3 = r[(int64_t)W * C4 + C4];
  const float4 gv = gout[((b * OH + oy) * OW + ox) * C4 + c];
  gin[i] = make_float4(pool_pick(v0.x, v1.x, v2.x, v3.x, k, gv.x), pool_pick(v0.y, v1.y, v2.y, v3.y, k, gv.y),
                       pool_pick(v0.z, v1.z, v2.z, v3.z, k, gv.z), pool_pick(v0.w, v1.w, v2.w, v3.w, k, gv.w));
}

// ------------------------------------------------------------------------------------------------ heads
__device__ __forceinline__ float warp_sum0(float v) {      // lane 0's tree sum, broadcast (every lane sees the same bits)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}

// ROUTED (the target cache): image b's f0 is entry route[b][0] of cache_f0 for a hit (>= 0), else miss slot
// -(route[b][0] + 1) of f0.  The dropout stays keyed on b.
template <int C>
__device__ __forceinline__ const float* routed_f0(const float* f0, const float* cache_f0, const int32_t* route, int b, int HW) {
  const int r = route[2 * b];
  return r >= 0 ? cache_f0 + (int64_t)r * HW * C : f0 + (int64_t)(-r - 1) * HW * C;
}

template <int C, bool ROUTED>
__global__ void __launch_bounds__(256) lpips_head_forward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                 const float* __restrict__ lin, int HW, int W, int tap, int train,
                                                                 const uint32_t* __restrict__ seed, float* __restrict__ partials,
                                                                 int n_chunks, const int32_t* __restrict__ route,
                                                                 const float* __restrict__ cache_f0) {
  constexpr int NPL = C / 32;
  __shared__ float wsum[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  float wl[NPL];
#pragma unroll
  for (int j = 0; j < NPL; ++j) wl[j] = lin[lane + 32 * j];
  const uint32_t himg = train ? dbw_lpips_hash_image(*seed, (uint32_t)tap, (uint32_t)b) : 0u;
  const float* f0b = ROUTED ? routed_f0<C>(f0, cache_f0, route, b, HW) : f0;
  float acc = 0.f;
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C, base0 = ROUTED ? (int64_t)p * C : base;
    float u0[NPL], u1[NPL], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      u0[j] = f0b[base0 + lane + 32 * j]; u1[j] = f1[base + lane + 32 * j];
      s0 = fmaf(u0[j], u0[j], s0); s1 = fmaf(u1[j], u1[j], s1);
    }
    const float d0 = __fsqrt_rn(warp_sum0(s0)) + LP_EPS, d1 = __fsqrt_rn(warp_sum0(s1)) + LP_EPS;
    const uint32_t yx = ((uint32_t)(p / W) << 16) | (uint32_t)(p % W);
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      const float e = __fdiv_rn(u0[j], d0) - __fdiv_rn(u1[j], d1);
      float wm = wl[j];
      if (train) wm = dbw_lpips_keep(himg, (uint32_t)(lane + 32 * j), yx) ? 2.f * wm : 0.f;
      v = fmaf(wm, e * e, v);
    }
    acc += warp_sum0(v);
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += wsum[w];
    partials[(int64_t)b * n_chunks + blockIdx.x] = s;
  }
}

// g <- (d value / d f1 + (accumulate ? g : 0)) * [f1 > 0]; d value / d f1 is scaled by grad_value[b] / HW
template <int C, bool ROUTED>
__global__ void __launch_bounds__(256) lpips_head_backward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                  const float* __restrict__ lin, int HW, int W, int tap, int train,
                                                                  const uint32_t* __restrict__ seed,
                                                                  const float* __restrict__ grad_value, int accumulate,
                                                                  float* __restrict__ g, const int32_t* __restrict__ route,
                                                                  const float* __restrict__ cache_f0) {
  constexpr int NPL = C / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  const float gs = __fdiv_rn(grad_value[b], (float)HW);
  float wl[NPL];
#pragma unroll
  for (int j = 0; j < NPL; ++j) wl[j] = lin[lane + 32 * j] * gs;
  const uint32_t himg = train ? dbw_lpips_hash_image(*seed, (uint32_t)tap, (uint32_t)b) : 0u;
  const float* f0b = ROUTED ? routed_f0<C>(f0, cache_f0, route, b, HW) : f0;
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C, base0 = ROUTED ? (int64_t)p * C : base;
    float u0[NPL], u1[NPL], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      u0[j] = f0b[base0 + lane + 32 * j]; u1[j] = f1[base + lane + 32 * j];
      s0 = fmaf(u0[j], u0[j], s0); s1 = fmaf(u1[j], u1[j], s1);
    }
    const float r1 = __fsqrt_rn(warp_sum0(s1));
    const float d0 = __fsqrt_rn(warp_sum0(s0)) + LP_EPS, d1 = r1 + LP_EPS;
    const uint32_t yx = ((uint32_t)(p / W) << 16) | (uint32_t)(p % W);
    float q[NPL], dot = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      const float e = __fdiv_rn(u0[j], d0) - __fdiv_rn(u1[j], d1);
      float wm = wl[j];
      if (train) wm = dbw_lpips_keep(himg, (uint32_t)(lane + 32 * j), yx) ? 2.f * wm : 0.f;
      q[j] = -2.f * wm * e;                                    // d value / d n1
      dot = fmaf(q[j], u1[j], dot);
    }
    dot = warp_sum0(dot);
    const float k = r1 > 0.f ? __fdiv_rn(dot, d1 * d1 * r1) : 0.f;   // an all-zero feature: only the 1/d1 term
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      float v = __fdiv_rn(q[j], d1) - u1[j] * k;
      const int64_t o = base + lane + 32 * j;
      if (accumulate) v += g[o];
      g[o] = u1[j] > 0.f ? v : 0.f;
    }
  }
}

// value[b] = sum over the requested levels k, in order, of (sum of the level's partials, in chunk order) / (H_k W_k); the
// levels not requested have no chunks.  Then, with a seed (LPIPS), the seed is saved for the backward and advanced.
struct PartDesc { int64_t off[5], chunks[5]; float inv_hw[5]; };

__global__ void lpips_reduce_kernel(const float* __restrict__ partials, PartDesc pd, int B, float* __restrict__ value,
                                    uint32_t* __restrict__ seed, uint32_t* __restrict__ seed_used) {
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float v = 0.f;
    for (int k = 0; k < 5; ++k) {
      if (pd.chunks[k] == 0) continue;
      const float* p = partials + pd.off[k] + (int64_t)b * pd.chunks[k];
      float s = 0.f;
      for (int64_t c = 0; c < pd.chunks[k]; ++c) s += p[c];
      v += s * pd.inv_hw[k];
    }
    value[b] = v;
  }
  if (seed && threadIdx.x == 0) { *seed_used = *seed; *seed = *seed + 1u; }
}

__global__ void lpips_prepare_kernel(const float* __restrict__ w, float* __restrict__ fwd, float* __restrict__ bwd, int Cin, int Cout) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)Cout * Cin * 9) return;
  const int tap = (int)(i % 9), ci = (int)((i / 9) % Cin), co = (int)(i / (9 * (int64_t)Cin));
  const float v = __uint_as_float(tf32_rna(w[i]));
  fwd[((int64_t)co * 9 + tap) * Cin + ci] = v;
  bwd[((int64_t)ci * 9 + (8 - tap)) * Cout + co] = v;           // (2-ky)*3 + (2-kx) = 8 - tap
}

// ------------------------------------------------------------------------------------------------ VGG feature loss
// the constants of a dbw_vgg_loss_forward, written by it into the workspace: the head weight of each level (the first C_k
// of 512 floats: 1 with sum_channels, else 1 / C_k, exact for C_k = 64..512), then the identity input transform (shift
// 0, scale 1, 4 floats each)
constexpr int VGG_CONSTS = 5 * 512 + 8;

__global__ void vgg_consts_kernel(float* __restrict__ c, int sum_channels) {
  for (int i = threadIdx.x; i < VGG_CONSTS; i += blockDim.x) {
    const int k = i / 512;
    float v;
    if (k < 5) v = sum_channels ? 1.f : __fdiv_rn(1.f, (float)(k < 3 ? 64 << k : 512));
    else v = i < 5 * 512 + 4 ? 0.f : 1.f;
    c[i] = v;
  }
}

// the un-normalised head: per pixel w * sum_c (f0 - f1)^2, one warp per pixel; partials as lpips_head_forward_kernel
// writes them
template <int C>
__global__ void __launch_bounds__(256) vgg_head_plain_forward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                     float w, int HW, float* __restrict__ partials, int n_chunks) {
  constexpr int NPL = C / 32;
  __shared__ float wsum[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  float acc = 0.f;
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C;
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      const float e = f0[base + lane + 32 * j] - f1[base + lane + 32 * j];
      v = fmaf(w, e * e, v);
    }
    acc += warp_sum0(v);
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += wsum[w8];
    partials[(int64_t)b * n_chunks + blockIdx.x] = s;
  }
}

// g <- (d value / d f1 + (accumulate ? g : 0)) * [f1 > 0]; d value / d f1 = 2 w (f1 - f0) grad_value[b] / HW
template <int C>
__global__ void __launch_bounds__(256) vgg_head_plain_backward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                      float w, int HW, const float* __restrict__ grad_value,
                                                                      int accumulate, float* __restrict__ g) {
  constexpr int NPL = C / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  const float k = 2.f * w * __fdiv_rn(grad_value[b], (float)HW);
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      const int64_t o = base + lane + 32 * j;
      const float u1 = f1[o];
      float v = k * (u1 - f0[o]);
      if (accumulate) v += g[o];
      g[o] = u1 > 0.f ? v : 0.f;
    }
  }
}

// g *= [act > 0]: the ReLU of a tap whose level is not requested, between its pool's backward and its input gradient
__global__ void vgg_relu_mask_kernel(const float4* __restrict__ act, float4* __restrict__ g, int64_t n4) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 a = act[i];
  float4 v = g[i];
  v.x = a.x > 0.f ? v.x : 0.f; v.y = a.y > 0.f ? v.y : 0.f; v.z = a.z > 0.f ? v.z : 0.f; v.w = a.w > 0.f ? v.w : 0.f;
  g[i] = v;
}

// ------------------------------------------------------------------------------------------------ target cache
constexpr int FP_CHUNKS = 32;                // fingerprint partials per image
constexpr int LOOKUP_THREADS = 512;

// part[b][blockIdx.x] = this CTA's share of the fingerprint of image b (n floats each) of x
__global__ void __launch_bounds__(256) lpips_fingerprint_kernel(const float* __restrict__ x, int64_t n, uint64_t* __restrict__ part) {
  __shared__ uint64_t wsum[8];
  const int64_t b = blockIdx.y;
  const uint32_t* u = reinterpret_cast<const uint32_t*>(x) + b * n;
  uint64_t s = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += dbw_lpips_fp_term((uint64_t)i, u[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t t = 0;
    for (int w = 0; w < 8; ++w) t += wsum[w];
    part[b * FP_CHUNKS + blockIdx.x] = t;
  }
}

__global__ void lpips_fingerprint_sum_kernel(const uint64_t* __restrict__ part, int64_t N, uint64_t* __restrict__ fp) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= N) return;
  uint64_t t = 0;
  for (int c = 0; c < FP_CHUNKS; ++c) t += part[e * FP_CHUNKS + c];
  fp[e] = t;
}

// one CTA per image b of x: route[b][1] = the first cache entry whose fingerprint matches and whose stored image is the same
// bit for bit, or -1
__global__ void __launch_bounds__(LOOKUP_THREADS) lpips_lookup_kernel(const float* __restrict__ x, int64_t n,
                                                                      const uint64_t* __restrict__ part,
                                                                      const uint64_t* __restrict__ cache_fp,
                                                                      const float* __restrict__ cache_img, int64_t N,
                                                                      int32_t* __restrict__ route) {
  __shared__ uint64_t fp;
  const int64_t b = blockIdx.x;
  if (threadIdx.x == 0) {
    uint64_t t = 0;
    for (int c = 0; c < FP_CHUNKS; ++c) t += part[b * FP_CHUNKS + c];
    fp = t;
  }
  __syncthreads();
  const uint32_t* u = reinterpret_cast<const uint32_t*>(x) + b * n;
  auto same_image = [&](int64_t e) {
    const uint32_t* v = reinterpret_cast<const uint32_t*>(cache_img) + e * n;
    int diff = 0;
    for (int64_t i = threadIdx.x; i < n && !diff; i += blockDim.x) diff = u[i] != v[i];
    return !__syncthreads_or(diff);
  };
  const int hit = dbw_lpips_find(fp, cache_fp, N, same_image);
  if (threadIdx.x == 0) route[2 * b + 1] = hit;
}

__global__ void lpips_route_kernel(int32_t* __restrict__ route, int64_t B, int* __restrict__ n_miss, int32_t* __restrict__ n_hits) {
  if (threadIdx.x != 0) return;
  const int m = dbw_lpips_route(route, B);
  *n_miss = m;
  if (n_hits) *n_hits = (int32_t)(B - m);
}

// the arena, in floats: tap[k] (N, H_k W_k, C_k) for k = 0..4, the N uint64 fingerprints, the N images (N, 3, H, W).  Every
// tap holds a multiple of 64 floats per image, so an arena of N images is N times the bytes of one.
struct CacheLayout { int64_t tap[5], fp, img, total; };

CacheLayout cache_layout_of(int64_t N, int H, int W) {
  const Dims d = dims_of(1, H, W);
  CacheLayout C; int64_t o = 0;
  for (int k = 0; k < 5; ++k) { C.tap[k] = o; o += N * d.H[k] * d.W[k] * LP_TAP_C[k]; }
  C.fp = o; o += 2 * N;
  C.img = o; o += N * 3 * (int64_t)H * W;
  C.total = o;
  return C;
}

// ------------------------------------------------------------------------------------------------ launchers
// the dynamic shared-memory limit is a per-device attribute: set before every launch (cheap), as the raster kernels do
template <bool BOUNDED>
int set_attrs() {
  cudaError_t e = cudaFuncSetAttribute(lpips_conv3x3_kernel<128, BOUNDED>, cudaFuncAttributeMaxDynamicSharedMemorySize, CvCfg<128>::SMEM);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(lpips_conv3x3_kernel<64, BOUNDED>, cudaFuncAttributeMaxDynamicSharedMemorySize, CvCfg<64>::SMEM);
  if (e != cudaSuccess) return dbw_fail_("lpips: cudaFuncSetAttribute", e);
  return 0;
}

// count: NULL, or the device count of images to compute (the grid still covers B)
template <bool BOUNDED>
int conv3x3_launch(const float* in, const float* wt, const float* bias, const float* mask, float* out, int64_t B, int H, int W, int Cin,
                   int Cout, int relu, const int* count, cudaStream_t st) {
  if (const int rc = set_attrs<BOUNDED>()) return rc;
  const int64_t M = B * H * W;
  if (M == 0) return 0;
  if (Cout == 64) {
    const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)(Cout / 64));
    lpips_conv3x3_kernel<64, BOUNDED><<<grid, CV_THREADS, CvCfg<64>::SMEM, st>>>(in, wt, bias, mask, out, (int)M, H, W, Cin, Cout, relu,
                                                                                 count);
  } else {
    const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)(Cout / 128));
    lpips_conv3x3_kernel<128, BOUNDED><<<grid, CV_THREADS, CvCfg<128>::SMEM, st>>>(in, wt, bias, mask, out, (int)M, H, W, Cin, Cout,
                                                                                   relu, count);
  }
  LP_LAUNCH_CK("lpips_conv3x3_kernel");
  return 0;
}

int conv3x3(const float* in, const float* wt, const float* bias, const float* mask, float* out, int64_t B, int H, int W, int Cin,
            int Cout, int relu, cudaStream_t st, const int* count = nullptr) {
  return count ? conv3x3_launch<true>(in, wt, bias, mask, out, B, H, W, Cin, Cout, relu, count, st)
               : conv3x3_launch<false>(in, wt, bias, mask, out, B, H, W, Cin, Cout, relu, nullptr, st);
}

// route, count: NULL, or the miss chain's gather (output image s < *count reads image route[s][1] of x)
int conv_first(const float* x, const float* w, const float* bias, const float* shift, const float* scale, int normalize, float* out,
               int64_t B, int H, int W, cudaStream_t st, const int32_t* route = nullptr, const int* count = nullptr) {
  const int64_t M = B * H * W;
  const unsigned grid = (unsigned)((4 * M + 255) / 256);
  if (count)
    lpips_conv_first_kernel<true><<<grid, 256, 0, st>>>(x, w, bias, shift, scale, normalize, out, M, H, W, route, count);
  else
    lpips_conv_first_kernel<false><<<grid, 256, 0, st>>>(x, w, bias, shift, scale, normalize, out, M, H, W, nullptr, nullptr);
  LP_LAUNCH_CK("lpips_conv_first_kernel");
  return 0;
}

int dgrad_last(const float* gz, const float* w, const float* scale, int normalize, float* out, int64_t B, int H, int W,
               cudaStream_t st) {
  const int64_t M = B * H * W;
  lpips_dgrad_last_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(gz, w, scale, normalize, out, M, H, W);
  LP_LAUNCH_CK("lpips_dgrad_last_kernel");
  return 0;
}

int pool(const float* in, float* out, int64_t B, int H, int W, int C, cudaStream_t st, const int* count = nullptr) {
  const int64_t n = B * (H / 2) * (W / 2) * (C / 4);
  if (n == 0) return 0;
  const unsigned grid = (unsigned)((n + 255) / 256);
  if (count)
    lpips_pool_kernel<true><<<grid, 256, 0, st>>>((const float4*)in, (float4*)out, n, H, W, C / 4, count);
  else
    lpips_pool_kernel<false><<<grid, 256, 0, st>>>((const float4*)in, (float4*)out, n, H, W, C / 4, nullptr);
  LP_LAUNCH_CK("lpips_pool_kernel");
  return 0;
}

int pool_backward(const float* in, const float* gout, float* gin, int64_t B, int H, int W, int C, cudaStream_t st) {
  const int64_t n = B * H * W * (C / 4);
  if (n == 0) return 0;
  lpips_pool_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float4*)in, (const float4*)gout, (float4*)gin, n,
                                                                          H, W, C / 4);
  LP_LAUNCH_CK("lpips_pool_backward_kernel");
  return 0;
}

template <int C>
void head_forward_c(dim3 grid, const float* f0, const float* f1, const float* lin, int HW, int W, int tap, int train,
                    const uint32_t* seed, float* part, int n, const int32_t* route, const float* cache_f0, cudaStream_t st) {
  if (route)
    lpips_head_forward_kernel<C, true><<<grid, 256, 0, st>>>(f0, f1, lin, HW, W, tap, train, seed, part, n, route, cache_f0);
  else
    lpips_head_forward_kernel<C, false><<<grid, 256, 0, st>>>(f0, f1, lin, HW, W, tap, train, seed, part, n, nullptr, nullptr);
}

// partials (B, head_chunks(H, W)); C is one of 64, 128, 256, 512.  route, cache_f0: NULL, or image b's f0 per route[b][0]
int head_forward(const float* f0, const float* f1, const float* lin, int64_t B, int H, int W, int C, int tap, int train,
                 const uint32_t* seed, float* part, cudaStream_t st, const int32_t* route = nullptr, const float* cache_f0 = nullptr) {
  const int n = (int)head_chunks(H, W);
  const dim3 grid((unsigned)n, (unsigned)B);
  const int HW = H * W;
  switch (C) {
    case 64: head_forward_c<64>(grid, f0, f1, lin, HW, W, tap, train, seed, part, n, route, cache_f0, st); break;
    case 128: head_forward_c<128>(grid, f0, f1, lin, HW, W, tap, train, seed, part, n, route, cache_f0, st); break;
    case 256: head_forward_c<256>(grid, f0, f1, lin, HW, W, tap, train, seed, part, n, route, cache_f0, st); break;
    default: head_forward_c<512>(grid, f0, f1, lin, HW, W, tap, train, seed, part, n, route, cache_f0, st); break;
  }
  LP_LAUNCH_CK("lpips_head_forward_kernel");
  return 0;
}

template <int C>
void head_backward_c(dim3 grid, const float* f0, const float* f1, const float* lin, int HW, int W, int tap, int train,
                     const uint32_t* seed, const float* grad_value, int accumulate, float* g, const int32_t* route,
                     const float* cache_f0, cudaStream_t st) {
  if (route)
    lpips_head_backward_kernel<C, true><<<grid, 256, 0, st>>>(f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g, route,
                                                              cache_f0);
  else
    lpips_head_backward_kernel<C, false><<<grid, 256, 0, st>>>(f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g,
                                                               nullptr, nullptr);
}

int head_backward(const float* f0, const float* f1, const float* lin, int64_t B, int H, int W, int C, int tap, int train,
                  const uint32_t* seed, const float* grad_value, int accumulate, float* g, cudaStream_t st,
                  const int32_t* route = nullptr, const float* cache_f0 = nullptr) {
  const dim3 grid((unsigned)head_chunks(H, W), (unsigned)B);
  const int HW = H * W;
  switch (C) {
    case 64: head_backward_c<64>(grid, f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g, route, cache_f0, st); break;
    case 128: head_backward_c<128>(grid, f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g, route, cache_f0, st); break;
    case 256: head_backward_c<256>(grid, f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g, route, cache_f0, st); break;
    default: head_backward_c<512>(grid, f0, f1, lin, HW, W, tap, train, seed, grad_value, accumulate, g, route, cache_f0, st); break;
  }
  LP_LAUNCH_CK("lpips_head_backward_kernel");
  return 0;
}

int check_head_args(const char* what, int64_t B, int H, int W, int C, int tap) {
  if (B < 1 || B > 65535 || H < 1 || W < 1 || H > 32767 || W > 32767 || (C != 64 && C != 128 && C != 256 && C != 512) || tap < 0 ||
      tap > 4)
    return dbw_fail_(what, cudaSuccess);
  return 0;
}

// B, H, W for the trunk through the deepest of `levels` (its tap at least 1x1) and the conv kernels' int32 pixel indices;
// a level mask outside 1..31 fails too
int check_sizes(const char* what, int64_t B, int H, int W, int levels) {
  if (levels < 1 || levels > ALL_LEVELS) return dbw_fail_(what, cudaSuccess);
  const int min_hw = 1 << deepest(levels);
  if (B < 1 || B > 65535 || H < min_hw || W < min_hw || H > 32767 || W > 32767 || B * H * W * 64 >= ((int64_t)1 << 40) ||
      B * H * W >= ((int64_t)1 << 31) - CV_BM)
    return dbw_fail_(what, cudaSuccess);
  return 0;
}

// what a caller reads of net: the conv weights and their prepared copies, the input transform when `transform`, the lin
// weights when `lin`
bool net_ok(const DbwLpipsNet* net, bool transform, bool lin) {
  if (!net || !net->prepared || (transform && (!net->shift || !net->scale))) return false;
  for (int l = 0; l < LP_LAYERS; ++l) if (!net->conv_w[l] || !net->conv_b[l]) return false;
  for (int k = 0; k < 5; ++k) if (lin && !net->lin_w[k]) return false;
  return true;
}

// what differs between the two terms on the trunk: LPIPS (every level, the normalised head with the learned lin weights,
// dropout, the 2x - 1 option, an optional target cache for in0) and the VGG feature loss (the requested levels, either head,
// constant weights and input transform read from the workspace)
struct Term {
  int levels;
  bool normalized;                    // lpips_head_* with lin[k], else vgg_head_plain_* with w[k]
  const float* lin[5];
  float w[5];
  int train;                          // dropout keyed by *seed: the device seed in the forward, the one it saved in the backward
  uint32_t* seed;
  int normalize;                      // x -> 2x - 1, then (x - shift) / scale
  const float *shift, *scale;
  const DbwLpipsTargetCache* cache;   // NULL, or in0's target cache with the route and hit count of the cached calls
  int32_t* route;
  int32_t* n_hits;
};

constexpr int64_t LPIPS_TAIL = 64;    // the seed the forward used, then the target cache's miss count

Term lpips_term(const DbwLpipsNet* net, int normalize, int train, uint32_t* seed, const DbwLpipsTargetCache* cache = nullptr,
                int32_t* route = nullptr, int32_t* n_hits = nullptr) {
  Term t{ALL_LEVELS, true, {}, {}, train, seed, normalize, net->shift, net->scale, cache, route, n_hits};
  for (int k = 0; k < 5; ++k) t.lin[k] = net->lin_w[k];
  return t;
}

// consts: what vgg_consts_kernel wrote, in the workspace's last region
Term vgg_term(const DbwLpipsNet* net, const DbwVggLossOptions* opt, const float* consts) {
  Term t{opt->levels, opt->normalize_features != 0, {}, {}, 0, nullptr, 0, net->shift, net->scale, nullptr, nullptr, nullptr};
  // the first layer applies (x - shift) / scale: the ImageNet statistics, or the identity of the constants
  if (!opt->normalize_input) { t.shift = consts + 5 * 512; t.scale = consts + 5 * 512 + 4; }
  for (int k = 0; k < 5; ++k) { t.lin[k] = consts + 512 * k; t.w[k] = opt->sum_channels ? 1.f : 1.f / (float)LP_TAP_C[k]; }
  return t;
}

// layers 0..last of one image batch x, through the term's input transform: out[l] receives layer l's activation, the pool
// before level k writes pool_out[k].  With route and count (the miss chain), only the images of route[s][1] for slots
// s < *count, compacted in slot order.
int trunk(const DbwLpipsNet* net, const Term& t, const float* x, float* const* out, float* const* pool_out, const Dims& d, int last,
          cudaStream_t st, const int32_t* route = nullptr, const int* count = nullptr) {
  const float* prep = (const float*)net->prepared;
  const int64_t B = d.B;
  if (const int rc = conv_first(x, net->conv_w[0], net->conv_b[0], t.shift, t.scale, t.normalize, out[0], B, d.H[0], d.W[0], st,
                                route, count))
    return rc;
  const float* cur = out[0];
  for (int l = 1; l <= last; ++l) {
    const int lv = LP_LEVEL[l];
    if (lv != LP_LEVEL[l - 1]) {
      if (const int rc = pool(cur, pool_out[lv], B, d.H[lv - 1], d.W[lv - 1], LP_CIN[l], st, count)) return rc;
      cur = pool_out[lv];
    }
    if (const int rc = conv3x3(cur, prep + wfwd_off(l), net->conv_b[l], nullptr, out[l], B, d.H[lv], d.W[lv], LP_CIN[l], LP_COUT[l], 1,
                               st, count))
      return rc;
    cur = out[l];
  }
  return 0;
}

// the outputs of one chain through layer `last`: keep[l] where given, else (as for the pools) whichever scratch tensor the
// layer does not read
void chain_outputs(float* const* keep, int last, float* S0, float* S1, float** out, float** pool_out) {
  const float* cur = nullptr;
  for (int l = 0; l <= last; ++l) {
    if (l > 0 && LP_LEVEL[l] != LP_LEVEL[l - 1]) {
      pool_out[LP_LEVEL[l]] = cur == S0 ? S1 : S0;
      cur = pool_out[LP_LEVEL[l]];
    }
    out[l] = keep[l] ? keep[l] : (cur == S0 ? S1 : S0);
    cur = out[l];
  }
}

bool cache_ok(const DbwLpipsTargetCache* c) { return c && c->arena && c->N >= 1 && c->N < ((int64_t)1 << 31); }

// the plain head of C channels (64, 128, 256 or 512): partials (B, head_chunks(H, W)) as head_forward writes them
int head_plain_forward(const float* f0, const float* f1, float w, int64_t B, int H, int W, int C, float* part, cudaStream_t st) {
  const int n = (int)head_chunks(H, W), HW = H * W;
  const dim3 grid((unsigned)n, (unsigned)B);
  switch (C) {
    case 64: vgg_head_plain_forward_kernel<64><<<grid, 256, 0, st>>>(f0, f1, w, HW, part, n); break;
    case 128: vgg_head_plain_forward_kernel<128><<<grid, 256, 0, st>>>(f0, f1, w, HW, part, n); break;
    case 256: vgg_head_plain_forward_kernel<256><<<grid, 256, 0, st>>>(f0, f1, w, HW, part, n); break;
    default: vgg_head_plain_forward_kernel<512><<<grid, 256, 0, st>>>(f0, f1, w, HW, part, n); break;
  }
  LP_LAUNCH_CK("vgg_head_plain_forward_kernel");
  return 0;
}

int head_plain_backward(const float* f0, const float* f1, float w, int64_t B, int H, int W, int C, const float* grad_value,
                        int accumulate, float* g, cudaStream_t st) {
  const dim3 grid((unsigned)head_chunks(H, W), (unsigned)B);
  const int HW = H * W;
  switch (C) {
    case 64: vgg_head_plain_backward_kernel<64><<<grid, 256, 0, st>>>(f0, f1, w, HW, grad_value, accumulate, g); break;
    case 128: vgg_head_plain_backward_kernel<128><<<grid, 256, 0, st>>>(f0, f1, w, HW, grad_value, accumulate, g); break;
    case 256: vgg_head_plain_backward_kernel<256><<<grid, 256, 0, st>>>(f0, f1, w, HW, grad_value, accumulate, g); break;
    default: vgg_head_plain_backward_kernel<512><<<grid, 256, 0, st>>>(f0, f1, w, HW, grad_value, accumulate, g); break;
  }
  LP_LAUNCH_CK("vgg_head_plain_backward_kernel");
  return 0;
}

// the whole forward into a workspace of layout L: the target cache's lookup of in0, in0's chain (over the misses only when
// cached), in1's chain, the heads of the requested levels, one reduction
int forward_impl(const DbwLpipsNet* net, const Term& t, const float* in0, const float* in1, const Dims& d, const Layout& L,
                 float* ws, float* value, cudaStream_t st) {
  const int64_t B = d.B;
  const int last = LP_TAP_LAYER[deepest(t.levels)];
  // imgs keeps only its requested taps; rec every activation for the backward, or like imgs only its taps
  float* keep0[LP_LAYERS] = {};
  float* keep1[LP_LAYERS] = {};
  for (int l = 0; l <= last; ++l) {
    const int lv = LP_LEVEL[l];
    if (LP_TAP_LAYER[lv] == l && wants(t.levels, lv)) keep0[l] = ws + L.tap0[lv];
    if (L.act[l] >= 0) keep1[l] = ws + L.act[l];
  }
  float *out0[LP_LAYERS], *out1[LP_LAYERS], *pool0[5], *pool1[5];
  chain_outputs(keep0, last, ws + L.s0, ws + L.s1, out0, pool0);
  chain_outputs(keep1, last, ws + L.s0, ws + L.s1, out1, pool1);
  const float* cache_tap[5] = {};
  if (t.cache) {
    // look imgs up (fingerprint partials in S1, the miss count beside the seed), then run its chain over the misses only:
    // their taps land in the first n_miss images of tap0
    const CacheLayout C = cache_layout_of(t.cache->N, d.H[0], d.W[0]);
    const float* arena = (const float*)t.cache->arena;
    for (int k = 0; k < 5; ++k) cache_tap[k] = arena + C.tap[k];
    const int64_t n = 3 * (int64_t)d.H[0] * d.W[0];
    uint64_t* part = (uint64_t*)(ws + L.s1);
    int* n_miss = (int*)(ws + L.tail) + 1;
    lpips_fingerprint_kernel<<<dim3(FP_CHUNKS, (unsigned)B), 256, 0, st>>>(in0, n, part);
    LP_LAUNCH_CK("lpips_fingerprint_kernel");
    lpips_lookup_kernel<<<(unsigned)B, LOOKUP_THREADS, 0, st>>>(in0, n, part, (const uint64_t*)(arena + C.fp), arena + C.img,
                                                                t.cache->N, t.route);
    LP_LAUNCH_CK("lpips_lookup_kernel");
    lpips_route_kernel<<<1, 32, 0, st>>>(t.route, B, n_miss, t.n_hits);
    LP_LAUNCH_CK("lpips_route_kernel");
    if (const int rc = trunk(net, t, in0, out0, pool0, d, last, st, t.route, n_miss)) return rc;
  } else if (const int rc = trunk(net, t, in0, out0, pool0, d, last, st)) {
    return rc;
  }
  if (const int rc = trunk(net, t, in1, out1, pool1, d, last, st)) return rc;
  PartDesc pd;
  for (int k = 0; k < 5; ++k) {
    pd.off[k] = L.part_off[k]; pd.chunks[k] = L.chunks[k]; pd.inv_hw[k] = 1.f / (float)(d.H[k] * d.W[k]);
    if (!wants(t.levels, k)) continue;
    const float *f0 = ws + L.tap0[k], *f1 = out1[LP_TAP_LAYER[k]];
    float* part = ws + L.partials + L.part_off[k];
    if (const int rc = t.normalized ? head_forward(f0, f1, t.lin[k], B, d.H[k], d.W[k], LP_TAP_C[k], k, t.train, t.seed, part, st,
                                                   t.route, cache_tap[k])
                                    : head_plain_forward(f0, f1, t.w[k], B, d.H[k], d.W[k], LP_TAP_C[k], part, st))
      return rc;
  }
  lpips_reduce_kernel<<<1, 256, 0, st>>>(ws + L.partials, pd, (int)B, value, t.seed, t.seed ? (uint32_t*)(ws + L.tail) : nullptr);
  LP_LAUNCH_CK("lpips_reduce_kernel");
  return 0;
}

int backward_impl(const DbwLpipsNet* net, const Term& t, const float* grad_value, const Dims& d, const Layout& L, float* ws,
                  float* grad_in1, cudaStream_t st) {
  const int64_t B = d.B;
  const int last = LP_TAP_LAYER[deepest(t.levels)];
  const float* prep = (const float*)net->prepared;
  const float* cache_tap[5] = {};
  if (t.cache) {
    const CacheLayout C = cache_layout_of(t.cache->N, d.H[0], d.W[0]);
    for (int k = 0; k < 5; ++k) cache_tap[k] = (const float*)t.cache->arena + C.tap[k];
  }
  float* G[2] = {ws + L.s0, ws + L.s1};
  int cur = 0;                        // G[cur] holds the gradient at the pre-activation of layer l
  for (int l = last; l >= 1; --l) {
    const int lv = LP_LEVEL[l];
    const float* act = ws + L.act[l];
    if (l == LP_TAP_LAYER[lv]) {
      const bool bottom = l == last;
      if (!bottom) {                  // G[cur] holds the gradient at the next pool's output: route it back to this tap
        if (const int rc = pool_backward(act, G[cur], G[cur ^ 1], B, d.H[lv], d.W[lv], LP_COUT[l], st)) return rc;
        cur ^= 1;
      }
      if (wants(t.levels, lv)) {
        const float* f0 = ws + L.tap0[lv];
        if (const int rc = t.normalized ? head_backward(f0, act, t.lin[lv], B, d.H[lv], d.W[lv], LP_TAP_C[lv], lv, t.train, t.seed,
                                                        grad_value, !bottom, G[cur], st, t.route, cache_tap[lv])
                                        : head_plain_backward(f0, act, t.w[lv], B, d.H[lv], d.W[lv], LP_TAP_C[lv], grad_value, !bottom,
                                                              G[cur], st))
          return rc;
      } else {                        // the deepest level is always requested
        const int64_t n4 = B * d.H[lv] * d.W[lv] * LP_COUT[l] / 4;
        if (n4 > 0) {
          vgg_relu_mask_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>((const float4*)act, (float4*)G[cur], n4);
          LP_LAUNCH_CK("vgg_relu_mask_kernel");
        }
      }
    }
    // input gradient of layer l; masked by the ReLU below unless a pool sits in between
    const bool after_pool = LP_LEVEL[l - 1] != lv;
    if (const int rc = conv3x3(G[cur], prep + wbwd_off(l), nullptr, after_pool ? nullptr : ws + L.act[l - 1], G[cur ^ 1], B,
                               d.H[lv], d.W[lv], LP_COUT[l], LP_CIN[l], 0, st))
      return rc;
    cur ^= 1;
  }
  return dgrad_last(G[cur], net->conv_w[0], t.scale, t.normalize, grad_in1, B, d.H[0], d.W[0], st);
}

// LPIPS's forward and backward, with or without the target cache
int lpips_forward(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const float* in0, const float* in1, int64_t B, int H,
                  int W, int normalize, int train, int save_for_backward, uint32_t* seed, float* value, int32_t* route,
                  int32_t* n_hits, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  const Dims d = dims_of(B, H, W);
  const Layout L = layout_of(d, ALL_LEVELS, save_for_backward != 0, LPIPS_TAIL);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_lpips_forward: workspace too small", cudaSuccess);
  return forward_impl(net, lpips_term(net, normalize, train, seed, cache, route, n_hits), in0, in1, d, L, (float*)workspace, value,
                      st);
}

int lpips_backward(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const int32_t* route, const float* grad_value, int64_t B,
                   int H, int W, int normalize, int train, float* grad_in1, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  const Dims d = dims_of(B, H, W);
  const Layout L = layout_of(d, ALL_LEVELS, true, LPIPS_TAIL);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_lpips_backward: workspace too small", cudaSuccess);
  float* ws = (float*)workspace;
  return backward_impl(net, lpips_term(net, normalize, train, (uint32_t*)(ws + L.tail), cache, (int32_t*)route), grad_value, d, L, ws,
                       grad_in1, st);
}

int check_cache(const char* what, const DbwLpipsTargetCache* cache, int H, int W, int normalize) {
  if (!cache_ok(cache)) return dbw_fail_(what, cudaSuccess);
  if (cache->H != H || cache->W != W || (cache->normalize != 0) != (normalize != 0)) return dbw_fail_(what, cudaSuccess);
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ C-ABI
extern "C" int dbw_lpips_workspace_bytes(int64_t B, int32_t H, int32_t W, int32_t save_for_backward, size_t* workspace_bytes,
                                         size_t* prepared_bytes) {
  if (const int rc = check_sizes("dbw_lpips_workspace_bytes: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)",
                                B, H, W, ALL_LEVELS)) return rc;
  if (!workspace_bytes || !prepared_bytes) return dbw_fail_("dbw_lpips_workspace_bytes: null pointer argument", cudaSuccess);
  *workspace_bytes = (size_t)layout_of(dims_of(B, H, W), ALL_LEVELS, save_for_backward != 0, LPIPS_TAIL).total * 4;
  *prepared_bytes = (size_t)wprep_total() * 4;
  return 0;
}

extern "C" int dbw_lpips_prepare_weights(const DbwLpipsNet* net, void* stream) {
  if (!net_ok(net, true, false)) return dbw_fail_("dbw_lpips_prepare_weights: null pointer argument", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  float* p = (float*)net->prepared;
  for (int l = 1; l < LP_LAYERS; ++l) {
    const int64_t n = (int64_t)9 * LP_CIN[l] * LP_COUT[l];
    lpips_prepare_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(net->conv_w[l], p + wfwd_off(l), p + wbwd_off(l), LP_CIN[l],
                                                                      LP_COUT[l]);
    LP_LAUNCH_CK("lpips_prepare_kernel");
  }
  return 0;
}

extern "C" int dbw_lpips_forward(const DbwLpipsNet* net, const float* in0, const float* in1, int64_t B, int32_t H, int32_t W,
                                 int32_t normalize, int32_t train, int32_t save_for_backward, uint32_t* seed, float* value,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = check_sizes("dbw_lpips_forward: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B, H, W,
                                  ALL_LEVELS))
    return rc;
  if (!net_ok(net, true, true) || !in0 || !in1 || !seed || !value || !workspace)
    return dbw_fail_("dbw_lpips_forward: null pointer argument", cudaSuccess);
  return lpips_forward(net, nullptr, in0, in1, B, H, W, normalize, train, save_for_backward, seed, value, nullptr, nullptr, workspace,
                       workspace_bytes, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_backward(const DbwLpipsNet* net, const float* grad_value, int64_t B, int32_t H, int32_t W,
                                  int32_t normalize, int32_t train, float* grad_in1, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  if (const int rc = check_sizes("dbw_lpips_backward: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B, H, W,
                                  ALL_LEVELS))
    return rc;
  if (!net_ok(net, true, true) || !grad_value || !grad_in1 || !workspace)
    return dbw_fail_("dbw_lpips_backward: null pointer argument", cudaSuccess);
  return lpips_backward(net, nullptr, nullptr, grad_value, B, H, W, normalize, train, grad_in1, workspace, workspace_bytes,
                        (cudaStream_t)stream);
}

extern "C" int dbw_lpips_cache_bytes(int32_t H, int32_t W, size_t* bytes_per_image) {
  if (const int rc = check_sizes("dbw_lpips_cache_bytes: bad sizes (16 <= H, W <= 32767)", 1, H, W, ALL_LEVELS)) return rc;
  if (!bytes_per_image) return dbw_fail_("dbw_lpips_cache_bytes: null pointer argument", cudaSuccess);
  *bytes_per_image = (size_t)cache_layout_of(1, H, W).total * 4;
  return 0;
}

extern "C" int dbw_lpips_cache_targets(const DbwLpipsNet* net, const float* imgs, const DbwLpipsTargetCache* cache, int64_t chunk,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  if (!cache) return dbw_fail_("dbw_lpips_cache_targets: null pointer argument", cudaSuccess);
  if (const int rc = check_sizes("dbw_lpips_cache_targets: bad sizes (1 <= chunk <= 65535, 16 <= H, W <= 32767, chunk*H*W < 2^31 - 128)",
                                chunk, cache->H, cache->W, ALL_LEVELS))
    return rc;
  if (!net_ok(net, true, true) || !imgs || !cache_ok(cache) || !workspace)
    return dbw_fail_("dbw_lpips_cache_targets: null pointer argument or bad cache (arena, 1 <= N < 2^31)", cudaSuccess);
  const int H = cache->H, W = cache->W;
  const Layout L = layout_of(dims_of(chunk, H, W), ALL_LEVELS, false, LPIPS_TAIL);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_lpips_cache_targets: workspace too small", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  const CacheLayout C = cache_layout_of(cache->N, H, W);
  const Term t = lpips_term(net, cache->normalize, 0, nullptr);
  float* arena = (float*)cache->arena;
  float* ws = (float*)workspace;
  const int64_t n = 3 * (int64_t)H * W;
  float* img = arena + C.img;
  cudaError_t e = cudaMemcpyAsync(img, imgs, (size_t)(cache->N * n) * 4, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return dbw_fail_("dbw_lpips_cache_targets: cudaMemcpyAsync", e);
  // chunk by chunk: the fingerprints (partials in S1), then the taps straight into the arena, by the kernels (and so to the
  // bits) of the per-call forward
  for (int64_t n0 = 0; n0 < cache->N; n0 += chunk) {
    const int64_t nb = cache->N - n0 < chunk ? cache->N - n0 : chunk;
    const Dims d = dims_of(nb, H, W);
    uint64_t* part = (uint64_t*)(ws + L.s1);
    lpips_fingerprint_kernel<<<dim3(FP_CHUNKS, (unsigned)nb), 256, 0, st>>>(img + n0 * n, n, part);
    LP_LAUNCH_CK("lpips_fingerprint_kernel");
    lpips_fingerprint_sum_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, st>>>(part, nb, (uint64_t*)(arena + C.fp) + n0);
    LP_LAUNCH_CK("lpips_fingerprint_sum_kernel");
    float* keep[LP_LAYERS] = {};
    for (int k = 0; k < 5; ++k) keep[LP_TAP_LAYER[k]] = arena + C.tap[k] + n0 * d.H[k] * d.W[k] * LP_TAP_C[k];
    float *out[LP_LAYERS], *pool_out[5];
    chain_outputs(keep, LP_LAYERS - 1, ws + L.s0, ws + L.s1, out, pool_out);
    if (const int rc = trunk(net, t, img + n0 * n, out, pool_out, d, LP_LAYERS - 1, st)) return rc;
  }
  return 0;
}

extern "C" int dbw_lpips_forward_cached(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const float* in0, const float* in1,
                                        int64_t B, int32_t H, int32_t W, int32_t normalize, int32_t train, int32_t save_for_backward,
                                        uint32_t* seed, float* value, int32_t* route, int32_t* n_hits, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  if (const int rc = check_sizes("dbw_lpips_forward_cached: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B,
                                H, W, ALL_LEVELS))
    return rc;
  if (!net_ok(net, true, true) || !in0 || !in1 || !seed || !value || !route || !workspace)
    return dbw_fail_("dbw_lpips_forward_cached: null pointer argument", cudaSuccess);
  if (const int rc = check_cache("dbw_lpips_forward_cached: bad cache (NULL arena, N < 1, or another H, W or normalize)", cache, H, W,
                                 normalize))
    return rc;
  return lpips_forward(net, cache, in0, in1, B, H, W, normalize, train, save_for_backward, seed, value, route, n_hits, workspace,
                       workspace_bytes, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_backward_cached(const DbwLpipsNet* net, const DbwLpipsTargetCache* cache, const int32_t* route,
                                         const float* grad_value, int64_t B, int32_t H, int32_t W, int32_t normalize, int32_t train,
                                         float* grad_in1, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = check_sizes("dbw_lpips_backward_cached: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B,
                                H, W, ALL_LEVELS))
    return rc;
  if (!net_ok(net, true, true) || !route || !grad_value || !grad_in1 || !workspace)
    return dbw_fail_("dbw_lpips_backward_cached: null pointer argument", cudaSuccess);
  if (const int rc = check_cache("dbw_lpips_backward_cached: bad cache (NULL arena, N < 1, or another H, W or normalize)", cache, H, W,
                                 normalize))
    return rc;
  return lpips_backward(net, cache, route, grad_value, B, H, W, normalize, train, grad_in1, workspace, workspace_bytes,
                        (cudaStream_t)stream);
}

// single layers, for tests and per-layer timing (scripts/bench_lpips.py)
extern "C" int dbw_lpips_conv3x3(const float* in, const float* wt, const float* bias, const float* mask, float* out, int64_t B,
                                 int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t relu, void* stream) {
  if (B < 1 || H < 1 || W < 1 || B * H * W >= ((int64_t)1 << 31) - CV_BM || Cin < 32 || Cin % 32 || Cout < 64 || Cout % 64 ||
      (Cout != 64 && Cout % 128))
    return dbw_fail_("dbw_lpips_conv3x3: bad sizes (C_in % 32 == 0, C_out = 64 or a multiple of 128, B*H*W < 2^31 - 128)", cudaSuccess);
  if (!in || !wt || !out) return dbw_fail_("dbw_lpips_conv3x3: null pointer argument", cudaSuccess);
  return conv3x3(in, wt, bias, mask, out, B, H, W, Cin, Cout, relu, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_conv_first(const float* x, const float* w, const float* bias, const float* shift, const float* scale,
                                    int32_t normalize, float* out, int64_t B, int32_t H, int32_t W, void* stream) {
  if (B < 1 || H < 1 || W < 1) return dbw_fail_("dbw_lpips_conv_first: bad sizes", cudaSuccess);
  if (!x || !w || !bias || !shift || !scale || !out) return dbw_fail_("dbw_lpips_conv_first: null pointer argument", cudaSuccess);
  return conv_first(x, w, bias, shift, scale, normalize, out, B, H, W, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_dgrad_last(const float* g, const float* w, const float* scale, int32_t normalize, float* out, int64_t B,
                                    int32_t H, int32_t W, void* stream) {
  if (B < 1 || H < 1 || W < 1) return dbw_fail_("dbw_lpips_dgrad_last: bad sizes", cudaSuccess);
  if (!g || !w || !scale || !out) return dbw_fail_("dbw_lpips_dgrad_last: null pointer argument", cudaSuccess);
  return dgrad_last(g, w, scale, normalize, out, B, H, W, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_maxpool(const float* in, float* out, int64_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (B < 1 || H < 1 || W < 1 || C < 4 || C % 4) return dbw_fail_("dbw_lpips_maxpool: bad sizes", cudaSuccess);
  if (!in || !out) return dbw_fail_("dbw_lpips_maxpool: null pointer argument", cudaSuccess);
  return pool(in, out, B, H, W, C, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_maxpool_backward(const float* in, const float* gout, float* gin, int64_t B, int32_t H, int32_t W, int32_t C,
                                          void* stream) {
  if (B < 1 || H < 1 || W < 1 || C < 4 || C % 4) return dbw_fail_("dbw_lpips_maxpool_backward: bad sizes", cudaSuccess);
  if (!in || !gout || !gin) return dbw_fail_("dbw_lpips_maxpool_backward: null pointer argument", cudaSuccess);
  return pool_backward(in, gout, gin, B, H, W, C, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_head_forward(const float* f0, const float* f1, const float* lin, int64_t B, int32_t H, int32_t W, int32_t C,
                                      int32_t tap, int32_t train, const uint32_t* seed, float* partials, void* stream) {
  if (const int rc = check_head_args("dbw_lpips_head_forward: bad sizes (1 <= B <= 65535, 1 <= H, W <= 32767, C = 64, 128, 256 or "
                                     "512, 0 <= tap <= 4)", B, H, W, C, tap))
    return rc;
  if (!f0 || !f1 || !lin || (train && !seed) || !partials)
    return dbw_fail_("dbw_lpips_head_forward: null pointer argument", cudaSuccess);
  return head_forward(f0, f1, lin, B, H, W, C, tap, train, seed, partials, (cudaStream_t)stream);
}

extern "C" int dbw_lpips_head_backward(const float* f0, const float* f1, const float* lin, int64_t B, int32_t H, int32_t W, int32_t C,
                                       int32_t tap, int32_t train, const uint32_t* seed, const float* grad_value,
                                       int32_t accumulate, float* g, void* stream) {
  if (const int rc = check_head_args("dbw_lpips_head_backward: bad sizes (1 <= B <= 65535, 1 <= H, W <= 32767, C = 64, 128, 256 or "
                                     "512, 0 <= tap <= 4)", B, H, W, C, tap))
    return rc;
  if (!f0 || !f1 || !lin || (train && !seed) || !grad_value || !g)
    return dbw_fail_("dbw_lpips_head_backward: null pointer argument", cudaSuccess);
  return head_backward(f0, f1, lin, B, H, W, C, tap, train, seed, grad_value, accumulate, g, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------ VGG feature loss (C-ABI)
#define VGG_SIZES "(levels: bits 0..4, not 0; 1 <= B <= 65535, 2^(deepest level - 1) <= H, W <= 32767, B*H*W < 2^31 - 128)"

extern "C" int dbw_vgg_loss_workspace_bytes(int64_t B, int32_t H, int32_t W, const DbwVggLossOptions* opt, int32_t save_for_backward,
                                            size_t* workspace_bytes) {
  if (const int rc = check_sizes("dbw_vgg_loss_workspace_bytes: bad options or sizes " VGG_SIZES, B, H, W, opt ? opt->levels : 0))
    return rc;
  if (!workspace_bytes) return dbw_fail_("dbw_vgg_loss_workspace_bytes: null pointer argument", cudaSuccess);
  *workspace_bytes = (size_t)layout_of(dims_of(B, H, W), opt->levels, save_for_backward != 0, VGG_CONSTS).total * 4;
  return 0;
}

extern "C" int dbw_vgg_loss_forward(const DbwLpipsNet* net, const DbwVggLossOptions* opt, const float* in0, const float* in1, int64_t B,
                                    int32_t H, int32_t W, int32_t save_for_backward, float* value, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (const int rc = check_sizes("dbw_vgg_loss_forward: bad options or sizes " VGG_SIZES, B, H, W, opt ? opt->levels : 0)) return rc;
  if (!net_ok(net, opt->normalize_input, false) || !in0 || !in1 || !value || !workspace)
    return dbw_fail_("dbw_vgg_loss_forward: null pointer argument", cudaSuccess);
  const Dims d = dims_of(B, H, W);
  const Layout L = layout_of(d, opt->levels, save_for_backward != 0, VGG_CONSTS);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_vgg_loss_forward: workspace too small", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  vgg_consts_kernel<<<1, 256, 0, st>>>(ws + L.tail, opt->sum_channels);
  LP_LAUNCH_CK("vgg_consts_kernel");
  return forward_impl(net, vgg_term(net, opt, ws + L.tail), in0, in1, d, L, ws, value, st);
}

extern "C" int dbw_vgg_loss_backward(const DbwLpipsNet* net, const DbwVggLossOptions* opt, const float* grad_value, int64_t B,
                                     int32_t H, int32_t W, float* grad_in1, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = check_sizes("dbw_vgg_loss_backward: bad options or sizes " VGG_SIZES, B, H, W, opt ? opt->levels : 0)) return rc;
  if (!net_ok(net, opt->normalize_input, false) || !grad_value || !grad_in1 || !workspace)
    return dbw_fail_("dbw_vgg_loss_backward: null pointer argument", cudaSuccess);
  const Dims d = dims_of(B, H, W);
  const Layout L = layout_of(d, opt->levels, true, VGG_CONSTS);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_vgg_loss_backward: workspace too small", cudaSuccess);
  float* ws = (float*)workspace;
  return backward_impl(net, vgg_term(net, opt, ws + L.tail), grad_value, d, L, ws, grad_in1, (cudaStream_t)stream);
}

// the plain head alone, for tests: the launchers of the whole term
extern "C" int dbw_vgg_head_forward(const float* f0, const float* f1, float w, int64_t B, int32_t H, int32_t W, int32_t C,
                                    float* partials, void* stream) {
  if (const int rc = check_head_args("dbw_vgg_head_forward: bad sizes (1 <= B <= 65535, 1 <= H, W <= 32767, C = 64, 128, 256 or 512)",
                                     B, H, W, C, 0))
    return rc;
  if (!f0 || !f1 || !partials) return dbw_fail_("dbw_vgg_head_forward: null pointer argument", cudaSuccess);
  return head_plain_forward(f0, f1, w, B, H, W, C, partials, (cudaStream_t)stream);
}

extern "C" int dbw_vgg_head_backward(const float* f0, const float* f1, float w, int64_t B, int32_t H, int32_t W, int32_t C,
                                     const float* grad_value, int32_t accumulate, float* g, void* stream) {
  if (const int rc = check_head_args("dbw_vgg_head_backward: bad sizes (1 <= B <= 65535, 1 <= H, W <= 32767, C = 64, 128, 256 or 512)",
                                     B, H, W, C, 0))
    return rc;
  if (!f0 || !f1 || !grad_value || !g) return dbw_fail_("dbw_vgg_head_backward: null pointer argument", cudaSuccess);
  return head_plain_backward(f0, f1, w, B, H, W, C, grad_value, accumulate, g, (cudaStream_t)stream);
}
