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

// workspace layout, in floats: rec activations of the 13 layers (only its 5 taps when no backward follows), the 5 taps of
// imgs, two scratch tensors of B*H*W*64 (pool outputs and the intermediates not kept in the forward, the running gradient
// in the backward), the head partials, the seed the forward used
struct Layout {
  int64_t act[LP_LAYERS], tap0[5], s0, s1, partials, seed, total;
  int64_t chunks[5], part_off[5];
};

bool is_tap_layer(int l) { return l == 1 || l == 3 || l == 6 || l == 9 || l == 12; }

Layout layout_of(const Dims& d, bool save) {
  Layout L; int64_t o = 0;
  for (int l = 0; l < LP_LAYERS; ++l) {
    L.act[l] = -1;
    if (!save && !is_tap_layer(l)) continue;
    L.act[l] = o; o += align64(d.B * d.H[LP_LEVEL[l]] * d.W[LP_LEVEL[l]] * LP_COUT[l]);
  }
  for (int k = 0; k < 5; ++k) { L.tap0[k] = o; o += align64(d.B * d.H[k] * d.W[k] * LP_TAP_C[k]); }
  const int64_t big = align64(d.B * d.H[0] * d.W[0] * 64);
  L.s0 = o; o += big;
  L.s1 = o; o += big;
  L.partials = o;
  int64_t p = 0;
  for (int k = 0; k < 5; ++k) {
    L.chunks[k] = ((int64_t)d.H[k] * d.W[k] + HEAD_PIX - 1) / HEAD_PIX;
    L.part_off[k] = p; p += d.B * L.chunks[k];
  }
  o += align64(p);
  L.seed = o; o += 64;
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
template <int BN>
__global__ void __launch_bounds__(CV_THREADS, 2) lpips_conv3x3_kernel(const float* __restrict__ in, const float* __restrict__ wt,
                                                                      const float* __restrict__ bias, const float* __restrict__ mask,
                                                                      float* __restrict__ out, int M, int H, int W, int Cin,
                                                                      int Cout, int relu) {
  using C = CvCfg<BN>;
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
// zero padding is of the scaled image
__global__ void __launch_bounds__(256) lpips_conv_first_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, const float* __restrict__ shift,
                                                               const float* __restrict__ scale, int normalize,
                                                               float* __restrict__ out, int64_t M, int H, int W) {
  __shared__ float ws[27][64];       // [(ci*3+ky)*3+kx][co]
  __shared__ float bs[64];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) ws[i % 27][i / 27] = w[i];
  if (threadIdx.x < 64) bs[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (q >= 4 * M) return;
  const int64_t m = q >> 2;
  const int cg = (int)(q & 3) * 16;
  const int64_t HW = (int64_t)H * W, b = m / HW;
  const int rem = (int)(m - b * HW), y = rem / W, xx = rem - (rem / W) * W;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = bs[cg + j];
  for (int ci = 0; ci < 3; ++ci) {
    const float sh = shift[ci], sc = scale[ci];
    const float* plane = x + (b * 3 + ci) * HW;
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
__global__ void lpips_pool_kernel(const float4* __restrict__ in, float4* __restrict__ out, int64_t n_out, int H, int W, int C4) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const int OH = H / 2, OW = W / 2;
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

template <int C>
__global__ void __launch_bounds__(256) lpips_head_forward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                 const float* __restrict__ lin, int HW, int W, int tap, int train,
                                                                 const uint32_t* __restrict__ seed, float* __restrict__ partials,
                                                                 int n_chunks) {
  constexpr int NPL = C / 32;
  __shared__ float wsum[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  float wl[NPL];
#pragma unroll
  for (int j = 0; j < NPL; ++j) wl[j] = lin[lane + 32 * j];
  const uint32_t himg = train ? dbw_lpips_hash_image(*seed, (uint32_t)tap, (uint32_t)b) : 0u;
  float acc = 0.f;
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C;
    float u0[NPL], u1[NPL], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      u0[j] = f0[base + lane + 32 * j]; u1[j] = f1[base + lane + 32 * j];
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
template <int C>
__global__ void __launch_bounds__(256) lpips_head_backward_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                  const float* __restrict__ lin, int HW, int W, int tap, int train,
                                                                  const uint32_t* __restrict__ seed,
                                                                  const float* __restrict__ grad_value, int accumulate,
                                                                  float* __restrict__ g) {
  constexpr int NPL = C / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.y;
  const float gs = __fdiv_rn(grad_value[b], (float)HW);
  float wl[NPL];
#pragma unroll
  for (int j = 0; j < NPL; ++j) wl[j] = lin[lane + 32 * j] * gs;
  const uint32_t himg = train ? dbw_lpips_hash_image(*seed, (uint32_t)tap, (uint32_t)b) : 0u;
  for (int s = 0; s < HEAD_PIX / 8; ++s) {
    const int p = blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / 8) + s;
    if (p >= HW) break;
    const int64_t base = ((int64_t)b * HW + p) * C;
    float u0[NPL], u1[NPL], s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      u0[j] = f0[base + lane + 32 * j]; u1[j] = f1[base + lane + 32 * j];
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

// value[b] = sum over taps of (sum of the tap's partials, in chunk order) / (H_k W_k); then the seed is saved for the
// backward and advanced
struct PartDesc { int64_t off[5], chunks[5]; float inv_hw[5]; };

__global__ void lpips_reduce_kernel(const float* __restrict__ partials, PartDesc pd, int B, float* __restrict__ value,
                                    uint32_t* __restrict__ seed, uint32_t* __restrict__ seed_used) {
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float v = 0.f;
    for (int k = 0; k < 5; ++k) {
      const float* p = partials + pd.off[k] + (int64_t)b * pd.chunks[k];
      float s = 0.f;
      for (int64_t c = 0; c < pd.chunks[k]; ++c) s += p[c];
      v += s * pd.inv_hw[k];
    }
    value[b] = v;
  }
  if (threadIdx.x == 0) { *seed_used = *seed; *seed = *seed + 1u; }
}

__global__ void lpips_prepare_kernel(const float* __restrict__ w, float* __restrict__ fwd, float* __restrict__ bwd, int Cin, int Cout) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)Cout * Cin * 9) return;
  const int tap = (int)(i % 9), ci = (int)((i / 9) % Cin), co = (int)(i / (9 * (int64_t)Cin));
  const float v = __uint_as_float(tf32_rna(w[i]));
  fwd[((int64_t)co * 9 + tap) * Cin + ci] = v;
  bwd[((int64_t)ci * 9 + (8 - tap)) * Cout + co] = v;           // (2-ky)*3 + (2-kx) = 8 - tap
}

// ------------------------------------------------------------------------------------------------ launchers
// the dynamic shared-memory limit is a per-device attribute: set before every launch (cheap), as the raster kernels do
int set_attrs() {
  cudaError_t e = cudaFuncSetAttribute(lpips_conv3x3_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, CvCfg<128>::SMEM);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(lpips_conv3x3_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, CvCfg<64>::SMEM);
  if (e != cudaSuccess) return dbw_fail_("lpips: cudaFuncSetAttribute", e);
  return 0;
}

int conv3x3(const float* in, const float* wt, const float* bias, const float* mask, float* out, int64_t B, int H, int W, int Cin,
            int Cout, int relu, cudaStream_t st) {
  if (const int rc = set_attrs()) return rc;
  const int64_t M = B * H * W;
  if (M == 0) return 0;
  if (Cout == 64) {
    const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)(Cout / 64));
    lpips_conv3x3_kernel<64><<<grid, CV_THREADS, CvCfg<64>::SMEM, st>>>(in, wt, bias, mask, out, (int)M, H, W, Cin, Cout, relu);
  } else {
    const dim3 grid((unsigned)((M + CV_BM - 1) / CV_BM), (unsigned)(Cout / 128));
    lpips_conv3x3_kernel<128><<<grid, CV_THREADS, CvCfg<128>::SMEM, st>>>(in, wt, bias, mask, out, (int)M, H, W, Cin, Cout, relu);
  }
  LP_LAUNCH_CK("lpips_conv3x3_kernel");
  return 0;
}

int conv_first(const float* x, const float* w, const float* bias, const float* shift, const float* scale, int normalize, float* out,
               int64_t B, int H, int W, cudaStream_t st) {
  const int64_t M = B * H * W;
  lpips_conv_first_kernel<<<(unsigned)((4 * M + 255) / 256), 256, 0, st>>>(x, w, bias, shift, scale, normalize, out, M, H, W);
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

int pool(const float* in, float* out, int64_t B, int H, int W, int C, cudaStream_t st) {
  const int64_t n = B * (H / 2) * (W / 2) * (C / 4);
  if (n == 0) return 0;
  lpips_pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float4*)in, (float4*)out, n, H, W, C / 4);
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

int head_forward(int k, const float* f0, const float* f1, const float* lin, const Dims& d, const Layout& L, int train,
                 const uint32_t* seed, float* ws, cudaStream_t st) {
  const dim3 grid((unsigned)L.chunks[k], (unsigned)d.B);
  const int HW = d.H[k] * d.W[k];
  float* part = ws + L.partials + L.part_off[k];
  const int n = (int)L.chunks[k];
  switch (LP_TAP_C[k]) {
    case 64: lpips_head_forward_kernel<64><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, part, n); break;
    case 128: lpips_head_forward_kernel<128><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, part, n); break;
    case 256: lpips_head_forward_kernel<256><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, part, n); break;
    default: lpips_head_forward_kernel<512><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, part, n); break;
  }
  LP_LAUNCH_CK("lpips_head_forward_kernel");
  return 0;
}

int head_backward(int k, const float* f0, const float* f1, const float* lin, const Dims& d, const Layout& L, int train,
                  const uint32_t* seed, const float* grad_value, int accumulate, float* g, cudaStream_t st) {
  const dim3 grid((unsigned)L.chunks[k], (unsigned)d.B);
  const int HW = d.H[k] * d.W[k];
  switch (LP_TAP_C[k]) {
    case 64: lpips_head_backward_kernel<64><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, grad_value, accumulate, g); break;
    case 128: lpips_head_backward_kernel<128><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, grad_value, accumulate, g); break;
    case 256: lpips_head_backward_kernel<256><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, grad_value, accumulate, g); break;
    default: lpips_head_backward_kernel<512><<<grid, 256, 0, st>>>(f0, f1, lin, HW, d.W[k], k, train, seed, grad_value, accumulate, g); break;
  }
  LP_LAUNCH_CK("lpips_head_backward_kernel");
  return 0;
}

int check_dims(const char* what, int64_t B, int H, int W) {
  if (B < 1 || B > 65535 || H < 16 || W < 16 || H > 32767 || W > 32767 || B * H * W * 64 >= ((int64_t)1 << 40) ||
      B * H * W >= ((int64_t)1 << 31) - CV_BM)
    return dbw_fail_(what, cudaSuccess);
  return 0;
}

bool net_ok(const DbwLpipsNet* net) {
  if (!net || !net->shift || !net->scale || !net->prepared) return false;
  for (int l = 0; l < LP_LAYERS; ++l) if (!net->conv_w[l] || !net->conv_b[l]) return false;
  for (int k = 0; k < 5; ++k) if (!net->lin_w[k]) return false;
  return true;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ C-ABI
extern "C" int dbw_lpips_workspace_bytes(int64_t B, int32_t H, int32_t W, int32_t save_for_backward, size_t* workspace_bytes,
                                         size_t* prepared_bytes) {
  if (const int rc = check_dims("dbw_lpips_workspace_bytes: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)",
                                B, H, W)) return rc;
  if (!workspace_bytes || !prepared_bytes) return dbw_fail_("dbw_lpips_workspace_bytes: null pointer argument", cudaSuccess);
  *workspace_bytes = (size_t)layout_of(dims_of(B, H, W), save_for_backward != 0).total * 4;
  *prepared_bytes = (size_t)wprep_total() * 4;
  return 0;
}

extern "C" int dbw_lpips_prepare_weights(const DbwLpipsNet* net, void* stream) {
  if (!net_ok(net)) return dbw_fail_("dbw_lpips_prepare_weights: null pointer argument", cudaSuccess);
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
  if (const int rc = check_dims("dbw_lpips_forward: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B, H, W))
    return rc;
  if (!net_ok(net) || !in0 || !in1 || !seed || !value || !workspace)
    return dbw_fail_("dbw_lpips_forward: null pointer argument", cudaSuccess);
  const Dims d = dims_of(B, H, W);
  const bool save = save_for_backward != 0;
  const Layout L = layout_of(d, save);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_lpips_forward: workspace too small", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const float* prep = (const float*)net->prepared;
  float *S0 = ws + L.s0, *S1 = ws + L.s1, *T[5];
  for (int k = 0; k < 5; ++k) T[k] = ws + L.tap0[k];
  // imgs keeps only its taps: the other layers alternate between the scratch tensors (pool outputs go to S0)
  float* out0[LP_LAYERS] = {S1, T[0], S1, T[1], S1, S0, T[2], S1, S0, T[3], S1, S0, T[4]};
  // rec keeps every activation for the backward, or like imgs only its taps
  float* out1[LP_LAYERS];
  for (int l = 0; l < LP_LAYERS; ++l) out1[l] = L.act[l] >= 0 ? ws + L.act[l] : out0[l];
  for (int img = 0; img < 2; ++img) {
    float* const* out = img ? out1 : out0;
    if (const int rc = conv_first(img ? in1 : in0, net->conv_w[0], net->conv_b[0], net->shift, net->scale, normalize, out[0], B, H, W, st))
      return rc;
    const float* cur = out[0];
    for (int l = 1; l < LP_LAYERS; ++l) {
      const int lv = LP_LEVEL[l];
      if (lv != LP_LEVEL[l - 1]) {
        if (const int rc = pool(cur, S0, B, d.H[lv - 1], d.W[lv - 1], LP_CIN[l], st)) return rc;
        cur = S0;
      }
      if (const int rc = conv3x3(cur, prep + wfwd_off(l), net->conv_b[l], nullptr, out[l], B, d.H[lv], d.W[lv], LP_CIN[l], LP_COUT[l], 1, st))
        return rc;
      cur = out[l];
    }
  }
  for (int k = 0; k < 5; ++k)
    if (const int rc = head_forward(k, T[k], out1[LP_TAP_LAYER[k]], net->lin_w[k], d, L, train, seed, ws, st)) return rc;
  PartDesc pd;
  for (int k = 0; k < 5; ++k) { pd.off[k] = L.part_off[k]; pd.chunks[k] = L.chunks[k]; pd.inv_hw[k] = 1.f / (float)(d.H[k] * d.W[k]); }
  lpips_reduce_kernel<<<1, 256, 0, st>>>(ws + L.partials, pd, (int)B, value, seed, (uint32_t*)(ws + L.seed));
  LP_LAUNCH_CK("lpips_reduce_kernel");
  return 0;
}

extern "C" int dbw_lpips_backward(const DbwLpipsNet* net, const float* grad_value, int64_t B, int32_t H, int32_t W,
                                  int32_t normalize, int32_t train, float* grad_in1, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  if (const int rc = check_dims("dbw_lpips_backward: bad sizes (1 <= B <= 65535, 16 <= H, W <= 32767, B*H*W < 2^31 - 128)", B, H, W))
    return rc;
  if (!net_ok(net) || !grad_value || !grad_in1 || !workspace)
    return dbw_fail_("dbw_lpips_backward: null pointer argument", cudaSuccess);
  const Dims d = dims_of(B, H, W);
  const Layout L = layout_of(d, true);
  if (workspace_bytes < (size_t)L.total * 4) return dbw_fail_("dbw_lpips_backward: workspace too small", cudaSuccess);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const float* prep = (const float*)net->prepared;
  const uint32_t* seed_used = (const uint32_t*)(ws + L.seed);
  float* G[2] = {ws + L.s0, ws + L.s1};
  int cur = 0;                        // G[cur] holds the gradient at the pre-activation of layer l
  for (int l = LP_LAYERS - 1; l >= 1; --l) {
    const int lv = LP_LEVEL[l];
    const float* act = ws + L.act[l];
    if (l == LP_TAP_LAYER[lv]) {
      const bool deepest = lv == 4;
      if (!deepest) {                 // G[cur] holds the gradient at the next pool's output: route it back to this tap
        if (const int rc = pool_backward(act, G[cur], G[cur ^ 1], B, d.H[lv], d.W[lv], LP_COUT[l], st)) return rc;
        cur ^= 1;
      }
      if (const int rc = head_backward(lv, ws + L.tap0[lv], act, net->lin_w[lv], d, L, train, seed_used, grad_value, !deepest, G[cur], st))
        return rc;
    }
    // input gradient of layer l; masked by the ReLU below unless a pool sits in between
    const bool after_pool = LP_LEVEL[l - 1] != lv;
    if (const int rc = conv3x3(G[cur], prep + wbwd_off(l), nullptr, after_pool ? nullptr : ws + L.act[l - 1], G[cur ^ 1], B,
                               d.H[lv], d.W[lv], LP_COUT[l], LP_CIN[l], 0, st))
      return rc;
    cur ^= 1;
  }
  return dgrad_last(G[cur], net->conv_w[0], net->scale, normalize, grad_in1, B, H, W, st);
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
