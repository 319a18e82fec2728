// dbw_data.cu -- sm_90a training views held on the device (see include/dbw_render.h, "Training views"; the per-element math
// is dbw_data_math.cuh):
//   resample_u8      Pillow's Image.resize(size, BILINEAR) of decoded uint8 RGB images, bit for bit: a horizontal and a
//                    vertical pass (in Pillow's order) of integer multiply-adds over coefficient tables the host builds;
//   gather_views     one batch of (B, 3, H, W) float32 images (x / 255, correctly rounded) and its per-view camera tensors,
//                    gathered from the resident views by B indices read on the device, in one capturable launch;
//   subsample_points the first n entries of a keyed permutation of the ground-truth cloud, per view.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/dbw_render.h"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

#include "dbw_data_math.cuh"

constexpr int DATA_THREADS = 256;

// ------------------------------------------------------------------ resample_u8
// one thread per output pixel of n images; `src` (n, src_rows, src_w, 3), `dst` (n, dst_rows, dst_w, 3).  horizontal: output
// (r, c) reads taps along row r + row0 from column bounds[2 c]; vertical: output (r, c) reads taps down column c from row
// bounds[2 r]
template <bool HORIZONTAL>
__global__ void __launch_bounds__(DATA_THREADS)
resample_u8_kernel(const unsigned char* __restrict__ src, int src_rows, int src_w, int row0, unsigned char* __restrict__ dst,
                   int dst_rows, int dst_w, const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk, int ksize,
                   long long n_pixels) {
  const long long i = (long long)blockIdx.x * DATA_THREADS + threadIdx.x;
  if (i >= n_pixels) return;
  const long long per_img = (long long)dst_rows * dst_w;
  const int img = (int)(i / per_img);
  const int r = (int)((i % per_img) / dst_w), c = (int)(i % dst_w);
  const unsigned char* s = src + (size_t)img * src_rows * src_w * 3;
  const int o = HORIZONTAL ? c : r;
  const int first = bounds[2 * o], taps = bounds[2 * o + 1];
  const unsigned char* p = HORIZONTAL ? s + ((size_t)(r + row0) * src_w + first) * 3 : s + ((size_t)first * src_w + c) * 3;
  resample_pixel(p, HORIZONTAL ? 3 : 3ll * src_w, taps, kk + (size_t)o * ksize, dst + (size_t)i * 3);
}

namespace {

struct ResamplePlan {
  bool horizontal, vertical, vertical_first;
  int ksize_h, ksize_v, tmp_rows, row0;
  size_t off_bh, off_kh, off_bv, off_kv, off_tmp, bytes;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

ResamplePlan resample_plan(int n, int in_h, int in_w, int out_h, int out_w, std::vector<int32_t>* bh, std::vector<int32_t>* kh,
                           std::vector<int32_t>* bv, std::vector<int32_t>* kv) {
  ResamplePlan P{};
  P.horizontal = out_w != in_w;
  P.vertical = out_h != in_h;
  P.vertical_first = P.horizontal && P.vertical && resample_vertical_first(in_h, in_w, out_h);
  P.ksize_h = resample_ksize(in_w, out_w);
  P.ksize_v = resample_ksize(in_h, out_h);
  bh->assign((size_t)2 * out_w, 0);
  kh->assign((size_t)out_w * P.ksize_h, 0);
  bv->assign((size_t)2 * out_h, 0);
  kv->assign((size_t)out_h * P.ksize_v, 0);
  resample_coeffs(in_w, out_w, bh->data(), kh->data());
  resample_coeffs(in_h, out_h, bv->data(), kv->data());
  // horizontal first: Pillow's horizontal pass covers only the input rows the vertical pass reads, and the vertical bounds
  // are shifted to them.  Vertical first: the intermediate is the (out_h, in_w) image of the first resize.
  P.row0 = (*bv)[0];
  P.tmp_rows = (*bv)[2 * out_h - 2] + (*bv)[2 * out_h - 1] - P.row0;
  if (P.vertical_first)
    P.row0 = 0, P.tmp_rows = out_h;
  else if (P.horizontal)
    for (int i = 0; i < out_h; ++i) (*bv)[2 * i] -= P.row0;
  else
    P.row0 = 0, P.tmp_rows = in_h;
  P.off_bh = 0;
  P.off_kh = align256(P.off_bh + bh->size() * 4);
  P.off_bv = align256(P.off_kh + kh->size() * 4);
  P.off_kv = align256(P.off_bv + bv->size() * 4);
  P.off_tmp = align256(P.off_kv + kv->size() * 4);
  const size_t tmp_w = P.vertical_first ? (size_t)in_w : (size_t)out_w;
  P.bytes = P.off_tmp + (P.horizontal && P.vertical ? (size_t)n * P.tmp_rows * tmp_w * 3 : 0);
  return P;
}

bool resample_args_ok(int n, int in_h, int in_w, int out_h, int out_w) {
  if (n < 1 || in_h < 1 || in_w < 1 || out_h < 1 || out_w < 1) return false;
  return (long long)n * in_h * in_w * 3 <= (1ll << 40) && (long long)n * out_h * out_w * 3 <= (1ll << 40);
}

}  // namespace

extern "C" int dbw_resample_u8_workspace_bytes(int32_t n, int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, size_t* bytes) {
  if (!bytes) return dbw_fail_("dbw_resample_u8_workspace_bytes: null argument", cudaSuccess);
  if (!resample_args_ok(n, in_h, in_w, out_h, out_w))
    return dbw_fail_("dbw_resample_u8_workspace_bytes: sizes must be positive", cudaSuccess);
  std::vector<int32_t> bh, kh, bv, kv;
  *bytes = resample_plan(n, in_h, in_w, out_h, out_w, &bh, &kh, &bv, &kv).bytes;
  return 0;
}

extern "C" int dbw_resample_u8(int32_t n, int32_t in_h, int32_t in_w, const uint8_t* src, int32_t out_h, int32_t out_w, uint8_t* dst,
                               void* workspace, size_t workspace_bytes, void* stream) {
  if (!src || !dst) return dbw_fail_("dbw_resample_u8: null image", cudaSuccess);
  if (!resample_args_ok(n, in_h, in_w, out_h, out_w))
    return dbw_fail_("dbw_resample_u8: sizes must be positive", cudaSuccess);
  std::vector<int32_t> bh, kh, bv, kv;
  const ResamplePlan P = resample_plan(n, in_h, in_w, out_h, out_w, &bh, &kh, &bv, &kv);
  if (!workspace || workspace_bytes < P.bytes) return dbw_fail_("dbw_resample_u8: workspace too small", cudaSuccess);
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const std::vector<int32_t>* tabs[4] = {&bh, &kh, &bv, &kv};
  const size_t offs[4] = {P.off_bh, P.off_kh, P.off_bv, P.off_kv};
  for (int t = 0; t < 4; ++t) {
    // pageable source: the call returns once the table has been staged, so the vectors may go out of scope
    cudaError_t e = cudaMemcpyAsync(ws + offs[t], tabs[t]->data(), tabs[t]->size() * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return dbw_fail_("dbw_resample_u8: coefficient table copy", e);
  }
  const int32_t *d_bh = (const int32_t*)(ws + P.off_bh), *d_kh = (const int32_t*)(ws + P.off_kh);
  const int32_t *d_bv = (const int32_t*)(ws + P.off_bv), *d_kv = (const int32_t*)(ws + P.off_kv);
  if (!P.horizontal && !P.vertical) {                              // Pillow copies the image
    cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)n * in_h * in_w * 3, cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? 0 : dbw_fail_("dbw_resample_u8: copy", e);
  }
  if (P.vertical_first) {
    unsigned char* tmp = (unsigned char*)(ws + P.off_tmp);
    long long np = (long long)n * out_h * in_w;
    resample_u8_kernel<false><<<(unsigned)((np + DATA_THREADS - 1) / DATA_THREADS), DATA_THREADS, 0, s>>>(
        src, in_h, in_w, 0, tmp, out_h, in_w, d_bv, d_kv, P.ksize_v, np);
    dbw_count_launch_();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return dbw_fail_("resample_u8_kernel<vertical>", e);
    np = (long long)n * out_h * out_w;
    resample_u8_kernel<true><<<(unsigned)((np + DATA_THREADS - 1) / DATA_THREADS), DATA_THREADS, 0, s>>>(
        tmp, out_h, in_w, 0, dst, out_h, out_w, d_bh, d_kh, P.ksize_h, np);
    dbw_count_launch_();
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : dbw_fail_("resample_u8_kernel<horizontal>", e);
  }
  const unsigned char* cur = src;
  int cur_rows = in_h;
  if (P.horizontal) {
    unsigned char* out = P.vertical ? (unsigned char*)(ws + P.off_tmp) : dst;
    const long long np = (long long)n * P.tmp_rows * out_w;
    resample_u8_kernel<true><<<(unsigned)((np + DATA_THREADS - 1) / DATA_THREADS), DATA_THREADS, 0, s>>>(
        src, in_h, in_w, P.row0, out, P.tmp_rows, out_w, d_bh, d_kh, P.ksize_h, np);
    dbw_count_launch_();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return dbw_fail_("resample_u8_kernel<horizontal>", e);
    cur = out;
    cur_rows = P.tmp_rows;
  }
  if (P.vertical) {
    const long long np = (long long)n * out_h * out_w;
    resample_u8_kernel<false><<<(unsigned)((np + DATA_THREADS - 1) / DATA_THREADS), DATA_THREADS, 0, s>>>(
        cur, cur_rows, out_w, 0, dst, out_h, out_w, d_bv, d_kv, P.ksize_v, np);
    dbw_count_launch_();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return dbw_fail_("resample_u8_kernel<vertical>", e);
  }
  return 0;
}

// ------------------------------------------------------------------ gather_views
struct GatherFields {
  const uint32_t* src[DBW_GATHER_MAX_FIELDS];
  uint32_t* dst[DBW_GATHER_MAX_FIELDS];
  long long words[DBW_GATHER_MAX_FIELDS];
  int n;
};

// CTA row blockIdx.y = batch entry b; the CTAs of a row stride over the view's pixels (uint8 images) and over the words of
// each field.  An index outside [0, n_views) writes NaN words.
__global__ void __launch_bounds__(DATA_THREADS)
gather_views_kernel(const int64_t* __restrict__ idx, int n_views, const unsigned char* __restrict__ views, int hw,
                    float* __restrict__ imgs, GatherFields F) {
  const int b = blockIdx.y;
  const int64_t v = idx[b];
  const bool ok = v >= 0 && v < n_views;
  const long long t0 = (long long)blockIdx.x * DATA_THREADS + threadIdx.x, step = (long long)gridDim.x * DATA_THREADS;
  if (views) {
    const unsigned char* s = views + (size_t)(ok ? v : 0) * hw * 3;
    float* o = imgs + (size_t)b * 3 * hw;
    for (long long p = t0; p < hw; p += step) {
      float c0 = __int_as_float(0x7fc00000), c1 = c0, c2 = c0;
      if (ok) {
        c0 = u8_to_unit(s[3 * p]);
        c1 = u8_to_unit(s[3 * p + 1]);
        c2 = u8_to_unit(s[3 * p + 2]);
      }
      o[p] = c0;
      o[hw + p] = c1;
      o[2 * (size_t)hw + p] = c2;
    }
  }
#pragma unroll
  for (int f = 0; f < DBW_GATHER_MAX_FIELDS; ++f) {         // unrolled: the parameter struct is never indexed at run time
    if (f >= F.n) break;
    const long long w = F.words[f];
    const uint32_t* s = F.src[f] + (size_t)(ok ? v : 0) * w;
    uint32_t* o = F.dst[f] + (size_t)b * w;
    for (long long p = t0; p < w; p += step) o[p] = ok ? s[p] : 0x7fc00000u;
  }
}

extern "C" int dbw_gather_views(int32_t n_views, int32_t batch, const int64_t* idx, const uint8_t* views, int32_t height, int32_t width,
                                float* imgs, const DbwGatherField* fields, int32_t n_fields, void* stream) {
  if (!idx || n_views < 1 || batch < 1 || batch > 65535) return dbw_fail_("dbw_gather_views: bad index buffer or batch", cudaSuccess);
  if (n_fields < 0 || n_fields > DBW_GATHER_MAX_FIELDS || (n_fields > 0 && !fields))
    return dbw_fail_("dbw_gather_views: bad field table", cudaSuccess);
  if (views && (!imgs || height < 1 || width < 1 || (long long)height * width > INT32_MAX / 3))
    return dbw_fail_("dbw_gather_views: bad image arguments", cudaSuccess);
  if (!views && n_fields == 0) return dbw_fail_("dbw_gather_views: nothing to gather", cudaSuccess);
  GatherFields F{};
  F.n = n_fields;
  long long most = views ? (long long)height * width : 0;
  for (int f = 0; f < n_fields; ++f) {
    if (!fields[f].src || !fields[f].dst || fields[f].words_per_view < 1)
      return dbw_fail_("dbw_gather_views: a field has no buffer or no words", cudaSuccess);
    F.src[f] = (const uint32_t*)fields[f].src;
    F.dst[f] = (uint32_t*)fields[f].dst;
    F.words[f] = fields[f].words_per_view;
    if (F.words[f] > most) most = F.words[f];
  }
  long long ctas = (most + DATA_THREADS - 1) / DATA_THREADS;
  if (ctas > 1024) ctas = 1024;
  gather_views_kernel<<<dim3((unsigned)ctas, (unsigned)batch), DATA_THREADS, 0, (cudaStream_t)stream>>>(
      idx, n_views, views, views ? height * width : 0, imgs, F);
  dbw_count_launch_();
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("gather_views_kernel", e);
}

// ------------------------------------------------------------------ subsample_points
// CTA row blockIdx.y = batch entry b; thread j copies point perm(j) of the cloud, `row_words` 32-bit words, to out[b, j].
// An index outside [0, n_views) writes NaN words.
__global__ void __launch_bounds__(DATA_THREADS)
subsample_points_kernel(const uint32_t* __restrict__ points, long long P, int h, int row_words, const int64_t* __restrict__ idx,
                        int n_views, unsigned long long seed, unsigned long long step, long long n_out, uint32_t* __restrict__ out) {
  const long long j = (long long)blockIdx.x * DATA_THREADS + threadIdx.x;
  if (j >= n_out) return;
  const int b = blockIdx.y;
  const int64_t v = idx[b];
  uint32_t* o = out + ((size_t)b * n_out + j) * row_words;
  if (v < 0 || v >= n_views) {
    for (int w = 0; w < row_words; ++w) o[w] = 0x7fc00000u;
    return;
  }
  const uint64_t src = perm_index((uint64_t)j, (uint64_t)P, h, perm_key(seed, step, (uint64_t)v));
  const uint32_t* s = points + src * row_words;
  for (int w = 0; w < row_words; ++w) o[w] = s[w];
}

extern "C" int dbw_subsample_points(int64_t n_points, int32_t row_words, const void* points, int32_t n_views, int32_t batch,
                                    const int64_t* idx, uint64_t seed, uint64_t step, int64_t n_out, void* out, void* stream) {
  if (!points || !idx || !out || n_points < 1 || n_points > (1ll << 48) || row_words < 1 || n_views < 1)
    return dbw_fail_("dbw_subsample_points: null buffer or empty cloud", cudaSuccess);
  if (batch < 1 || batch > 65535 || n_out < 1 || n_out > n_points)
    return dbw_fail_("dbw_subsample_points: batch must be in [1, 65535] and n_out in [1, n_points]", cudaSuccess);
  const long long ctas = (n_out + DATA_THREADS - 1) / DATA_THREADS;
  if (ctas > INT32_MAX) return dbw_fail_("dbw_subsample_points: n_out too large", cudaSuccess);
  subsample_points_kernel<<<dim3((unsigned)ctas, (unsigned)batch), DATA_THREADS, 0, (cudaStream_t)stream>>>(
      (const uint32_t*)points, n_points, perm_half_bits((uint64_t)n_points), row_words, idx, n_views, seed, step, n_out,
      (uint32_t*)out);
  dbw_count_launch_();
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : dbw_fail_("subsample_points_kernel", e);
}
