// dbw_optim.cu -- sm_90a Adam over every parameter tensor of the model in ONE launch (see include/dbw_render.h, "Optimiser").
//
// The tensors ("segments", at most DBW_ADAM_MAX_SEGMENTS) are cut into chunks of four consecutive elements; the chunks of
// all active segments form one index space that the grid strides over.  Every CTA builds the same table in shared memory
// -- the segment records, each segment's first chunk, its per-step coefficients (bias corrections in double from the
// device counter) -- and a thread finds the segment of its chunk by bisection over the at most 64 first-chunk entries.
// A chunk is moved as float4 where the segment's parameter and moments are 16-byte aligned (the gradient, which may be an
// odd-offset view of the gradient bucket, falls back to four scalar loads on its own); a segment's tail and unaligned
// segments go element by element.  28 bytes of traffic per element, no arithmetic to speak of: bandwidth-bound.
//
// The step counters are advanced by the kernel itself.  Every CTA reads them before it touches anything else; when a CTA is
// done it adds one to an arrival count kept in bits 40.. of step[0], and the CTA that arrives last removes the count and
// increments the counters of the active segments -- no CTA can still be about to read them.  The count lives in the
// caller's buffer, so concurrent updates of different optimisers on different streams do not share state.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dbw_render.h"
#include "dbw_optim_math.cuh"

extern int dbw_fail_(const char* what, cudaError_t e);
extern void dbw_count_launch_(void);

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_MAX_CTAS = 8 * 132;                      // 8 CTAs of 256 threads on each of the H100's 132 SMs
constexpr int ADAM_ARRIVAL_SHIFT = 40;                      // step values stay below 2^40
constexpr unsigned long long ADAM_STEP_MASK = (1ull << ADAM_ARRIVAL_SHIFT) - 1;

struct AdamGroups { DbwAdamGroup g[DBW_ADAM_MAX_GROUPS]; };

__device__ __forceinline__ bool adam_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__global__ void __launch_bounds__(ADAM_THREADS)
adam_step_kernel(const DbwAdamSegment* __restrict__ segments, int n_segments, AdamGroups groups, int n_groups,
                 const float* __restrict__ lr, unsigned long long* __restrict__ step) {
  __shared__ DbwAdamSegment s_seg[DBW_ADAM_MAX_SEGMENTS];
  __shared__ DbwAdamCoef s_coef[DBW_ADAM_MAX_SEGMENTS];
  __shared__ long long s_first[DBW_ADAM_MAX_SEGMENTS + 1];  // first chunk of each segment; [n_segments] = all chunks
  __shared__ int s_vec[DBW_ADAM_MAX_SEGMENTS];              // bit 0: param and moments 16-byte aligned; bit 1: the gradient too
  const int tid = threadIdx.x;
  if (tid < n_segments) {
    DbwAdamSegment sg = segments[tid];
    if (sg.group < 0 || sg.group >= n_groups || sg.n <= 0 || !sg.param || !sg.grad || !sg.exp_avg || !sg.exp_avg_sq) sg.active = 0;
    s_seg[tid] = sg;
    if (sg.active) {
      const DbwAdamGroup g = groups.g[sg.group];
      const int64_t t = (int64_t)(step[tid] & ADAM_STEP_MASK) + 1;
      s_coef[tid] = dbw_adam_coef(g.beta1, g.beta2, g.eps, g.weight_decay, lr[sg.group], t);
      s_vec[tid] = (adam_aligned16(sg.param) && adam_aligned16(sg.exp_avg) && adam_aligned16(sg.exp_avg_sq) ? 1 : 0) |
                   (adam_aligned16(sg.grad) ? 2 : 0);
    }
  }
  __syncthreads();
  if (tid == 0) {
    long long c = 0;
    for (int s = 0; s < n_segments; ++s) {
      s_first[s] = c;
      if (s_seg[s].active) c += (s_seg[s].n + 3) >> 2;
    }
    s_first[n_segments] = c;
  }
  __syncthreads();

  const long long n_chunks = s_first[n_segments];
  for (long long chunk = (long long)blockIdx.x * ADAM_THREADS + tid; chunk < n_chunks; chunk += (long long)gridDim.x * ADAM_THREADS) {
    int lo = 0, hi = n_segments;                            // the last segment whose first chunk is <= chunk (empty ones sort before it)
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (s_first[mid] <= chunk) lo = mid; else hi = mid;
    }
    const DbwAdamSegment& sg = s_seg[lo];
    const DbwAdamCoef& c = s_coef[lo];
    const int64_t e = (chunk - s_first[lo]) << 2;
    const int vec = s_vec[lo];
    if ((vec & 1) && e + 4 <= sg.n) {
      float4 p = *reinterpret_cast<const float4*>(sg.param + e);
      float4 m = *reinterpret_cast<const float4*>(sg.exp_avg + e);
      float4 v = *reinterpret_cast<const float4*>(sg.exp_avg_sq + e);
      float4 g;
      if (vec & 2) g = __ldg(reinterpret_cast<const float4*>(sg.grad + e));
      else g = make_float4(__ldg(sg.grad + e), __ldg(sg.grad + e + 1), __ldg(sg.grad + e + 2), __ldg(sg.grad + e + 3));
      dbw_adam_update(c, g.x, p.x, m.x, v.x);
      dbw_adam_update(c, g.y, p.y, m.y, v.y);
      dbw_adam_update(c, g.z, p.z, m.z, v.z);
      dbw_adam_update(c, g.w, p.w, m.w, v.w);
      *reinterpret_cast<float4*>(sg.param + e) = p;
      *reinterpret_cast<float4*>(sg.exp_avg + e) = m;
      *reinterpret_cast<float4*>(sg.exp_avg_sq + e) = v;
    } else {
      const int64_t end = (e + 4 < sg.n) ? e + 4 : sg.n;
      for (int64_t i = e; i < end; ++i) {
        float p = sg.param[i], m = sg.exp_avg[i], v = sg.exp_avg_sq[i];
        dbw_adam_update(c, __ldg(sg.grad + i), p, m, v);
        sg.param[i] = p; sg.exp_avg[i] = m; sg.exp_avg_sq[i] = v;
      }
    }
  }

  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const unsigned long long arrived = atomicAdd(step, 1ull << ADAM_ARRIVAL_SHIFT) >> ADAM_ARRIVAL_SHIFT;
    if (arrived == gridDim.x - 1) {                         // the last CTA: every other one has read its counters
      atomicAdd(step, 0ull - ((unsigned long long)gridDim.x << ADAM_ARRIVAL_SHIFT));
      for (int s = 0; s < n_segments; ++s)
        if (s_seg[s].active) step[s] += 1;
    }
  }
}

extern "C" int dbw_adam_step(const DbwAdamSegment* segments, int32_t n_segments, int64_t n_total, const DbwAdamGroup* groups,
                             int32_t n_groups, const float* lr, int64_t* step, void* stream) {
  if (n_segments < 1 || n_segments > DBW_ADAM_MAX_SEGMENTS || n_groups < 1 || n_groups > DBW_ADAM_MAX_GROUPS || n_total <= 0)
    return dbw_fail_("dbw_adam_step: bad sizes (1 <= n_segments <= DBW_ADAM_MAX_SEGMENTS, 1 <= n_groups <= DBW_ADAM_MAX_GROUPS, "
                     "n_total > 0)", cudaSuccess);
  if (!segments || !groups || !lr || !step) return dbw_fail_("dbw_adam_step: null pointer argument", cudaSuccess);
  AdamGroups by_value;
  for (int g = 0; g < DBW_ADAM_MAX_GROUPS; ++g) by_value.g[g] = groups[g < n_groups ? g : 0];
  const int64_t chunks = (n_total >> 2) + n_segments;       // at most one partial chunk per segment
  const int64_t want = (chunks + ADAM_THREADS - 1) / ADAM_THREADS;
  const int grid = (int)(want < ADAM_MAX_CTAS ? want : ADAM_MAX_CTAS);
  adam_step_kernel<<<grid, ADAM_THREADS, 0, (cudaStream_t)stream>>>(segments, n_segments, by_value, n_groups, lr,
                                                                    reinterpret_cast<unsigned long long*>(step));
  dbw_count_launch_();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return dbw_fail_("adam_step_kernel", e);
  return 0;
}
