// dbw_comm.cu -- the step's ONE gradient exchange (SURVEY.md 8e) as a hand-written all-reduce over NVLink / NVSwitch
// peer memory: a plain kernel (no NCCL, no host synchronisation), so that it is captured INSIDE the step's CUDA graph --
// an ncclAllReduce has to be issued after the graph replay instead (capturing it hung).
//
// One process per GPU.  Every rank owns an arena (cudaMalloc, exported with cudaIpcGetMemHandle, opened by its peers):
//     control:  flagsA[world], flagsB[world] (written BY the peers), epoch, grid-barrier counters
//     flat      the gradient bucket itself (dbw_comm_buffer: the caller's tensors live HERE, nothing is staged)
//     inbox     world slices: the addends the peers push for the slice of the sum this rank owns
// all_reduce(n) is a PUSH protocol -- every remote access is a posted store, no rank ever waits for a load over NVLink:
//     scatter   element i of my bucket goes to inbox[my rank] of its owner (owner = i / slice); my own slice stays local
//     barrier A (every rank's pushes have landed)
//     reduce    the owner adds its world inbox slices in rank order and stores the sum into EVERY rank's bucket
//     barrier B (every rank's results have landed)
// Every sum is formed once, by its owner, in rank order: the result is bit-identical on all ranks.  Hazards: a peer writes
// results into my bucket only after barrier A, which I pass only after my scatter has read it; my next scatter writes the
// peers' inboxes only after barrier B of this epoch, which an owner signals after its reduce has read them.
// Barriers are epoch-stamped flags stored into the PEERS' arenas with st.release.sys and polled locally with
// ld.acquire.sys; a poll that exceeds ~30 s sets the arena's error word instead of hanging the GPU.
//
// Small exchanges (<= ONE_SHOT_BYTES: the step's scene-tensor gradients, parallel.GradSumPoint, ~0.15 MB) are latency bound and
// take the FLAGGED ONE-SHOT path, no barrier at all: every rank pushes its whole vector into its slot of EVERY rank's `ll` region
// as 64-bit words {value, epoch} (one posted store each: value and flag arrive together), then adds the world copies itself,
// in rank order (bit-identical again), spinning per word until its flag shows this epoch -- one NVLink one-way trip.  A rank
// stamps "I have finished reading" (flagsB) without waiting, and every exchange (either path) starts by checking the peers'
// stamps of the previous one, long since there: that is what keeps a fast rank from overwriting words a slow one still reads.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/dbw_render.h"

int dbw_fail_(const char* what, cudaError_t e);
void dbw_count_launch_(void);
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return dbw_fail_(#call, _e); } while (0)

#define COMM_MAX_WORLD 8
#define COMM_BLOCKS 96
#define COMM_SMALL_BLOCKS 16
#define COMM_THREADS 512
#define ONE_SHOT_BYTES (512 * 1024)
#define CTRL_BYTES 4096

struct CommDev {
  int world, rank;
  unsigned* ctrl[COMM_MAX_WORLD];        // each rank's control block: [0,world) flagsA, [64, 64+world) flagsB
  float* flat[COMM_MAX_WORLD];           // each rank's bucket
  float* inbox[COMM_MAX_WORLD];          // each rank's inbox: world slices of slice_floats
  unsigned long long* ll[COMM_MAX_WORLD];  // each rank's flagged one-shot region: world slots of LL_CAP_FLOATS {value, epoch} words
  size_t cap_floats, slice_floats;
};
#define LL_CAP_FLOATS (ONE_SHOT_BYTES / 4)
// local control words (indices into ctrl[rank]): 128 epoch, 129 grid-barrier arrivals, 130 barrier base, 131 error
#define CW_FLAGS_A 0
#define CW_FLAGS_B 64
#define CW_EPOCH 128
#define CW_ARRIVE 129
#define CW_BASE 130
#define CW_ERROR 131

struct Comm {
  CommDev d;
  void* arena;
  void* peer_base[COMM_MAX_WORLD];
  size_t arena_bytes;
  bool connected;
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ float4 ld_peer(const float4* p) {          // peer memory is never served from a stale L1 line
  float4 v; asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory"); return v;
}

#define SPIN_LIMIT (60000000000ll)       // ~30 s of SM clocks: ranks may reach their first exchange seconds apart (start-up skew)

// barrier over the blocks of THIS kernel (all co-resident: COMM_BLOCKS <= SMs)
__device__ __forceinline__ void grid_barrier(unsigned* ctl, unsigned target) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(&ctl[CW_ARRIVE], 1u);
    const long long t0 = clock64();
    while (ld_acquire_gpu(&ctl[CW_ARRIVE]) < target) if (clock64() - t0 > SPIN_LIMIT) { ctl[CW_ERROR] = 1u; break; }
  }
  __syncthreads();
}

// barrier over the ranks: block 0 stamps `epoch` into flag word `which + rank` of every peer and waits for every peer's stamp
__device__ __forceinline__ void rank_barrier(const CommDev& c, unsigned* ctl, int which, unsigned epoch) {
  if (blockIdx.x == 0 && threadIdx.x < c.world) {
    const int p = threadIdx.x;
    st_release_sys(c.ctrl[p] + which + c.rank, epoch);
    const long long t0 = clock64();
    while (ld_acquire_sys(ctl + which + p) < epoch) if (clock64() - t0 > SPIN_LIMIT) { ctl[CW_ERROR] = 2u; break; }
  }
}

// deferred barrier B of the PREVIOUS exchange: every peer has finished reading the inbox this one is about to overwrite
__device__ __forceinline__ void wait_previous_exchange(const CommDev& c, unsigned* ctl, unsigned prev_epoch) {
  if (threadIdx.x < c.world) {
    const long long t0 = clock64();
    while (ld_acquire_sys(ctl + CW_FLAGS_B + threadIdx.x) < prev_epoch) if (clock64() - t0 > SPIN_LIMIT) { ctl[CW_ERROR] = 3u; break; }
  }
  __syncthreads();
}

__device__ __forceinline__ void st_peer(float4* p, float4 v) {       // posted store into a peer's arena
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

template <int W>
__global__ void __launch_bounds__(COMM_THREADS) all_reduce_kernel(const CommDev c, float* __restrict__ buf, size_t n4) {
  unsigned* ctl = c.ctrl[c.rank];
  const unsigned epoch = ctl[CW_EPOCH] + 1u, base = ctl[CW_BASE];     // stable until block 0 advances them after barrier A
  const int G = gridDim.x, r = c.rank;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)G * blockDim.x;
  const float4* src = reinterpret_cast<const float4*>(buf);
  const size_t slice = (n4 + W - 1) / W;                              // float4 elements per owner
  const size_t cap4 = c.slice_floats / 4;                             // inbox stride between the ranks' slices
  wait_previous_exchange(c, ctl, epoch - 1u);
  // ---- scatter: push every element to its owner's inbox (my own slice: a local copy)
  for (size_t i0 = tid; i0 < n4; i0 += 4 * nthr) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) { const size_t i = i0 + (size_t)u * nthr; if (i < n4) v[u] = src[i]; }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const size_t i = i0 + (size_t)u * nthr;
      if (i < n4) {
        const int owner = (int)(i / slice);
        st_peer(reinterpret_cast<float4*>(c.inbox[owner]) + (size_t)r * cap4 + (i - (size_t)owner * slice), v[u]);
      }
    }
  }
  grid_barrier(ctl, base + 1u * G);
  rank_barrier(c, ctl, CW_FLAGS_A, epoch);                            // A: every rank's pushes into my inbox have landed
  grid_barrier(ctl, base + 2u * G);
  if (blockIdx.x == 0 && threadIdx.x == 0) { ctl[CW_EPOCH] = epoch; ctl[CW_BASE] = base + 3u * G; }
  // ---- reduce my slice in rank order, broadcast the sums into every rank's bucket
  const size_t lo = (size_t)r * slice, hi = lo + slice < n4 ? lo + slice : n4;
  const float4* in = reinterpret_cast<const float4*>(c.inbox[r]);
  for (size_t i = lo + tid; i < hi; i += nthr) {
    float4 v[W];
#pragma unroll
    for (int q = 0; q < W; ++q) v[q] = ld_peer(in + (size_t)q * cap4 + (i - lo));      // local memory, written remotely: not via L1
    float4 acc = v[0];
#pragma unroll
    for (int q = 1; q < W; ++q) { acc.x += v[q].x; acc.y += v[q].y; acc.z += v[q].z; acc.w += v[q].w; }
#pragma unroll
    for (int q = 0; q < W; ++q) st_peer(reinterpret_cast<float4*>(c.flat[(r + q) % W]) + i, acc);
  }
  grid_barrier(ctl, base + 3u * G);
  rank_barrier(c, ctl, CW_FLAGS_B, epoch);                            // B: every owner's sums have landed in my bucket
}

// flagged one-shot variant for small vectors (n <= LL_CAP_FLOATS): see the header
template <int W>
__global__ void __launch_bounds__(COMM_THREADS) all_reduce_small_kernel(const CommDev c, float* __restrict__ buf, size_t n) {
  unsigned* ctl = c.ctrl[c.rank];
  const unsigned epoch = ctl[CW_EPOCH] + 1u, base = ctl[CW_BASE];     // stable until the LAST block of this kernel advances them
  const int G = gridDim.x, r = c.rank;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)G * blockDim.x;
  wait_previous_exchange(c, ctl, epoch - 1u);
  // ---- push {value, epoch} into slot `r` of every rank's region
  for (size_t i = tid; i < n; i += nthr) {
    const unsigned long long w = ((unsigned long long)epoch << 32) | (unsigned long long)__float_as_uint(buf[i]);
#pragma unroll
    for (int q = 0; q < W; ++q) {
      unsigned long long* dst = c.ll[(r + q) % W] + (size_t)r * LL_CAP_FLOATS + i;
      asm volatile("st.volatile.global.u64 [%0], %1;" :: "l"(dst), "l"(w) : "memory");
    }
  }
  // ---- every rank forms every sum itself, in rank order, as the words arrive
  const unsigned long long* in = c.ll[r];
  bool late = false;
  for (size_t i = tid; i < n; i += nthr) {
    float acc = 0.f;
#pragma unroll
    for (int q = 0; q < W; ++q) {
      const unsigned long long* src = in + (size_t)q * LL_CAP_FLOATS + i;
      unsigned long long w;
      const long long t0 = clock64();
      for (;;) {
        asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(w) : "l"(src) : "memory");
        if ((unsigned)(w >> 32) == epoch) break;
        if (clock64() - t0 > SPIN_LIMIT) { late = true; break; }
      }
      const float v = __uint_as_float((unsigned)w);
      acc = q == 0 ? v : acc + v;
    }
    buf[i] = acc;
  }
  if (late) ctl[CW_ERROR] = 2u;
  // ---- the last block to finish advances the epoch and tells the peers this rank's region may be overwritten (not waited for)
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&ctl[CW_ARRIVE], 1u) + 1u == base + (unsigned)G;
  __syncthreads();
  if (s_last) {
    if (threadIdx.x == 0) { ctl[CW_EPOCH] = epoch; ctl[CW_BASE] = base + (unsigned)G; }
    if (threadIdx.x < c.world) st_release_sys(c.ctrl[threadIdx.x] + CW_FLAGS_B + r, epoch);
  }
}

static size_t arena_layout(size_t cap_floats, size_t world, size_t* off_flat, size_t* off_inbox, size_t* slice_floats,
                           size_t* off_ll = nullptr) {
  const size_t cap = (cap_floats + 3) / 4 * 4;
  const size_t slice = ((cap / 4 + world - 1) / world) * 4;
  *off_flat = CTRL_BYTES; *off_inbox = CTRL_BYTES + cap * sizeof(float); *slice_floats = slice;
  const size_t ll = (*off_inbox + world * slice * sizeof(float) + 255) / 256 * 256;
  if (off_ll) *off_ll = ll;
  return ll + world * (size_t)LL_CAP_FLOATS * sizeof(unsigned long long);
}

extern "C" int dbw_comm_create(int32_t world, int32_t rank, size_t max_floats, void** comm_out) {
  if (!comm_out || world < 1 || world > COMM_MAX_WORLD || rank < 0 || rank >= world || max_floats == 0)
    return dbw_fail_("dbw_comm_create: bad arguments (1 <= world <= 8, 0 <= rank < world, max_floats > 0)", cudaSuccess);
  Comm* c = new Comm();
  memset(c, 0, sizeof(Comm));
  c->d.world = world; c->d.rank = rank; c->d.cap_floats = (max_floats + 3) / 4 * 4;
  size_t od, orr, sl;
  c->arena_bytes = arena_layout(max_floats, world, &od, &orr, &sl);
  cudaError_t e = cudaMalloc(&c->arena, c->arena_bytes);
  if (e != cudaSuccess) { delete c; return dbw_fail_("dbw_comm_create: cudaMalloc", e); }
  e = cudaMemset(c->arena, 0, c->arena_bytes);
  if (e != cudaSuccess) { cudaFree(c->arena); delete c; return dbw_fail_("dbw_comm_create: cudaMemset", e); }
  CK(cudaDeviceSynchronize());
  *comm_out = c;
  return 0;
}

extern "C" int dbw_comm_ipc_handle(void* comm, void* out_handle64) {
  Comm* c = (Comm*)comm;
  if (!c || !out_handle64) return dbw_fail_("dbw_comm_ipc_handle: null argument", cudaSuccess);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, c->arena));
  memcpy(out_handle64, &h, 64);
  return 0;
}

extern "C" int dbw_comm_connect(void* comm, const void* all_handles) {
  Comm* c = (Comm*)comm;
  if (!c || !all_handles) return dbw_fail_("dbw_comm_connect: null argument", cudaSuccess);
  size_t od, orr, sl, oll;
  arena_layout(c->d.cap_floats, c->d.world, &od, &orr, &sl, &oll);
  for (int p = 0; p < c->d.world; ++p) {
    void* base = c->arena;
    if (p != c->d.rank) {
      cudaIpcMemHandle_t h;
      memcpy(&h, (const char*)all_handles + (size_t)p * 64, 64);
      CK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    }
    c->peer_base[p] = base;
    char* b = (char*)base;
    c->d.ctrl[p] = (unsigned*)b;
    c->d.flat[p] = (float*)(b + od);
    c->d.inbox[p] = (float*)(b + orr);
    c->d.ll[p] = (unsigned long long*)(b + oll);
  }
  c->d.slice_floats = sl;
  c->connected = true;
  return 0;
}

extern "C" int dbw_comm_buffer(void* comm, float** out) {
  Comm* c = (Comm*)comm;
  if (!c || !out) return dbw_fail_("dbw_comm_buffer: null argument", cudaSuccess);
  size_t od, orr, sl;
  arena_layout(c->d.cap_floats, c->d.world, &od, &orr, &sl);
  *out = (float*)((char*)c->arena + od);
  return 0;
}

extern "C" int dbw_comm_all_reduce(void* comm, float* buf, size_t n_floats, void* stream) {
  Comm* c = (Comm*)comm;
  if (!c || !buf) return dbw_fail_("dbw_comm_all_reduce: null argument", cudaSuccess);
  if (c->connected && buf != c->d.flat[c->d.rank]) return dbw_fail_("dbw_comm_all_reduce: buf must be the arena's bucket (dbw_comm_buffer)", cudaSuccess);
  if (!c->connected) return dbw_fail_("dbw_comm_all_reduce: dbw_comm_connect has not run", cudaSuccess);
  if (n_floats % 4 || n_floats > c->d.cap_floats) return dbw_fail_("dbw_comm_all_reduce: n_floats must be a multiple of 4 and <= the capacity", cudaSuccess);
  if (((uintptr_t)buf) % 16) return dbw_fail_("dbw_comm_all_reduce: buf must be 16-byte aligned", cudaSuccess);
  if (c->d.world == 1 || n_floats == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n4 = n_floats / 4;
  if (n_floats <= LL_CAP_FLOATS) {
    switch (c->d.world) {
      case 2: all_reduce_small_kernel<2><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 3: all_reduce_small_kernel<3><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 4: all_reduce_small_kernel<4><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 5: all_reduce_small_kernel<5><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 6: all_reduce_small_kernel<6><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 7: all_reduce_small_kernel<7><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      case 8: all_reduce_small_kernel<8><<<COMM_SMALL_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n_floats); break;
      default: return dbw_fail_("dbw_comm_all_reduce: world sizes 2..8 are compiled in (one NVSwitch node)", cudaSuccess);
    }
    dbw_count_launch_();
    cudaError_t e1 = cudaGetLastError();
    if (e1 != cudaSuccess) return dbw_fail_("all_reduce_small_kernel", e1);
    return 0;
  }
  switch (c->d.world) {
    case 2: all_reduce_kernel<2><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 3: all_reduce_kernel<3><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 4: all_reduce_kernel<4><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 5: all_reduce_kernel<5><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 6: all_reduce_kernel<6><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 7: all_reduce_kernel<7><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    case 8: all_reduce_kernel<8><<<COMM_BLOCKS, COMM_THREADS, 0, st>>>(c->d, buf, n4); break;
    default: return dbw_fail_("dbw_comm_all_reduce: world sizes 2..8 are compiled in (one NVSwitch node)", cudaSuccess);
  }
  dbw_count_launch_();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return dbw_fail_("all_reduce_kernel", e);
  return 0;
}

// 0: fine; 1 / 2 / 3: a grid barrier / rank barrier / the wait for the previous exchange timed out (a peer did not arrive within ~30 s) -- results are then garbage
extern "C" int dbw_comm_error(void* comm, int32_t* out) {
  Comm* c = (Comm*)comm;
  if (!c || !out) return dbw_fail_("dbw_comm_error: null argument", cudaSuccess);
  unsigned v = 0;
  CK(cudaMemcpy(&v, (unsigned*)c->arena + CW_ERROR, sizeof(unsigned), cudaMemcpyDeviceToHost));
  *out = (int32_t)v;
  return 0;
}

extern "C" int dbw_comm_destroy(void* comm) {
  Comm* c = (Comm*)comm;
  if (!c) return 0;
  cudaDeviceSynchronize();
  if (c->connected)
    for (int p = 0; p < c->d.world; ++p) if (p != c->d.rank && c->peer_base[p]) cudaIpcCloseMemHandle(c->peer_base[p]);
  cudaFree(c->arena);
  delete c;
  return 0;
}
