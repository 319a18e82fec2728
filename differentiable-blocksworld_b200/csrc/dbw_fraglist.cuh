// dbw_fraglist.cuh -- the K nearest fragments of one pixel as a SORTED LIST IN SHARED MEMORY (raster_forward_kernel).
//
// Round 1 kept the list in registers (64-bit keys, fully unrolled sorted insertion: ~110 instructions per insertion and
// 3K registers per thread, which capped the K=10 kernel at 38 % occupancy and made K=25 spill).  The list now lives in
// shared memory, one column per thread (entry k of thread t at index k*NT + t: conflict-free), sorted on insertion; an
// insertion is one 128-bit + one 32-bit shared load/store pair per shifted entry, the register cost is the entry count.
// Each entry carries everything shading needs -- no geometry is re-derived for the kept fragments:
//     A[k] = (pz, bits, signed squared distance, u)      V[k] = v
//     bits = triangle slot (20 bits) | closest edge (2 bits: 0 = v0v1, 1 = v0v2, 2 = v1v2) << 20 | outside (sd >= 0) << 22
//            | texture map of the face (9 bits) << 23
// Order = (depth, slot): the tuple order of PyTorch3D's CPU rasterizer queue (depth, then face index in the clipped mesh;
// SURVEY.md Appendix A5) up to the exact depth ties named at frag_key_less; the two halves of a z-clipped quad exclude each
// other (Appendix A3).
//
// The result depends on the order in which a pixel's candidates are OFFERED, through the quad rule alone: a half only
// yields to, or evicts, its other half while that one is in the list, and a half that was rejected or evicted earlier no
// longer excludes it (K = 1, halves A and B, a face C with pz_A < pz_C < pz_B and dist_B < |d_A|: offered A, B, C the list
// ends with C; C, A, B: with B; B, C, A: with A).  The reference offers faces in the clipped mesh's index order, where a
// quad's two halves are adjacent; the kernel's slots put the second half of face f at F + f.  So every view with z-clipped
// slots offers them in frag_order_key order, which is that index order: raster_forward_kernel sorts its tile list by it
// (frag_order_rank) or scans its slots in it (frag_order_slot, coarse_bin_kernel), and compacts in order.  Views without
// z-clipped slots cannot depend on the order and skip the sort and the ordered bin compaction.
//
// Plain C++ apart from the __device__ markers: tests/host_math compiles it for the CPU and checks it against the oracle's
// queue under every offer order.
#pragma once
#include "dbw_math.cuh"

#define DBW_FRAG_SLOT_MASK 0x000fffff
#define DBW_FRAG_EDGE_SHIFT 20
#define DBW_FRAG_OUTSIDE_BIT (1 << 22)
#define DBW_FRAG_MAP_SHIFT 23
#define DBW_FRAG_MAX_MAPS 512

// Position of slot s of a view with F faces in the clipped mesh's face order: face s's first triangle (s < F), or the
// second triangle of face s - F right after it.  Strictly monotone in the clipped index (culled faces only leave gaps).
__device__ __forceinline__ int frag_order_key(int slot, int F) { return slot < F ? 2 * slot : 2 * (slot - F) + 1; }

// The slot at position i of that order (inverse of frag_order_key over the 2F slots of a view)
__device__ __forceinline__ int frag_order_slot(int i, int F) { return (i & 1) ? F + (i >> 1) : i >> 1; }

// Where entry j of n distinct listed slots goes when the list is sorted by frag_order_key: the number of entries before it
__device__ __forceinline__ int frag_order_rank(const int* slots, int n, int j, int F) {
  const int kj = frag_order_key(slots[j], F);
  int r = 0;
  for (int i = 0; i < n; ++i) r += frag_order_key(slots[i], F) < kj ? 1 : 0;
  return r;
}

// (pz, slot) < key of entry e ?   depths are >= 0, so their bit patterns order like the values.  Exact depth ties go by slot,
// which is the clipped index order except between the second half of a quad (slot F + f) and a face g > f.  Such a tie needs
// a clipped triangle, whose clipped vertex is interpolated, and another face to give bit-equal depths at a pixel centre; the
// (F-dependent) clipped-order comparison here cost 0.8 % of the dtu step, so ties keep the slot order.
__device__ __forceinline__ bool frag_key_less(unsigned pz_bits, int slot, float4 e) {
  const unsigned eb = __float_as_uint(e.x);
  return pz_bits < eb || (pz_bits == eb && slot < (__float_as_int(e.y) & DBW_FRAG_SLOT_MASK));
}

// Offer one candidate to the list of `n` entries (capacity K); returns the new entry count.
// A / V point at THIS thread's column; consecutive entries are `stride` elements apart.
__device__ __forceinline__ int fraglist_offer(float4* A, float* V, int stride, int n, int K, float pz, int slot, int edge,
                                              float sd, float dist, int neighbor, float u, float v, int map_id = 0) {
  const unsigned pzb = __float_as_uint(pz + 0.f);
  if (neighbor >= 0) {
    // the other half of a z-clipped quad: only the half with the smaller |dist| may stay (A3)
    for (int i = 0; i < n; ++i) {
      const float4 e = A[i * stride];
      if ((__float_as_int(e.y) & DBW_FRAG_SLOT_MASK) != neighbor) continue;
      if (!(dist < fabsf(e.z))) return n;
      for (int q = i; q < n - 1; ++q) { A[q * stride] = A[(q + 1) * stride]; V[q * stride] = V[(q + 1) * stride]; }
      --n;
      break;
    }
  }
  if (n == K) {
    if (!frag_key_less(pzb, slot, A[(K - 1) * stride])) return n;
    n = K - 1;                                   // the farthest entry is dropped
  }
  int i = n;
  while (i > 0) {
    const float4 e = A[(i - 1) * stride];
    if (!frag_key_less(pzb, slot, e)) break;
    A[i * stride] = e; V[i * stride] = V[(i - 1) * stride];
    --i;
  }
  A[i * stride] = make_float4(pz, __int_as_float(slot | (edge << DBW_FRAG_EDGE_SHIFT) | (sd < 0.f ? 0 : DBW_FRAG_OUTSIDE_BIT) |
                                                 (map_id << DBW_FRAG_MAP_SHIFT)), sd, u);
  V[i * stride] = v;
  return n + 1;
}
