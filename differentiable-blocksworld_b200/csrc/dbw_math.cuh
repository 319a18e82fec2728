// dbw_math.cuh -- per-(pixel, face) math shared by the forward and backward rasterization kernels.
//
// The operation order follows PyTorch3D 0.7.1's geometry_utils (SURVEY.md Appendix A4/A6), which is what the
// reference's MeshRasterizer executes (src/model/renderer.py:50-54).  Arithmetic that feeds a DISCRETE decision
// (edge-function signs -> inside test, pixel NDC coordinates) is written with non-contracting intrinsics so that it
// is bit-identical to an IEEE-754 evaluation without FMA; everything else may be contracted by the compiler.
// The header also compiles as plain C++ (tests/host_math: the same functions checked against the oracle on the CPU);
// the parts that only exist on the device (PTX: TMA, mbarrier, vector RED) are fenced with __CUDACC__.
#pragma once
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#define DBW_KEPS 1e-8f

struct f2 { float x, y; };
struct f3 { float x, y, z; };

__device__ __forceinline__ float edge_nc(f2 p, f2 a, f2 b) {
  // (p.x-a.x)*(b.y-a.y) - (p.y-a.y)*(b.x-a.x), no FMA contraction
  return __fsub_rn(__fmul_rn(p.x - a.x, b.y - a.y), __fmul_rn(p.y - a.y, b.x - a.x));
}

// rasterization_utils: PixToNonSquareNdc (SURVEY A2), bit-identical to the non-contracted evaluation
__device__ __forceinline__ float pix_to_ndc(int i, int S1, int S2) {
  float range = 2.0f;
  if (S1 > S2) range = __fdiv_rn(__fmul_rn((float)S1, range), (float)S2);
  const float offset = __fdiv_rn(range, 2.0f);
  return __fadd_rn(-offset, __fdiv_rn(__fadd_rn(__fmul_rn(range, (float)i), offset), (float)S1));
}

#ifdef __CUDACC__
// ------------------------------------------------------------------ TMA (bulk async copy) + mbarrier helpers (sm_90+)
// The per-tile face records are gathered global -> shared with cp.async.bulk (SASS: UBLKCP), one 64 B bulk copy per listed
// face, all completing on one shared-memory mbarrier (complete_tx::bytes) -- no register staging, no LDG/STS pairs.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
#endif  // __CUDACC__

// reciprocal of the CONTINUOUS normalisations (perspective correction, barycentric clipping): the 1-ulp MUFU
// approximation, as -prec-div=false (Makefile) makes the plain divisions.  Everything a discrete decision
// depends on (edge functions, pixel coordinates) uses the explicitly rounded intrinsics (__fmul_rn, __fdiv_rn, ...) and is
// not affected by either.  -DDBW_PRECISE_RCP restores the correctly rounded reciprocal.
#ifdef DBW_PRECISE_RCP
#define DBW_RCP(x) __frcp_rn(x)
#else
#define DBW_RCP(x) __fdividef(1.f, (x))
#endif

struct TriGeom {
  f2 v0, v1, v2;
  float z0, z1, z2;
  int face;      // original face id
  int neighbor;  // slot of the other half of a z-clipped quad, or -1
  int flags;     // bit0: clipped (barycentric conversion matrix present)
  float inv_area;            // 1 / (edge(v2; v0, v1) + kEpsilon)
  float il01, il02, il12;    // 1 / |b - a|^2 of the three edges, or -1 when |b - a|^2 <= kEpsilon (degenerate)
};

// record = 4 x float4: [v0xy v1xy] [v2xy z0 z1] [z2 face neighbor flags] [inv_area il01 il02 il12]
__device__ __forceinline__ TriGeom unpack_tri(float4 r0, float4 r1, float4 r2, float4 r3) {
  TriGeom t;
  t.v0 = {r0.x, r0.y}; t.v1 = {r0.z, r0.w}; t.v2 = {r1.x, r1.y};
  t.z0 = r1.z; t.z1 = r1.w; t.z2 = r2.x;
  t.face = __float_as_int(r2.y); t.neighbor = __float_as_int(r2.z); t.flags = __float_as_int(r2.w);
  t.inv_area = r3.x; t.il01 = r3.y; t.il02 = r3.z; t.il12 = r3.w;
  return t;
}

struct Bary {
  f3 b0;    // screen-space barycentrics
  f3 bp;    // perspective-corrected
  f3 bc;    // clipped + renormalised (what is interpolated with)
  bool inside;
  float pz;
};

// The three edge functions (exact, non-contracted) and the inside test.  inside <=> every barycentric > 0
// <=> every edge function has the sign of the (eps-shifted) area; this is the DISCRETE decision and is bit-identical
// to the IEEE evaluation of SURVEY A4 (z > 0 after clipping, so perspective correction keeps the signs).
struct Edges { float e0, e1, e2; bool inside; };
__device__ __forceinline__ Edges eval_edges(f2 p, const TriGeom& t) {
  Edges e;
  e.e0 = edge_nc(p, t.v1, t.v2); e.e1 = edge_nc(p, t.v2, t.v0); e.e2 = edge_nc(p, t.v0, t.v1);
  const float s = t.inv_area;
  e.inside = (e.e0 * s > 0.f) && (e.e1 * s > 0.f) && (e.e2 * s > 0.f);
  return e;
}

__device__ __forceinline__ f3 persp_forward(f3 b, float z0, float z1, float z2) {
  const float t0 = b.x * z1 * z2, t1 = z0 * b.y * z2, t2 = z0 * z1 * b.z;
  const float inv = DBW_RCP(fmaxf(t0 + t1 + t2, DBW_KEPS));     // one reciprocal, no slow-path division
  return {t0 * inv, t1 * inv, t2 * inv};
}

__device__ __forceinline__ f3 clip_forward(f3 b) {
  f3 w = {fmaxf(b.x, 0.f), fmaxf(b.y, 0.f), fmaxf(b.z, 0.f)};
  const float sum = fmaxf(w.x + w.y + w.z, 1e-5f);
  const float inv = DBW_RCP(sum);
  // Beyond a vertex two barycentrics are negative, the third is renormalised to EXACTLY 1 by a true division, and
  // every face sharing that vertex then ties at pz = z_vertex (broken by face index, SURVEY A5).  w * (1/w) is not
  // always 1, so keep that case exact; elsewhere one reciprocal replaces three divisions.
  return {w.x == sum ? 1.f : w.x * inv, w.y == sum ? 1.f : w.y * inv, w.z == sum ? 1.f : w.z * inv};
}

// continuous part: barycentrics (one reciprocal per normalisation instead of three IEEE divisions) and depth
__device__ __forceinline__ Bary bary_from_edges(const Edges& e, const TriGeom& t, bool persp, bool clipb) {
  Bary r;
  r.b0 = {e.e0 * t.inv_area, e.e1 * t.inv_area, e.e2 * t.inv_area};
  r.bp = persp ? persp_forward(r.b0, t.z0, t.z1, t.z2) : r.b0;
  r.inside = e.inside;
  r.bc = clipb ? clip_forward(r.bp) : r.bp;
  r.pz = r.bc.x * t.z0 + r.bc.y * t.z1 + r.bc.z * t.z2;
  return r;
}

__device__ __forceinline__ Bary eval_bary(f2 p, const TriGeom& t, bool persp, bool clipb) {
  return bary_from_edges(eval_edges(p, t), t, persp, clipb);
}

// squared distance from p to the segment a-b, il = 1/|b-a|^2 (or -1: degenerate -> distance to b)
__device__ __forceinline__ float seg_dist2(f2 p, f2 a, f2 b, float il) {
  const float bax = b.x - a.x, bay = b.y - a.y;
  if (il < 0.f) {
    const float dx = p.x - b.x, dy = p.y - b.y;
    return dx * dx + dy * dy;
  }
  float tt = (bax * (p.x - a.x) + bay * (p.y - a.y)) * il;
  tt = fminf(fmaxf(tt, 0.f), 1.f);
  const float dx = a.x + tt * bax - p.x, dy = a.y + tt * bay - p.y;
  return dx * dx + dy * dy;
}

__device__ __forceinline__ float tri_dist2(f2 p, const TriGeom& t) {
  const float e01 = seg_dist2(p, t.v0, t.v1, t.il01), e02 = seg_dist2(p, t.v0, t.v2, t.il02), e12 = seg_dist2(p, t.v1, t.v2, t.il12);
  return fminf(fminf(e01, e02), e12);
}

// same distance, plus WHICH segment realises it (0 = v0v1, 1 = v0v2, 2 = v1v2) with the tie order of tri_dist_backward:
// the forward records it with the fragment, so that the backward differentiates one segment instead of re-deriving three
__device__ __forceinline__ float tri_dist2_edge(f2 p, const TriGeom& t, int& edge) {
  const float e01 = seg_dist2(p, t.v0, t.v1, t.il01), e02 = seg_dist2(p, t.v0, t.v2, t.il02), e12 = seg_dist2(p, t.v1, t.v2, t.il12);
  edge = (e01 <= e02 && e01 <= e12) ? 0 : ((e02 <= e01 && e02 <= e12) ? 1 : 2);
  return fminf(fminf(e01, e02), e12);
}

// Conservative triangle / rectangle overlap for the tile binner: false only if one of the triangle's edge lines has the
// whole rectangle [x0,x1] x [y0,y1] strictly on its outer side (by more than a 1e-5 NDC margin, far above the rounding of
// the affine evaluation).  A face kept needlessly costs time, never correctness; degenerate faces are kept.
__device__ __forceinline__ bool tri_overlaps_rect(f2 v0, f2 v1, f2 v2, float x0, float x1, float y0, float y1) {
  const float area = (v2.x - v0.x) * (v1.y - v0.y) - (v2.y - v0.y) * (v1.x - v0.x);
  if (!(fabsf(area) > 1e-12f)) return true;
  const float sg = area > 0.f ? 1.f : -1.f;
  const f2 a[3] = {v1, v2, v0}, b[3] = {v2, v0, v1};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float cx = sg * (b[i].y - a[i].y), cy = -sg * (b[i].x - a[i].x);     // sg * edge(p; a, b) = cx (p.x - a.x) + cy (p.y - a.y)
    const float bx = cx > 0.f ? x1 : x0, by = cy > 0.f ? y1 : y0;              // the rectangle corner that maximises it
    if (cx * (bx - a[i].x) + cy * (by - a[i].y) < -1e-5f * (fabsf(cx) + fabsf(cy))) return false;
  }
  return true;
}

// ------------------------------------------------------------------ backward pieces (SURVEY A6)

__device__ __forceinline__ void edge_backward(f2 p, f2 a, f2 b, float g, f2& ga, f2& gb) {
  ga.x += g * (p.y - b.y); ga.y += g * (b.x - p.x);
  gb.x += g * (a.y - p.y); gb.y += g * (p.x - a.x);
}

__device__ __forceinline__ void bary_backward(f2 p, const TriGeom& t, f3 g, f2& g0, f2& g1, f2& g2) {
  const float e0 = edge_nc(p, t.v1, t.v2), e1 = edge_nc(p, t.v2, t.v0), e2 = edge_nc(p, t.v0, t.v1);
  const float inv = t.inv_area;
  const float garea = -(g.x * e0 + g.y * e1 + g.z * e2) * inv * inv;
  edge_backward(p, t.v1, t.v2, g.x * inv, g1, g2);
  edge_backward(p, t.v2, t.v0, g.y * inv, g2, g0);
  edge_backward(p, t.v0, t.v1, g.z * inv, g0, g1);
  // area = edge(v2; v0, v1): here the "point" v2 also receives gradient
  g2.x += garea * (t.v1.y - t.v0.y); g2.y += garea * (t.v0.x - t.v1.x);
  edge_backward(t.v2, t.v0, t.v1, garea, g0, g1);
}

__device__ __forceinline__ f3 persp_backward(f3 b, float z0, float z1, float z2, f3 g, float& gz0, float& gz1, float& gz2) {
  const float t0 = b.x * z1 * z2, t1 = z0 * b.y * z2, t2 = z0 * z1 * b.z;
  const float sum = t0 + t1 + t2;
  const float denom = fmaxf(sum, DBW_KEPS);
  const float inv = 1.f / denom;
  const float gden = (sum > DBW_KEPS) ? -(t0 * g.x + t1 * g.y + t2 * g.z) * inv * inv : 0.f;
  const float gt0 = gden + g.x * inv, gt1 = gden + g.y * inv, gt2 = gden + g.z * inv;
  gz0 += gt1 * b.y * z2 + gt2 * b.z * z1;
  gz1 += gt0 * b.x * z2 + gt2 * b.z * z0;
  gz2 += gt0 * b.x * z1 + gt1 * b.y * z0;
  return {gt0 * z1 * z2, gt1 * z0 * z2, gt2 * z0 * z1};
}

__device__ __forceinline__ f3 clip_backward(f3 b, f3 g) {
  const f3 w = {fmaxf(b.x, 0.f), fmaxf(b.y, 0.f), fmaxf(b.z, 0.f)};
  float s = w.x + w.y + w.z;
  float on = 1.f;
  if (s < 1e-5f) { on = 0.f; s = 1e-5f; }
  const float inv = 1.f / s;
  const float gsum = -(g.x * w.x + g.y * w.y + g.z * w.z) * inv * inv * on;
  return {b.x < 0.f ? 0.f : g.x * inv + gsum, b.y < 0.f ? 0.f : g.y * inv + gsum, b.z < 0.f ? 0.f : g.z * inv + gsum};
}

// gradient of seg_dist2 w.r.t. a and b (the closest point's parameter is treated as a constant)
__device__ __forceinline__ void seg_backward(f2 p, f2 a, f2 b, float il, float g, f2& ga, f2& gb) {
  const float bax = b.x - a.x, bay = b.y - a.y;
  if (il < 0.f) {
    gb.x += g * 2.f * (b.x - p.x); gb.y += g * 2.f * (b.y - p.y);
    return;
  }
  float tt = (bax * (p.x - a.x) + bay * (p.y - a.y)) * il;
  tt = fminf(fmaxf(tt, 0.f), 1.f);
  const float dx = a.x + tt * bax - p.x, dy = a.y + tt * bay - p.y;
  ga.x += g * (1.f - tt) * 2.f * dx; ga.y += g * (1.f - tt) * 2.f * dy;
  gb.x += g * tt * 2.f * dx;         gb.y += g * tt * 2.f * dy;
}

__device__ __forceinline__ void tri_dist_backward(f2 p, const TriGeom& t, float g, f2& g0, f2& g1, f2& g2) {
  const float e01 = seg_dist2(p, t.v0, t.v1, t.il01), e02 = seg_dist2(p, t.v0, t.v2, t.il02), e12 = seg_dist2(p, t.v1, t.v2, t.il12);
  if (e01 <= e02 && e01 <= e12) seg_backward(p, t.v0, t.v1, t.il01, g, g0, g1);
  else if (e02 <= e01 && e02 <= e12) seg_backward(p, t.v0, t.v2, t.il02, g, g0, g2);
  else seg_backward(p, t.v1, t.v2, t.il12, g, g1, g2);
}

// ------------------------------------------------------------------ texture fetch (SURVEY A7)
// TexturesUV.sample_textures: grid = 2*uv - 1 on the map flipped along H, F.grid_sample(bilinear,
// align_corners=True, padding_mode='border').  Row r of the flipped map is row H-1-r of the stored map.
struct TexTap {
  int i00, i01, i10, i11;   // texel indices (within the packed float4 texel buffer) of the 4 taps, or -1 if out of bounds
  float w00, w01, w10, w11; // nw, ne, sw, se weights
  float ix, iy;             // un-normalised (clipped) coordinates in the flipped map
  float mx, my;             // d(ix)/du, d(iy)/dv incl. the border-clip mask
  int x0, y0;
};

__device__ __forceinline__ TexTap tex_tap(float u, float v, int off, int H, int W) {
  TexTap t;
  const float gx = u * 2.f - 1.f, gy = v * 2.f - 1.f;
  float ix = ((gx + 1.f) / 2.f) * (float)(W - 1);
  float iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
  // clip_coordinates_set_grad: the borders themselves count as out of bounds for the gradient
  t.mx = (float)(W - 1); t.my = (float)(H - 1);
  if (ix <= 0.f) { ix = 0.f; t.mx = 0.f; } else if (ix >= (float)(W - 1)) { ix = (float)(W - 1); t.mx = 0.f; }
  if (iy <= 0.f) { iy = 0.f; t.my = 0.f; } else if (iy >= (float)(H - 1)) { iy = (float)(H - 1); t.my = 0.f; }
  const float fx0 = floorf(ix), fy0 = floorf(iy);
  const int x0 = (int)fx0, y0 = (int)fy0, x1 = x0 + 1, y1 = y0 + 1;
  const float ex = fx0 + 1.f, ey = fy0 + 1.f;       // south-east corner
  t.w00 = (ex - ix) * (ey - iy);
  t.w01 = (ix - fx0) * (ey - iy);
  t.w10 = (ex - ix) * (iy - fy0);
  t.w11 = (ix - fx0) * (iy - fy0);
  const bool x1ok = x1 <= W - 1, y1ok = y1 <= H - 1;
  const int r0 = (H - 1 - y0) * W, r1 = (H - 1 - y1) * W;
  t.i00 = off + r0 + x0;
  t.i01 = x1ok ? off + r0 + x1 : -1;
  t.i10 = y1ok ? off + r1 + x0 : -1;
  t.i11 = (x1ok && y1ok) ? off + r1 + x1 : -1;
  t.ix = ix; t.iy = iy; t.x0 = x0; t.y0 = y0;
  return t;
}

// Cell maps (DbwMapDesc.reserved = DBW_MAP_CELLS(f, p_left), include/dbw_render.h): a box-decimated map stored as its
// (TS/f) x (TS/f) cells instead of the TS x (p_left + TS + p_right) atlas that repeats each cell over f x f texels (and over
// the circular padding).  tex_tap runs on the logical atlas as before; the taps' texel indices are then replaced by cell
// indices (`off`: first cell of the map): atlas row H-1-y holds source row H-1-y, i.e. cell row (H-1-y)/f; atlas column x
// holds source column (x - p_left) mod TS, i.e. cell column ((x - p_left) mod TS)/f -- the padded columns wrap exactly as
// DBW_TEX_STAGE_EXPAND writes them.  Absent (border) taps stay -1.  TS = H: the textures are square.  f is a power of two
// (2 .. 128), so the divisions are shifts.
__device__ __forceinline__ void tap_to_cells(TexTap& t, int off, int H, int cells) {
  const int f = cells & 0xff, p_left = cells >> 8, TS = H;
  const int sh = ((f & 0xaa) != 0) | (((f & 0xcc) != 0) << 1) | (((f & 0xf0) != 0) << 2);      // log2(f)
  const int CS = TS >> sh;
  int sx0 = t.x0 - p_left;
  sx0 = sx0 < 0 ? sx0 + TS : (sx0 >= TS ? sx0 - TS : sx0);
  const int sx1 = sx0 + 1 >= TS ? 0 : sx0 + 1;
  const int r0 = H - 1 - t.y0;                      // r0 - 1 is used only when the row below exists (r0 >= 1)
  const int row0 = off + (r0 >> sh) * CS, row1 = off + ((r0 - 1) >> sh) * CS;
  const int c0 = sx0 >> sh, c1 = sx1 >> sh;
  t.i00 = row0 + c0;
  t.i01 = t.i01 >= 0 ? row0 + c1 : -1;
  t.i10 = t.i10 >= 0 ? row1 + c0 : -1;
  t.i11 = t.i11 >= 0 ? row1 + c1 : -1;
}

__device__ __forceinline__ f3 ld_texel(const float4* __restrict__ m, int i) {
  if (i < 0) return {0.f, 0.f, 0.f};
  const float4 t = __ldg(m + i);          // one 128-bit load per tap (RGB + pad)
  return {t.x, t.y, t.z};
}

#ifdef __CUDACC__
// vector reduction: one RED.128 per tap instead of three RED.32 (sm_90+)
__device__ __forceinline__ void red_add_v4(float4* addr, float a, float b, float c) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(addr), "f"(a), "f"(b), "f"(c), "f"(0.f) : "memory");
}
#endif  // __CUDACC__
