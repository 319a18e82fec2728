/*
 * oracle/raster_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the mesh rasterizer the reference's render hot path delegates to:
 * PyTorch3D 0.7.1 (pinned by the reference's environment.yml:21), reached from the reference at
 *   src/model/renderer.py:50-54  (RasterizationSettings + MeshRasterizer)
 *   src/model/renderer.py:94     (self.renderer(meshes, R=R, T=T, eps=EPS, **kwargs))
 * PyTorch3D is an un-vendored third-party dependency: its sources are NOT in the reference's tree and
 * it is not installed in this image, so this file restates the *published algorithm* of
 *   pytorch3d/csrc/rasterize_meshes/rasterize_meshes_cpu.cpp  (RasterizeMeshesNaiveCpu, RasterizeMeshesBackwardCpu)
 *   pytorch3d/csrc/utils/geometry_utils.h                     (edge function, barycentrics, perspective
 *                                                              correction, clipping, point-segment distance)
 * from SURVEY.md Appendix A (A2, A4, A5, A6).  **PARITY UNPINNED**: the reference ships no tests, golden
 * vectors or fixtures for this path (SURVEY.md section 4, section 8c), so nothing upstream pins these semantics;
 * the restatement is validated by (i) finite differences of its own float64 build, (ii) the reference's own
 * pure-torch functions extracted with `ast` (tests/test_oracle_vs_reference.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this.
 *
 * Build: see oracle/Makefile (-O2 -ffp-contract=off so every +,-,*,/ is a single IEEE-754 RN operation,
 * REAL=float and REAL=double variants; OpenMP over image rows for the CPU baseline).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifndef REAL
#define REAL float
#endif

#define K_EPSILON ((REAL)1e-8)
#define MAX_K 256

typedef struct { REAL x, y; } v2;
typedef struct { REAL x, y, z; } v3;

static inline REAL rmin(REAL a, REAL b) { return a < b ? a : b; }
static inline REAL rmax(REAL a, REAL b) { return a > b ? a : b; }

/* geometry_utils.h: EdgeFunctionForward */
static inline REAL edge_fn(v2 p, v2 a, v2 b) {
  return (p.x - a.x) * (b.y - a.y) - (p.y - a.y) * (b.x - a.x);
}

/* geometry_utils.h: BarycentricCoordinatesForward (SURVEY A4: area = edge(v2,v0,v1) + kEpsilon) */
static inline v3 bary_forward(v2 p, v2 v0, v2 v1, v2 v2_) {
  const REAL area = edge_fn(v2_, v0, v1) + K_EPSILON;
  v3 w;
  w.x = edge_fn(p, v1, v2_) / area;
  w.y = edge_fn(p, v2_, v0) / area;
  w.z = edge_fn(p, v0, v1) / area;
  return w;
}

/* geometry_utils.h: BarycentricPerspectiveCorrectionForward */
static inline v3 bary_persp_forward(v3 b, REAL z0, REAL z1, REAL z2) {
  const REAL t0 = b.x * z1 * z2;
  const REAL t1 = z0 * b.y * z2;
  const REAL t2 = z0 * z1 * b.z;
  const REAL denom = rmax(t0 + t1 + t2, K_EPSILON);
  v3 w = {t0 / denom, t1 / denom, t2 / denom};
  return w;
}

/* geometry_utils.h: BarycentricClipForward -- clamp negatives to 0, renormalise by max(sum, 1e-5) */
static inline v3 bary_clip_forward(v3 b) {
  v3 w = {rmax(b.x, (REAL)0), rmax(b.y, (REAL)0), rmax(b.z, (REAL)0)};
  const REAL s = rmax(w.x + w.y + w.z, (REAL)1e-5);
  w.x /= s; w.y /= s; w.z /= s;
  return w;
}

/* geometry_utils.h: PointLineDistanceForward (squared distance to the segment a-b) */
static inline REAL point_segment_dist2(v2 p, v2 a, v2 b) {
  const REAL bax = b.x - a.x, bay = b.y - a.y;
  const REAL l2 = bax * bax + bay * bay;
  if (l2 <= K_EPSILON) {
    const REAL dx = p.x - b.x, dy = p.y - b.y;
    return dx * dx + dy * dy;
  }
  REAL t = (bax * (p.x - a.x) + bay * (p.y - a.y)) / l2;
  t = rmin(rmax(t, (REAL)0), (REAL)1);
  const REAL qx = a.x + t * bax, qy = a.y + t * bay;
  const REAL dx = qx - p.x, dy = qy - p.y;
  return dx * dx + dy * dy;
}

/* geometry_utils.h: PointTriangleDistanceForward (min over the 3 edges, in the order e01, e02, e12) */
static inline REAL point_triangle_dist2(v2 p, v2 v0, v2 v1, v2 v2_) {
  const REAL e01 = point_segment_dist2(p, v0, v1);
  const REAL e02 = point_segment_dist2(p, v0, v2_);
  const REAL e12 = point_segment_dist2(p, v1, v2_);
  return rmin(rmin(e01, e02), e12);
}

/* rasterization_utils.h: PixToNonSquareNdc (SURVEY A2) */
static inline REAL pix_to_ndc(int i, int S1, int S2) {
  REAL range = (REAL)2;
  if (S1 > S2) range = ((REAL)S1 * range) / (REAL)S2;
  const REAL offset = range / (REAL)2;
  return -offset + (range * (REAL)i + offset) / (REAL)S1;
}

typedef struct { REAL z; int64_t f; REAL d; REAL b0, b1, b2; } cand_t;

/* tuple order of the CPU rasterizer's std::priority_queue<tuple<z, face, dist, b0, b1, b2>> */
static inline int cand_less(const cand_t* a, const cand_t* b) {
  if (a->z != b->z) return a->z < b->z;
  if (a->f != b->f) return a->f < b->f;
  return a->d < b->d;
}

/*
 * RasterizeMeshesNaiveCpu.  face_verts (Ftot,3,3) = NDC x, NDC y, view-space z (SURVEY A1),
 * packed over the N meshes of the batch; outputs (N,H,W,K[,3]).  Face ids written to pix_to_face are
 * packed ids (index into face_verts), -1 where fewer than K faces reach the pixel (SURVEY A5).
 */
void oracle_rasterize_forward(const REAL* face_verts, const int64_t* mesh_first, const int64_t* mesh_nfaces,
                              const int64_t* neighbor, int N, int H, int W, int K, REAL blur_radius,
                              int perspective_correct, int clip_barycentric, int cull_backfaces,
                              int64_t* pix_to_face, REAL* zbuf, REAL* bary, REAL* dists) {
  const REAL sqrt_blur = (REAL)sqrt((double)blur_radius);
  if (K > MAX_K) K = MAX_K;
  for (int n = 0; n < N; ++n) {
    const int64_t f0 = mesh_first[n], f1 = f0 + mesh_nfaces[n];
#pragma omp parallel for schedule(dynamic, 4)
    for (int yi = 0; yi < H; ++yi) {
      cand_t q[MAX_K + 1];
      /* rows run top->bottom in the image but +Y is up in NDC */
      const REAL yf = pix_to_ndc(H - 1 - yi, H, W);
      for (int xi = 0; xi < W; ++xi) {
        const REAL xf = pix_to_ndc(W - 1 - xi, W, H);
        const v2 p = {xf, yf};
        int qn = 0;
        for (int64_t f = f0; f < f1; ++f) {
          const REAL* fv = face_verts + f * 9;
          const v2 a = {fv[0], fv[1]}, b = {fv[3], fv[4]}, c = {fv[6], fv[7]};
          const REAL z0 = fv[2], z1 = fv[5], z2 = fv[8];
          const REAL xmin = rmin(rmin(a.x, b.x), c.x) - sqrt_blur, xmax = rmax(rmax(a.x, b.x), c.x) + sqrt_blur;
          const REAL ymin = rmin(rmin(a.y, b.y), c.y) - sqrt_blur, ymax = rmax(rmax(a.y, b.y), c.y) + sqrt_blur;
          const REAL zmin = rmin(rmin(z0, z1), z2);
          /* faces with a vertex behind the camera must have been clipped away before (SURVEY A3, A4) */
          if (p.x > xmax || p.x < xmin || p.y > ymax || p.y < ymin || zmin < K_EPSILON) continue;
          const REAL area = edge_fn(c, a, b);
          if (area <= K_EPSILON && area >= -K_EPSILON) continue;
          if (cull_backfaces && area < 0) continue;
          const v3 b0 = bary_forward(p, a, b, c);
          const v3 bp = perspective_correct ? bary_persp_forward(b0, z0, z1, z2) : b0;
          const v3 bc = clip_barycentric ? bary_clip_forward(bp) : bp;
          const REAL pz = bc.x * z0 + bc.y * z1 + bc.z * z2;
          if (pz < 0) continue;
          const REAL dist = point_triangle_dist2(p, a, b, c);
          const int inside = bp.x > 0 && bp.y > 0 && bp.z > 0;
          if (!inside && dist >= blur_radius) continue;
          cand_t cnd = {pz, f, inside ? -dist : dist, bc.x, bc.y, bc.z};
          /* a face split in two by z-clipping: only the half with the smaller |dist| may stay (SURVEY A3) */
          int handled = 0;
          const int64_t nb = neighbor ? neighbor[f] : -1;
          if (nb >= 0) {
            for (int i = 0; i < qn; ++i) {
              if (q[i].f == nb) {
                if (dist < (REAL)fabs((double)q[i].d)) {
                  for (int j = i; j + 1 < qn; ++j) q[j] = q[j + 1];
                  --qn;           /* drop the neighbour, then insert the new half below */
                } else {
                  handled = 1;    /* keep the neighbour, drop this half */
                }
                break;
              }
            }
          }
          if (handled) continue;
          /* keep the K smallest tuples, ascending (SURVEY A5) */
          int pos = qn;
          while (pos > 0 && cand_less(&cnd, &q[pos - 1])) { q[pos] = q[pos - 1]; --pos; }
          q[pos] = cnd;
          if (qn < K) ++qn;  /* else q[K] (the largest) falls off */
        }
        const int64_t o = (((int64_t)n * H + yi) * W + xi) * K;
        for (int k = 0; k < K; ++k) {
          if (k < qn) {
            pix_to_face[o + k] = q[k].f; zbuf[o + k] = q[k].z; dists[o + k] = q[k].d;
            bary[(o + k) * 3 + 0] = q[k].b0; bary[(o + k) * 3 + 1] = q[k].b1; bary[(o + k) * 3 + 2] = q[k].b2;
          } else {
            pix_to_face[o + k] = -1; zbuf[o + k] = -1; dists[o + k] = -1;
            bary[(o + k) * 3 + 0] = -1; bary[(o + k) * 3 + 1] = -1; bary[(o + k) * 3 + 2] = -1;
          }
        }
      }
    }
  }
}

/* ---------------------------- backward (SURVEY A6) ---------------------------- */

/* geometry_utils.h: EdgeFunctionBackward -- accumulates d edge(p,a,b) * g into gp, ga, gb */
static inline void edge_backward(v2 p, v2 a, v2 b, REAL g, v2* gp, v2* ga, v2* gb) {
  gp->x += g * (b.y - a.y); gp->y += g * (a.x - b.x);
  ga->x += g * (p.y - b.y); ga->y += g * (b.x - p.x);
  gb->x += g * (a.y - p.y); gb->y += g * (p.x - a.x);
}

/* geometry_utils.h: BarycentricCoordinatesBackward */
static inline void bary_backward(v2 p, v2 v0, v2 v1, v2 v2_, v3 g, v2* g0, v2* g1, v2* g2) {
  const REAL area = edge_fn(v2_, v0, v1) + K_EPSILON;
  const REAL area2 = area * area;
  const REAL e0 = edge_fn(p, v1, v2_), e1 = edge_fn(p, v2_, v0), e2 = edge_fn(p, v0, v1);
  const REAL garea = -(g.x * e0 + g.y * e1 + g.z * e2) / area2;
  v2 gp = {0, 0};
  edge_backward(p, v1, v2_, g.x / area, &gp, g1, g2);
  edge_backward(p, v2_, v0, g.y / area, &gp, g2, g0);
  edge_backward(p, v0, v1, g.z / area, &gp, g0, g1);
  edge_backward(v2_, v0, v1, garea, g2, g0, g1);
}

/* geometry_utils.h: BarycentricPerspectiveCorrectionBackward */
static inline v3 bary_persp_backward(v3 b, REAL z0, REAL z1, REAL z2, v3 g, REAL* gz0, REAL* gz1, REAL* gz2) {
  const REAL t0 = b.x * z1 * z2, t1 = z0 * b.y * z2, t2 = z0 * z1 * b.z;
  const REAL sum = t0 + t1 + t2;
  const REAL denom = rmax(sum, K_EPSILON);
  const REAL gden = (sum > K_EPSILON) ? (-(t0 * g.x + t1 * g.y + t2 * g.z) / (denom * denom)) : (REAL)0;
  const REAL gt0 = gden + g.x / denom, gt1 = gden + g.y / denom, gt2 = gden + g.z / denom;
  v3 gb = {gt0 * z1 * z2, gt1 * z0 * z2, gt2 * z0 * z1};
  *gz0 += gt1 * b.y * z2 + gt2 * b.z * z1;
  *gz1 += gt0 * b.x * z2 + gt2 * b.z * z0;
  *gz2 += gt0 * b.x * z1 + gt1 * b.y * z0;
  return gb;
}

/* geometry_utils.h: BarycentricClipBackward (derivative of clamp + renormalise w.r.t. its input) */
static inline v3 bary_clip_backward(v3 b, v3 g) {
  const v3 w = {rmax(b.x, (REAL)0), rmax(b.y, (REAL)0), rmax(b.z, (REAL)0)};
  REAL s = w.x + w.y + w.z;
  REAL gs_on = 1;
  if (s < (REAL)1e-5) { gs_on = 0; s = (REAL)1e-5; }
  const REAL gsum = -(g.x * w.x + g.y * w.y + g.z * w.z) / (s * s) * gs_on;
  v3 r;
  r.x = (b.x < 0) ? (REAL)0 : (g.x / s + gsum);
  r.y = (b.y < 0) ? (REAL)0 : (g.y / s + gsum);
  r.z = (b.z < 0) ? (REAL)0 : (g.z / s + gsum);
  return r;
}

/* geometry_utils.h: PointLineDistanceBackward -- t is treated as a constant of the closest point */
static inline void point_segment_backward(v2 p, v2 a, v2 b, REAL g, v2* ga, v2* gb) {
  const REAL bax = b.x - a.x, bay = b.y - a.y;
  const REAL l2 = bax * bax + bay * bay;
  if (l2 <= K_EPSILON) {
    gb->x += g * (REAL)2 * (b.x - p.x); gb->y += g * (REAL)2 * (b.y - p.y);
    return;
  }
  REAL t = (bax * (p.x - a.x) + bay * (p.y - a.y)) / l2;
  t = rmin(rmax(t, (REAL)0), (REAL)1);
  const REAL dx = a.x + t * bax - p.x, dy = a.y + t * bay - p.y;
  ga->x += g * ((REAL)1 - t) * (REAL)2 * dx; ga->y += g * ((REAL)1 - t) * (REAL)2 * dy;
  gb->x += g * t * (REAL)2 * dx;             gb->y += g * t * (REAL)2 * dy;
}

/*
 * RasterizeMeshesBackwardCpu: grad_face_verts (Ftot,3,3) must be zero-filled by the caller.
 * Single-threaded on purpose (upstream is, and accumulation order stays deterministic).
 */
void oracle_rasterize_backward(const REAL* face_verts, const int64_t* pix_to_face, const REAL* grad_zbuf,
                               const REAL* grad_bary, const REAL* grad_dists, int N, int H, int W, int K,
                               int perspective_correct, int clip_barycentric, REAL* grad_face_verts) {
  for (int n = 0; n < N; ++n)
    for (int yi = 0; yi < H; ++yi) {
      const REAL yf = pix_to_ndc(H - 1 - yi, H, W);
      for (int xi = 0; xi < W; ++xi) {
        const REAL xf = pix_to_ndc(W - 1 - xi, W, H);
        const v2 p = {xf, yf};
        const int64_t o = (((int64_t)n * H + yi) * W + xi) * K;
        for (int k = 0; k < K; ++k) {
          const int64_t f = pix_to_face[o + k];
          if (f < 0) continue;
          const REAL* fv = face_verts + f * 9;
          const v2 a = {fv[0], fv[1]}, b = {fv[3], fv[4]}, c = {fv[6], fv[7]};
          const REAL z0 = fv[2], z1 = fv[5], z2 = fv[8];
          const v3 b0 = bary_forward(p, a, b, c);
          const v3 bp = perspective_correct ? bary_persp_forward(b0, z0, z1, z2) : b0;
          const v3 bc = clip_barycentric ? bary_clip_forward(bp) : bp;
          const int inside = bp.x > 0 && bp.y > 0 && bp.z > 0;
          const REAL sign = inside ? (REAL)-1 : (REAL)1;
          const REAL gz = grad_zbuf ? grad_zbuf[o + k] : (REAL)0;
          const REAL gd = grad_dists ? grad_dists[o + k] : (REAL)0;
          v3 gb = {gz * z0, gz * z1, gz * z2};
          if (grad_bary) { gb.x += grad_bary[(o + k) * 3]; gb.y += grad_bary[(o + k) * 3 + 1]; gb.z += grad_bary[(o + k) * 3 + 2]; }
          v2 g0 = {0, 0}, g1 = {0, 0}, g2 = {0, 0};
          REAL gz0 = gz * bc.x, gz1 = gz * bc.y, gz2 = gz * bc.z;
          if (clip_barycentric) gb = bary_clip_backward(bp, gb);
          if (perspective_correct) gb = bary_persp_backward(b0, z0, z1, z2, gb, &gz0, &gz1, &gz2);
          bary_backward(p, a, b, c, gb, &g0, &g1, &g2);
          /* distance: only the closest of the three segments receives gradient */
          const REAL e01 = point_segment_dist2(p, a, b), e02 = point_segment_dist2(p, a, c), e12 = point_segment_dist2(p, b, c);
          const REAL gds = sign * gd;
          if (e01 <= e02 && e01 <= e12) point_segment_backward(p, a, b, gds, &g0, &g1);
          else if (e02 <= e01 && e02 <= e12) point_segment_backward(p, a, c, gds, &g0, &g2);
          else point_segment_backward(p, b, c, gds, &g1, &g2);
          REAL* g = grad_face_verts + f * 9;
          g[0] += g0.x; g[1] += g0.y; g[2] += gz0;
          g[3] += g1.x; g[4] += g1.y; g[5] += gz1;
          g[6] += g2.x; g[7] += g2.y; g[8] += gz2;
        }
      }
    }
}

int oracle_real_bytes(void) { return (int)sizeof(REAL); }
