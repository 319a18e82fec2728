// dbw_shade_math.cuh -- per-element math of Phong shading (dbw_shade.cu, and the phong hard-render kernels of dbw_render.cu):
// PyTorch3D's face normals and Meshes.verts_normals_packed normalisation, and phong_shading's lighting of one fragment
// (pytorch3d/renderer/lighting.py diffuse / specular, mesh/shading.py _apply_lighting) for the light types the reference's
// Renderer configures (src/model/renderer.py:70-81).  Plain C++ apart from the __device__ markers: tests/host_math compiles
// it for the CPU and checks it against float64.
//
// Needs DbwPhongShading / DBW_LIGHT_* from include/dbw_render.h.
#pragma once
#include <math.h>

#define DBW_SHADE_NORMALIZE_EPS 1e-6f     // F.normalize(..., eps=1e-6) of verts_normals_packed, diffuse and specular

struct DbwVec3 { float x, y, z; };

__device__ __forceinline__ DbwVec3 shade_v3(float x, float y, float z) { DbwVec3 r = {x, y, z}; return r; }
__device__ __forceinline__ DbwVec3 shade_load3(const float* p) { return shade_v3(p[0], p[1], p[2]); }
__device__ __forceinline__ DbwVec3 shade_sub(DbwVec3 a, DbwVec3 b) { return shade_v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float shade_dot(DbwVec3 a, DbwVec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ DbwVec3 shade_cross(DbwVec3 a, DbwVec3 b) {
  return shade_v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// F.normalize(v, eps): v / max(|v|, eps)
__device__ __forceinline__ DbwVec3 shade_normalize(DbwVec3 v) {
  const float n = fmaxf(sqrtf(shade_dot(v, v)), DBW_SHADE_NORMALIZE_EPS);
  return shade_v3(v.x / n, v.y / n, v.z / n);
}

// the area-weighted normal one face adds to each of its vertices: (v2 - v1) x (v0 - v1), |.| = twice its area
__device__ __forceinline__ DbwVec3 shade_face_normal(DbwVec3 v0, DbwVec3 v1, DbwVec3 v2) {
  return shade_cross(shade_sub(v2, v1), shade_sub(v0, v1));
}

// per-view light and camera: a directional light's direction re-expressed as direction @ R^T (src/model/renderer.py:87-89;
// a point light's location stays in the world), and the camera centre -T @ R^T (X_view = X_world @ R + T).  R row-major 3x3.
__device__ __forceinline__ void shade_view_setup(const DbwPhongShading& L, const float* R, const float* T, DbwVec3& light,
                                                 DbwVec3& camera) {
  const float* d = L.direction;
  light = L.light == DBW_LIGHT_DIRECTIONAL
              ? shade_v3(d[0] * R[0] + d[1] * R[1] + d[2] * R[2], d[0] * R[3] + d[1] * R[4] + d[2] * R[5],
                         d[0] * R[6] + d[1] * R[7] + d[2] * R[8])
              : shade_v3(d[0], d[1], d[2]);
  camera = shade_v3(-(T[0] * R[0] + T[1] * R[1] + T[2] * R[2]), -(T[0] * R[3] + T[1] * R[4] + T[2] * R[5]),
                    -(T[0] * R[6] + T[1] * R[7] + T[2] * R[8]));
}

// phong_shading's colour of one fragment: (ka La + kd diffuse) * texel + ks specular, with
//   diffuse  = Ld relu(n . l)
//   specular = Ls pow(relu(v . (2 (n . l) n - l)) [n . l > 0], shininess)
// n, l, v normalised with eps 1e-6; n the interpolated vertex normal, p the interpolated world position; l the per-view light
// direction (directional) or location - p (point); v = camera - p.  Ambient lights give ka La * texel.
__device__ __forceinline__ DbwVec3 shade_phong(const DbwPhongShading& L, DbwVec3 texel, DbwVec3 n_in, DbwVec3 p, DbwVec3 light,
                                               DbwVec3 camera) {
  float df[3] = {0.f, 0.f, 0.f}, sp[3] = {0.f, 0.f, 0.f};
  if (L.light != DBW_LIGHT_AMBIENT) {
    const DbwVec3 n = shade_normalize(n_in);
    const DbwVec3 l = shade_normalize(L.light == DBW_LIGHT_POINT ? shade_sub(light, p) : light);
    const float cos_nl = shade_dot(n, l);
    const float d = fmaxf(cos_nl, 0.f);
    const DbwVec3 v = shade_normalize(shade_sub(camera, p));
    const DbwVec3 r = shade_v3(2.f * cos_nl * n.x - l.x, 2.f * cos_nl * n.y - l.y, 2.f * cos_nl * n.z - l.z);
    const float alpha = cos_nl > 0.f ? fmaxf(shade_dot(v, r), 0.f) : 0.f;
    const float s = powf(alpha, L.shininess);
    for (int c = 0; c < 3; ++c) { df[c] = L.diffuse_color[c] * d; sp[c] = L.specular_color[c] * s; }
  }
  const float t[3] = {texel.x, texel.y, texel.z};
  float o[3];
  for (int c = 0; c < 3; ++c) o[c] = (L.ka[c] * L.ambient_color[c] + L.kd[c] * df[c]) * t[c] + L.ks[c] * sp[c];
  return shade_v3(o[0], o[1], o[2]);
}
