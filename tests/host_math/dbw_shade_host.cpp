// Host build of the Phong shading math (differentiable-blocksworld_b200/csrc/dbw_shade_math.cuh) for tests/test_phong_host.py:
// the vertex normals gathered through a vertex -> face list, as vertex_normals_kernel does per vertex, and the lighting of
// single fragments, as the phong hard-render kernels do.  Test infrastructure only.
#include <cmath>
#include <cstdint>

#define __device__
#define __forceinline__ inline

#include "../../include/dbw_render.h"
#include "../../differentiable-blocksworld_b200/csrc/dbw_shade_math.cuh"

extern "C" {

// verts (V,3), faces (F,3), the vertex -> face list (vf_end (V), vf_faces) -> normals (V,3)
void hs_vertex_normals(int V, const float* verts, const int* faces, const int* vf_end, const int* vf_faces, float* normals) {
  for (int v = 0; v < V; ++v) {
    DbwVec3 n = shade_v3(0.f, 0.f, 0.f);
    for (int k = v ? vf_end[v - 1] : 0; k < vf_end[v]; ++k) {
      const int* f = faces + 3 * vf_faces[k];
      const DbwVec3 fn = shade_face_normal(shade_load3(verts + 3 * f[0]), shade_load3(verts + 3 * f[1]), shade_load3(verts + 3 * f[2]));
      n = shade_v3(n.x + fn.x, n.y + fn.y, n.z + fn.z);
    }
    n = shade_normalize(n);
    normals[3 * v] = n.x; normals[3 * v + 1] = n.y; normals[3 * v + 2] = n.z;
  }
}

// n fragments of view b: texel, normal, point (n,3) each, with R (3,3), T (3) of the view -> colour (n,3)
void hs_phong(const DbwPhongShading* L, int n, const float* texel, const float* normal, const float* point, const float* R,
              const float* T, float* out) {
  DbwVec3 light, camera;
  shade_view_setup(*L, R, T, light, camera);
  for (int i = 0; i < n; ++i) {
    const DbwVec3 c = shade_phong(*L, shade_load3(texel + 3 * i), shade_load3(normal + 3 * i), shade_load3(point + 3 * i), light, camera);
    out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
  }
}

size_t hs_sizeof_shading(void) { return sizeof(DbwPhongShading); }

}
