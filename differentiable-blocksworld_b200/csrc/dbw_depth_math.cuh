// dbw_depth_math.cuh -- per-fragment depth (PyTorch3D's zbuf) and its derivative, for the depth outputs of the raster kernels
// (dbw_render_forward_depth / dbw_render_backward_depth, include/dbw_render.h).
//
// A fragment's depth is the pz the kernels already order their fragments by: the view-space z of the triangle slot's
// vertices interpolated with the barycentrics that are also interpolated with (perspective-corrected and clipped when those
// options are on), pz = bc . (z0, z1, z2) -- bary_from_edges in dbw_math.cuh.  For a z-clipped face the slot is the clipped
// triangle, so pz is the depth after the clip conversion, as PyTorch3D's rasterizer reports it.  Its gradient reaches the
// slot's vertices along two paths: directly through (z0, z1, z2), and through the barycentrics, i.e. through the pixel's
// position relative to the projected triangle.  The barycentric path goes through the same clip / perspective / edge
// backward as the colour's (dbw_math.cuh), and is taken even in a detach_bary pass: PyTorch3D detaches bary_coords, never zbuf.
// Plain C++ apart from the __device__ markers: tests/host_math compiles it for the CPU.
#pragma once
#include "dbw_math.cuh"

// d pz -> d (barycentrics that pz interpolates with) and d (z0, z1, z2) of the slot, accumulated into g_bc and gz
__device__ __forceinline__ void depth_interp_backward(const Bary& b, const TriGeom& t, float g_pz, f3& g_bc, float (&gz)[3]) {
  g_bc.x += g_pz * t.z0; g_bc.y += g_pz * t.z1; g_bc.z += g_pz * t.z2;
  gz[0] += g_pz * b.bc.x; gz[1] += g_pz * b.bc.y; gz[2] += g_pz * b.bc.z;
}

// The whole derivative of one fragment's depth pz at pixel p with respect to its slot's 9 vertex coordinates (x, y, z of
// v0, v1, v2, the layout of the triangle-slot gradients), ADDED into gv9: the interpolation, then clip_backward,
// persp_backward and bary_backward.  b: the fragment's Bary at p (eval_bary with the same persp / clipb).
__device__ __forceinline__ void depth_frag_backward(f2 p, const TriGeom& t, const Bary& b, bool persp, bool clipb, float g_pz,
                                                    float (&gv9)[9]) {
  f3 g = {0.f, 0.f, 0.f};
  float gz[3] = {0.f, 0.f, 0.f};
  depth_interp_backward(b, t, g_pz, g, gz);
  if (clipb) g = clip_backward(b.bp, g);
  if (persp) g = persp_backward(b.b0, t.z0, t.z1, t.z2, g, gz[0], gz[1], gz[2]);
  f2 g0 = {0.f, 0.f}, g1 = {0.f, 0.f}, g2 = {0.f, 0.f};
  bary_backward(p, t, g, g0, g1, g2);
  gv9[0] += g0.x; gv9[1] += g0.y; gv9[2] += gz[0];
  gv9[3] += g1.x; gv9[4] += g1.y; gv9[5] += gz[1];
  gv9[6] += g2.x; gv9[7] += g2.y; gv9[8] += gz[2];
}
