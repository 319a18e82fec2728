"""oracle/pt3d.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.  **PARITY UNPINNED** (see oracle/README.md).

CPU restatement (torch fp32 / fp64 + the C rasterizer in raster_oracle.c) of the PyTorch3D 0.7.1 pieces the
reference's render hot path calls.  PyTorch3D (pinned at the reference's environment.yml:21) is an un-vendored
dependency that is absent from the reference's tree; what is restated here is its published
algorithm as recorded in SURVEY.md Appendix A, anchored on the reference's call sites:

    PerspectiveCameras + MeshRasterizer.transform      <- src/model/renderer.py:53,62-67,94   (Appendix A1)
    clip_faces / convert_clipped_rasterization_...     <- src/model/renderer.py:46 (z_clip_value)  (A3)
    rasterize_meshes (naive CPU path, autograd)        <- src/model/renderer.py:50-54          (A2, A4-A6)
    TexturesUV.sample_textures                         <- src/model/renderer.py:226            (A7)
    ico_sphere / SubdivideMeshes / rotation_6d_to_matrix <- src/utils/mesh.py:105, src/model/dbw.py:78,285,299 (A8)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import ctypes
import math
import os
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def _lib(dtype):
    name = {torch.float32: 'liboracle_f32.so', torch.float64: 'liboracle_f64.so'}[dtype]
    if name not in _LIBS:
        path = os.path.join(_HERE, '_build', name)
        if not os.path.exists(path):
            raise RuntimeError(f'{path} missing: run `make -C oracle` (or __graft_entry__.build())')
        _LIBS[name] = ctypes.CDLL(path)
    return _LIBS[name]


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _real(dtype, v):
    return ctypes.c_float(v) if dtype == torch.float32 else ctypes.c_double(v)


# --------------------------------------------------------------------------------------------------------------
# A1. cameras: world -> view -> NDC (PerspectiveCameras(K=...), in_ndc=True; MeshRasterizer.transform)
# --------------------------------------------------------------------------------------------------------------
def world_to_ndc(verts_world, R, T, K, eps=1e-8):
    """verts_world (V,3) or (B,V,3); R (B,3,3); T (B,3); K (1,4,4) or (4,4) in the layout built by the reference at
    src/dataset/dtu.py:102-106.  Row-vector convention X_view = X_world @ R + T.  Returns (B,V,3) holding
    (x_ndc, y_ndc, z_view)."""
    B = R.shape[0]
    if verts_world.dim() == 2:
        verts_world = verts_world[None].expand(B, -1, -1)
    K = K.reshape(-1, 4, 4)[0].to(verts_world)
    verts_view = torch.bmm(verts_world, R.to(verts_world)) + T.to(verts_world)[:, None]
    ones = torch.ones_like(verts_view[..., :1])
    hom = torch.cat([verts_view, ones], dim=-1) @ K.t()          # [fx X + px Z, fy Y + py Z, 1, Z]
    denom = hom[..., 3:]
    sign = denom.sign() + (denom == 0).to(denom)
    denom = sign * denom.abs().clamp(min=eps)
    xy = hom[..., :2] / denom
    return torch.cat([xy, verts_view[..., 2:3]], dim=-1)           # z_ndc := z_view


# --------------------------------------------------------------------------------------------------------------
# A3. z-clipping of faces (clip.py: clip_faces, z_clip_value only, cull_to_frustum=False)
# --------------------------------------------------------------------------------------------------------------
def _intersect_clip_plane(fv, p1_ind, z_clip, perspective_correct):
    """fv (T,3,3); p1_ind (T,) index of the isolated vertex.  Returns (p1..p5) and their barycentrics (T,3)."""
    Tn = fv.shape[0]
    p2_ind, p3_ind = (p1_ind + 1) % 3, (p1_ind + 2) % 3
    ar = torch.arange(Tn)
    p1, p2, p3 = fv[ar, p1_ind], fv[ar, p2_ind], fv[ar, p3_ind]
    w2 = (p1[:, 2] - z_clip) / (p1[:, 2] - p2[:, 2])
    w3 = (p1[:, 2] - z_clip) / (p1[:, 2] - p3[:, 2])
    if perspective_correct:
        # interpolate in view space (un-project x,y by z), then re-project
        q1 = torch.cat([p1[:, :2] * p1[:, 2:3], p1[:, 2:3]], 1)
        q2 = torch.cat([p2[:, :2] * p2[:, 2:3], p2[:, 2:3]], 1)
        q3 = torch.cat([p3[:, :2] * p3[:, 2:3], p3[:, 2:3]], 1)
        p4 = q1 * (1 - w2[:, None]) + q2 * w2[:, None]
        p5 = q1 * (1 - w3[:, None]) + q3 * w3[:, None]
        p4 = torch.cat([p4[:, :2] / p4[:, 2:3], p4[:, 2:3]], 1)
        p5 = torch.cat([p5[:, :2] / p5[:, 2:3], p5[:, 2:3]], 1)
    else:
        p4 = p1 * (1 - w2[:, None]) + p2 * w2[:, None]
        p5 = p1 * (1 - w3[:, None]) + p3 * w3[:, None]
    onehot = lambda ind: F.one_hot(ind, 3).to(fv)
    b1, b2, b3 = onehot(p1_ind), onehot(p2_ind), onehot(p3_ind)
    b4 = b1 * (1 - w2[:, None]) + b2 * w2[:, None]
    b5 = b1 * (1 - w3[:, None]) + b3 * w3[:, None]
    return (p1, p2, p3, p4, p5), (b1, b2, b3, b4, b5)


def clip_faces(face_verts, mesh_first, mesh_nfaces, z_clip, perspective_correct):
    """face_verts (Ftot,3,3) packed.  Returns a namespace with clipped face_verts, per-mesh index arrays,
    faces_clipped_to_unclipped_idx, barycentric_conversion (Fc,3,3) or None, clipped_faces_neighbor_idx."""
    Ftot = face_verts.shape[0]
    behind = face_verts[:, :, 2] < z_clip
    n_behind = behind.sum(1)
    if int(n_behind.sum()) == 0:
        return SimpleNamespace(face_verts=face_verts, mesh_first=mesh_first, mesh_nfaces=mesh_nfaces,
                               to_unclipped=None, conversion=None, neighbor=None, u2c=None)
    case1 = n_behind == 0            # untouched
    case2 = n_behind == 3            # culled
    case3 = n_behind == 2            # -> one smaller triangle
    case4 = n_behind == 1            # -> quad -> two triangles
    delta = case4.long() - case2.long()
    delta_cum = delta.cumsum(0) - delta
    u2c = torch.arange(Ftot) + delta_cum                      # first clipped index of each unclipped face
    Fc = Ftot + int(delta.sum())
    # per-mesh bookkeeping
    counts = 1 + delta
    new_nfaces = torch.stack([counts[int(s):int(s) + int(n)].sum() for s, n in zip(mesh_first, mesh_nfaces)]).long()
    new_first = torch.cumsum(new_nfaces, 0) - new_nfaces
    fv_c = face_verts.new_zeros(Fc, 3, 3)
    conv = face_verts.new_zeros(Fc, 3, 3)
    c2u = torch.zeros(Fc, dtype=torch.long)
    neighbor = torch.full((Fc,), -1, dtype=torch.long)
    eye = torch.eye(3).to(face_verts)
    pieces_v, pieces_c, pieces_i = [], [], []
    if case1.any():
        idx = u2c[case1]
        pieces_i.append(idx); pieces_v.append(face_verts[case1]); pieces_c.append(eye[None].expand(len(idx), -1, -1))
        c2u[idx] = torch.nonzero(case1)[:, 0]
    if case3.any():
        fv = face_verts[case3]
        p1_ind = torch.nonzero(~behind[case3])[:, 1]            # the single vertex in front
        (p1, _, _, p4, p5), (b1, _, _, b4, b5) = _intersect_clip_plane(fv, p1_ind, z_clip, perspective_correct)
        idx = u2c[case3]
        pieces_i.append(idx); pieces_v.append(torch.stack([p4, p5, p1], 1)); pieces_c.append(torch.stack([b4, b5, b1], 1))
        c2u[idx] = torch.nonzero(case3)[:, 0]
    if case4.any():
        fv = face_verts[case4]
        p1_ind = torch.nonzero(behind[case4])[:, 1]             # the single vertex behind
        (_, p2, p3, p4, p5), (_, b2, b3, b4, b5) = _intersect_clip_plane(fv, p1_ind, z_clip, perspective_correct)
        idx = u2c[case4]
        pieces_i += [idx, idx + 1]
        pieces_v += [torch.stack([p4, p2, p5], 1), torch.stack([p5, p2, p3], 1)]
        pieces_c += [torch.stack([b4, b2, b5], 1), torch.stack([b5, b2, b3], 1)]
        src = torch.nonzero(case4)[:, 0]
        c2u[idx] = src; c2u[idx + 1] = src
        neighbor[idx] = idx + 1; neighbor[idx + 1] = idx
    if pieces_i:
        order = torch.cat(pieces_i)
        fv_c = fv_c.index_put((order,), torch.cat(pieces_v))
        conv = conv.index_put((order,), torch.cat(pieces_c))
    return SimpleNamespace(face_verts=fv_c, mesh_first=new_first, mesh_nfaces=new_nfaces,
                           to_unclipped=c2u, conversion=conv, neighbor=neighbor, u2c=u2c)


# --------------------------------------------------------------------------------------------------------------
# A2, A4-A6. rasterize_meshes (naive CPU kernel + its backward) as an autograd Function
# --------------------------------------------------------------------------------------------------------------
class _RasterizeFaceVerts(torch.autograd.Function):
    @staticmethod
    def forward(ctx, face_verts, mesh_first, mesh_nfaces, neighbor, image_size, blur_radius, K,
                perspective_correct, clip_barycentric, cull_backfaces):
        H, W = image_size
        N = mesh_first.shape[0]
        dt = face_verts.dtype
        fv = face_verts.detach().contiguous()
        p2f = torch.empty(N, H, W, K, dtype=torch.long)
        zbuf = torch.empty(N, H, W, K, dtype=dt)
        bary = torch.empty(N, H, W, K, 3, dtype=dt)
        dists = torch.empty(N, H, W, K, dtype=dt)
        mf, mn = mesh_first.contiguous(), mesh_nfaces.contiguous()
        nb = neighbor.contiguous() if neighbor is not None else None
        _lib(dt).oracle_rasterize_forward(_ptr(fv), _ptr(mf), _ptr(mn), _ptr(nb), N, H, W, K, _real(dt, blur_radius),
                                          int(perspective_correct), int(clip_barycentric), int(cull_backfaces),
                                          _ptr(p2f), _ptr(zbuf), _ptr(bary), _ptr(dists))
        ctx.save_for_backward(fv, p2f)
        ctx.cfg = (N, H, W, K, int(perspective_correct), int(clip_barycentric))
        ctx.mark_non_differentiable(p2f)
        return p2f, zbuf, bary, dists

    @staticmethod
    def backward(ctx, _g_p2f, g_zbuf, g_bary, g_dists):
        fv, p2f = ctx.saved_tensors
        N, H, W, K, pc, cb = ctx.cfg
        dt = fv.dtype
        g = torch.zeros_like(fv)
        gz = g_zbuf.contiguous() if g_zbuf is not None else None
        gb = g_bary.contiguous() if g_bary is not None else None
        gd = g_dists.contiguous() if g_dists is not None else None
        _lib(dt).oracle_rasterize_backward(_ptr(fv), _ptr(p2f), _ptr(gz), _ptr(gb), _ptr(gd), N, H, W, K, pc, cb, _ptr(g))
        return g, None, None, None, None, None, None, None, None, None


def rasterize_meshes(verts_ndc, faces, image_size, blur_radius=0.0, faces_per_pixel=8, perspective_correct=True,
                     clip_barycentric_coords=True, cull_backfaces=False, z_clip_value=None):
    """verts_ndc (N,V,3) = (x_ndc, y_ndc, z_view); faces (F,3) shared by the N meshes (Meshes.extend).
    Returns fragments (pix_to_face with batch-packed ids n*F+f, zbuf, bary_coords, dists), each (N,H,W,K[,3])."""
    N, V, _ = verts_ndc.shape
    Fn = faces.shape[0]
    face_verts = verts_ndc[:, faces].reshape(N * Fn, 3, 3)
    mesh_first = torch.arange(N, dtype=torch.long) * Fn
    mesh_nfaces = torch.full((N,), Fn, dtype=torch.long)
    clipped = SimpleNamespace(face_verts=face_verts, mesh_first=mesh_first, mesh_nfaces=mesh_nfaces,
                              to_unclipped=None, conversion=None, neighbor=None, u2c=None)
    if z_clip_value is not None:
        clipped = clip_faces(face_verts, mesh_first, mesh_nfaces, z_clip_value, perspective_correct)
    p2f, zbuf, bary, dists = _RasterizeFaceVerts.apply(
        clipped.face_verts, clipped.mesh_first, clipped.mesh_nfaces, clipped.neighbor, tuple(image_size),
        float(blur_radius), int(faces_per_pixel), perspective_correct, clip_barycentric_coords, cull_backfaces)
    clipped_idx = p2f            # face index in the CLIPPED face list (test diagnostics: which half of a split quad)
    if clipped.to_unclipped is not None:
        # convert_clipped_rasterization_to_original_faces
        valid = p2f >= 0
        idx = p2f.clamp(min=0)
        conv = clipped.conversion[idx]                                     # (N,H,W,K,3,3)
        bary_u = (bary[..., :, None] * conv).sum(-2)                       # row-vector times matrix
        bary = torch.where(valid[..., None], bary_u, bary)
        p2f = torch.where(valid, clipped.to_unclipped[idx], p2f)
    return SimpleNamespace(pix_to_face=p2f, zbuf=zbuf, bary_coords=bary, dists=dists, clipped_idx=clipped_idx,
                           unclipped_to_clipped=clipped.u2c)


# --------------------------------------------------------------------------------------------------------------
# A7. TexturesUV.sample_textures (align_corners=True, padding_mode='border', bilinear, map flipped along H)
# --------------------------------------------------------------------------------------------------------------
def sample_textures(fragments, faces_verts_uvs, face_map, maps):
    """faces_verts_uvs (F,3,2) per scene face; face_map (F,) map index per face; maps: list of (Ht,Wt,3).
    The scene's faces repeat for each mesh of the batch (packed id n*F+f).  Sampling each face's own map directly is
    equivalent to PyTorch3D's packed-atlas sampling up to fp32 rounding of the atlas' affine UV remap (SURVEY A7).
    Returns texels (N,H,W,K,3); empty slots give 0."""
    p2f, bary = fragments.pix_to_face, fragments.bary_coords
    N, H, W, K = p2f.shape
    Fn = faces_verts_uvs.shape[0]
    valid = p2f >= 0
    f_local = p2f.clamp(min=0) % Fn
    # interpolate_face_attributes: sum_i bary_i * attr_i (empty slots -> 0)
    uv_f = faces_verts_uvs.to(bary)[f_local]                                # (N,H,W,K,3,2)
    pixel_uvs = (bary[..., None] * uv_f).sum(-2) * valid[..., None].to(bary)
    texels = bary.new_zeros(N, H, W, K, 3)
    m_of = face_map[f_local]
    for m, tex in enumerate(maps):
        sel = valid & (m_of == m)
        if not bool(sel.any()):
            continue
        uv = pixel_uvs[sel]                                                 # (P,2)
        grid = (uv * 2.0 - 1.0)[None, :, None, :]                           # (1,P,1,2)
        tmap = torch.flip(tex.to(bary).permute(2, 0, 1)[None], [2])         # (1,3,Ht,Wt), flipped along H
        out = F.grid_sample(tmap, grid, mode='bilinear', align_corners=True, padding_mode='border')
        texels = texels.masked_scatter(sel[..., None].expand(-1, -1, -1, -1, 3), out[0, :, :, 0].t().reshape(-1))
    return texels


# --------------------------------------------------------------------------------------------------------------
# A8. mesh constructors
# --------------------------------------------------------------------------------------------------------------
def _ico_base():
    # level-0 constants as published (4 decimals, not re-normalised at level 0)
    a, b = 0.5257, 0.8507
    verts = [[-a, b, 0], [a, b, 0], [-a, -b, 0], [a, -b, 0], [0, -a, b], [0, a, b],
             [0, -a, -b], [0, a, -b], [b, 0, -a], [b, 0, a], [-b, 0, -a], [-b, 0, a]]
    faces = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
             [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
             [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    return verts, faces


def subdivide(verts, faces):
    """SubdivideMeshes: one new vertex at the middle of each unique edge, appended in edges_packed order
    (edges gathered as cat([e12, e20, e01]), sorted (lo, hi), uniqued by hash V*lo+hi); 4 sub-faces per face in the
    concatenation order f0,f1,f2,f3.  verts (V,3) float tensor, faces (F,3) long tensor."""
    V = verts.shape[0]
    v0, v1, v2 = faces.unbind(1)
    e01, e12, e20 = torch.stack([v0, v1], 1), torch.stack([v1, v2], 1), torch.stack([v2, v0], 1)
    edges = torch.cat([e12, e20, e01], 0)
    edges, _ = edges.sort(dim=1)
    key = edges[:, 0] * V + edges[:, 1]
    ukey, inverse = torch.unique(key, return_inverse=True)          # sorted unique
    uedges = torch.stack([ukey // V, ukey % V], 1)
    Fn = faces.shape[0]
    inv = inverse.reshape(3, Fn).t()                                 # face -> (edge id of e12, e20, e01)
    f_e12, f_e20, f_e01 = inv[:, 0] + V, inv[:, 1] + V, inv[:, 2] + V
    new_verts = torch.cat([verts, verts[uedges].mean(1)], 0)
    f0 = torch.stack([v0, f_e01, f_e20], 1)
    f1 = torch.stack([v1, f_e12, f_e01], 1)
    f2 = torch.stack([v2, f_e20, f_e12], 1)
    f3 = torch.stack([f_e12, f_e20, f_e01], 1)
    return new_verts, torch.cat([f0, f1, f2, f3], 0)


def ico_sphere(level=0):
    """pytorch3d.utils.ico_sphere: icosahedron constants, `level` subdivisions each followed by re-normalisation."""
    v, f = _ico_base()
    verts, faces = torch.tensor(v, dtype=torch.float32), torch.tensor(f, dtype=torch.long)
    for _ in range(level):
        verts, faces = subdivide(verts, faces)
        verts = verts / verts.norm(p=2, dim=1, keepdim=True)
    return verts, faces


def rotation_6d_to_matrix(d6):
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = F.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = F.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack((b1, b2, b3), dim=-2)


def matrix_to_rotation_6d(matrix):
    return matrix[..., :2, :].clone().reshape(*matrix.shape[:-2], 6)
