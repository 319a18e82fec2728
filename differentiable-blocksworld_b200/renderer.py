"""Drop-in for the reference's `Renderer` (src/model/renderer.py:24-132): same constructor kwargs, same
`forward(meshes, R, T, viz_purpose=False, **kwargs) -> (B,4,H,W)`, same `update_cameras(device=, K=)` /
`.cameras.K` probe (src/model/dbw.py:204-208) -- but the whole MeshRasterizer + LayeredShader + layered_rgb_blend
stack behind it is ONE pair of hand-written sm_90a kernels reached through the C-ABI of include/dbw_render.h.
There is no CPU / PyTorch fallback: a missing library or a non-CUDA tensor raises.
Shading types: 'raw' with ambient lights (training), 'flat' with a directional light (renderer_light), and 'phong' with
ambient, directional or point lights for hard single-layer renders (sigma 0, faces_per_pixel 1, and every viz_purpose
render); soft phong, gouraud and any backward through a lit render raise NotImplementedError."""
import ctypes
from copy import deepcopy

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import _lib
from ._lib import DbwMapDesc, DbwRenderSettings, DbwError, DbwPhongShading

LAYERED_SHADER = True
SHADING_TYPE = 'raw'
EPS = 1e-8          # renderer.py:20


class _Cameras:
    """The subset of PyTorch3D's PerspectiveCameras / FoVPerspectiveCameras state the hot path reads."""

    def __init__(self, name='fov', device=None, K=None, fov=60.0, **unused):
        self.name, self.K, self.device, self.fov = name, K, device, fov
        self._intr = None          # host copy of (fx, fy, px, py): read once, so that forward() never syncs

    def to(self, device):
        self.device = device
        if self.K is not None:
            self.K = self.K.to(device)
        return self

    def intrinsics(self):
        """(fx, fy, px, py) of the NDC projection x_ndc = fx X/Z + px (SURVEY Appendix A1)."""
        if self._intr is not None:
            return self._intr
        if self.K is not None:
            K = self.K.reshape(-1, 4, 4)[0].detach().cpu()
            self._intr = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
            return self._intr
        if self.name == 'perspective':
            return 1.0, 1.0, 0.0, 0.0                   # PerspectiveCameras defaults: focal_length=1, principal_point=0
        f = 1.0 / np.tan(np.deg2rad(self.fov) / 2)      # FoVPerspectiveCameras, aspect 1
        return f, f, 0.0, 0.0


def _c(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _RenderFn(torch.autograd.Function):
    """autograd seam over dbw_render_forward / dbw_render_backward (include/dbw_render.h)."""

    @staticmethod
    def forward(ctx, verts, maps, faces_alpha, R, T, faces, faces_uvs, face_map, map_table, cfg, face_shade=None, want_dists=False,
                want_ids=False):
        if not verts.is_cuda:
            raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
        s = cfg
        B, H, W, K = s.n_views, s.height, s.width, s.faces_per_pixel
        L = _lib.lib()
        verts, maps = verts.detach().contiguous().float(), maps.detach().contiguous().float()
        fa = faces_alpha.detach().contiguous().float() if faces_alpha is not None else None
        R, T = R.detach().contiguous().float(), T.detach().contiguous().float()
        fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(L.dbw_workspace_bytes(ctypes.byref(s), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
        ws = torch.empty(fwd.value, dtype=torch.uint8, device=verts.device)
        out = torch.empty(B, 4, H, W, dtype=torch.float32, device=verts.device)
        # the per-pixel face ids / distances are diagnostic outputs (render_edges, tests): the backward streams the fragment
        # records the forward keeps in its workspace (settings.save_fragment_state)
        ids = torch.empty(B, K, H, W, dtype=torch.int32, device=verts.device) if (want_ids or want_dists) else None
        dists = torch.empty(B, K, H, W, dtype=torch.float32, device=verts.device) if want_dists else None
        shade = face_shade.detach().contiguous().float() if face_shade is not None else None
        _lib.check(L.dbw_render_forward(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                        _c(map_table), _c(R), _c(T), _c(fa), _c(out), _c(ids), _c(ws), fwd.value,
                                        _c(shade), _c(dists), _stream()), 'dbw_render_forward')
        ctx.save_for_backward(verts, maps, fa, R, T, faces, faces_uvs, face_map, map_table, ws)
        ctx.cfg, ctx.bwd_bytes, ctx.lit = s, bwd.value, shade is not None
        if want_dists:
            ctx.mark_non_differentiable(ids, dists)
            return out, ids, dists
        if want_ids:
            ctx.mark_non_differentiable(ids)
            return out, ids
        return out

    @staticmethod
    def backward(ctx, g_out, _g_ids=None, _g_dists=None):
        if ctx.lit:
            raise NotImplementedError('flat-shaded (lit) renders are a visualisation path: no backward')
        verts, maps, fa, R, T, faces, faces_uvs, face_map, map_table, ws = ctx.saved_tensors
        s = ctx.cfg
        if not s.save_fragment_state:
            raise DbwError('this render was made with gradients disabled (no fragment records were kept)')
        L = _lib.lib()
        g_out = g_out.contiguous().float()
        need_v, need_m, need_a = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2] and fa is not None
        g_verts = g_fa = None
        if need_v and need_a:      # one zero-fill for both small gradients
            flat = torch.zeros(verts.numel() + fa.numel(), device=verts.device, dtype=torch.float32)
            g_verts, g_fa = flat[:verts.numel()].view_as(verts), flat[verts.numel():].view_as(fa)
        elif need_v:
            g_verts = torch.zeros_like(verts)
        elif need_a:
            g_fa = torch.zeros_like(fa)
        g_maps = torch.zeros_like(maps) if need_m else None
        scratch = torch.empty(ctx.bwd_bytes, dtype=torch.uint8, device=verts.device)
        need_R, need_T = ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        g_R = g_T = None
        if need_R or need_T:
            if s.verts_are_ndc:
                raise DbwError('R and T are not part of a render from NDC vertices (verts_are_ndc): they have no gradient')
            # the camera gradients share one zero-fill; a call with camera gradients also differentiates the static faces
            # (include/dbw_render.h), so g_verts then holds their vertices' rows too
            cam = torch.zeros(R.shape[0] * 12, device=verts.device, dtype=torch.float32)
            g_R = cam[:R.numel()].view_as(R) if need_R else None
            g_T = cam[R.numel():].view_as(T) if need_T else None
        _lib.check(L.dbw_render_backward(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                         _c(map_table), _c(R), _c(T), _c(fa), _c(ws), ws.numel(), _c(g_out), None,
                                         _c(g_verts), _c(g_fa), _c(g_maps), _c(g_R), _c(g_T), _c(scratch), scratch.numel(),
                                         _stream()), 'dbw_render_backward')
        return g_verts, g_maps, g_fa, g_R, g_T, None, None, None, None, None, None, None, None


class _RenderDepthFn(torch.autograd.Function):
    """autograd seam over dbw_render_forward_depth / dbw_render_backward_depth (include/dbw_render.h): the render of _RenderFn
    -- the same RGBA bits -- with the blended depth (B,1,H,W) and the per-fragment zbuf (B,K,H,W) as differentiable outputs.
    Outputs: rgba, then ids (also when only dists are asked, as _RenderFn) and dists (not differentiable), then depth and zbuf."""

    @staticmethod
    def forward(ctx, verts, maps, faces_alpha, R, T, faces, faces_uvs, face_map, map_table, cfg, want_depth, want_zbuf,
                want_ids=False, want_dists=False):
        if not verts.is_cuda:
            raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
        ctx.set_materialize_grads(False)
        s = cfg
        B, H, W, K = s.n_views, s.height, s.width, s.faces_per_pixel
        L = _lib.lib()
        verts, maps = verts.detach().contiguous().float(), maps.detach().contiguous().float()
        fa = faces_alpha.detach().contiguous().float() if faces_alpha is not None else None
        R, T = R.detach().contiguous().float(), T.detach().contiguous().float()
        fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(L.dbw_workspace_bytes(ctypes.byref(s), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
        dev = verts.device
        ws = torch.empty(fwd.value, dtype=torch.uint8, device=dev)
        out = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)
        ids = torch.empty(B, K, H, W, dtype=torch.int32, device=dev) if (want_ids or want_dists) else None
        dists = torch.empty(B, K, H, W, dtype=torch.float32, device=dev) if want_dists else None
        depth = torch.empty(B, 1, H, W, dtype=torch.float32, device=dev) if want_depth else None
        zbuf = torch.empty(B, K, H, W, dtype=torch.float32, device=dev) if want_zbuf else None
        _lib.check(L.dbw_render_forward_depth(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                              _c(map_table), _c(R), _c(T), _c(fa), _c(out), _c(ids), _c(ws), fwd.value, None,
                                              _c(dists), _c(zbuf), _c(depth), _stream()), 'dbw_render_forward_depth')
        ctx.save_for_backward(verts, maps, fa, R, T, faces, faces_uvs, face_map, map_table, ws)
        ctx.cfg, ctx.bwd_bytes = s, bwd.value
        extras = [t for t in (ids, dists) if t is not None]           # _RenderFn's layout: ids whenever dists are returned
        ctx.mark_non_differentiable(*extras)
        ctx.n_extras, ctx.want_depth = len(extras), want_depth
        return (out, *extras, *[t for t in (depth, zbuf) if t is not None])

    @staticmethod
    def backward(ctx, g_out, *grads):
        verts, maps, fa, R, T, faces, faces_uvs, face_map, map_table, ws = ctx.saved_tensors
        s = ctx.cfg
        if not s.save_fragment_state:
            raise DbwError('this render was made with gradients disabled (no fragment records were kept)')
        grads = list(grads[ctx.n_extras:])
        g_depth = grads.pop(0) if ctx.want_depth else None
        g_zbuf = grads.pop(0) if grads else None
        L = _lib.lib()
        dev = verts.device
        # outputs nothing read have no gradient (None); with neither depth gradient this is dbw_render_backward
        g_out = torch.zeros(s.n_views, 4, s.height, s.width, device=dev) if g_out is None else g_out.contiguous().float()
        g_depth = g_depth.contiguous().float() if g_depth is not None else None
        g_zbuf = g_zbuf.contiguous().float() if g_zbuf is not None else None
        need = ctx.needs_input_grad
        g_verts = torch.zeros_like(verts) if need[0] else None
        g_maps = torch.zeros_like(maps) if need[1] else None
        g_fa = torch.zeros_like(fa) if need[2] and fa is not None else None
        g_R = g_T = None
        if need[3] or need[4]:
            if s.verts_are_ndc:
                raise DbwError('R and T are not part of a render from NDC vertices (verts_are_ndc): they have no gradient')
            g_R, g_T = torch.zeros_like(R) if need[3] else None, torch.zeros_like(T) if need[4] else None
        scratch = torch.empty(ctx.bwd_bytes, dtype=torch.uint8, device=dev)
        _lib.check(L.dbw_render_backward_depth(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                               _c(map_table), _c(R), _c(T), _c(fa), _c(ws), ws.numel(), _c(g_out), None,
                                               _c(g_zbuf), _c(g_depth), _c(g_verts), _c(g_fa), _c(g_maps), _c(g_R), _c(g_T),
                                               _c(scratch), scratch.numel(), _stream()), 'dbw_render_backward_depth')
        return (g_verts, g_maps, g_fa, g_R, g_T) + (None,) * 9


class _ProjectFn(torch.autograd.Function):
    """autograd seam over dbw_camera_project / dbw_camera_project_backward (include/dbw_render.h)."""

    @staticmethod
    def forward(ctx, verts, R, T, intr, eps):
        if not verts.is_cuda:
            raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
        verts, R, T, intr = (t.detach().contiguous().float() for t in (verts, R, T, intr))
        B, V = R.shape[0], verts.shape[0]
        out = torch.empty(B, V, 3, dtype=torch.float32, device=verts.device)
        _lib.check(_lib.lib().dbw_camera_project(B, V, _c(verts), _c(R), _c(T), _c(intr), ctypes.c_float(eps), _c(out), _stream()),
                   'dbw_camera_project')
        ctx.save_for_backward(verts, R, T, intr)
        ctx.eps = eps
        return out

    @staticmethod
    def backward(ctx, g_ndc):
        verts, R, T, intr = ctx.saved_tensors
        need = ctx.needs_input_grad
        B, V = R.shape[0], verts.shape[0]
        # one zero-fill for every gradient wanted: vertices, then the 9 + 3 + 4 camera floats of each view
        sizes = [verts.numel() if need[0] else 0, R.numel() if need[1] else 0, T.numel() if need[2] else 0, intr.numel() if need[3] else 0]
        flat = torch.zeros(sum(sizes), dtype=torch.float32, device=verts.device)
        grads, o = [], 0
        for t, n in zip((verts, R, T, intr), sizes):
            grads.append(flat[o:o + n].view_as(t) if n else None)
            o += n
        _lib.check(_lib.lib().dbw_camera_project_backward(B, V, _c(verts), _c(R), _c(T), _c(intr), ctypes.c_float(ctx.eps),
                                                          _c(g_ndc.contiguous().float()), *[_c(g) for g in grads], _stream()),
                   'dbw_camera_project_backward')
        return (*grads, None)


def intrinsics_of(K):
    """(B,4) = (fx, fy, px, py) of per-view intrinsics K (B,4,4), read as K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] by device
    indexing (no host read; autograd scatters a gradient back into exactly those four entries).  The other entries of K --
    skew among them -- are ignored, as by the single-camera path."""
    K = K.reshape(-1, 4, 4)
    return torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], dim=-1)


def view_intrinsics(K, B):
    """(B,4) (fx, fy, px, py) of B views from K (B,4,4), or from one (1,4,4) / (4,4) K shared by all of them"""
    intr = intrinsics_of(K)
    if intr.shape[0] != B:
        if intr.shape[0] != 1:
            raise DbwError(f'K must hold 1 or {B} cameras (one per view), got {intr.shape[0]}')
        intr = intr.expand(B, -1)
    return intr


def project_verts(verts, R, T, K=None, eps=EPS, intr=None):
    """world vertices (V,3) -> (B,V,3) = (x_ndc, y_ndc, z_view), each view b through its own R[b], T[b] and intrinsics K[b]
    (B,4,4) (a single (1,4,4) / (4,4) K serves every view), or through intr (B,4) from view_intrinsics() when several passes
    share the cameras.  Differentiable with respect to all inputs."""
    if intr is None:
        intr = view_intrinsics(K, R.shape[0])
    return _ProjectFn.apply(verts, R, T, intr, float(eps))


def cameras_need_grad(R, T, K):
    """a render from these cameras differentiates them: its static faces then get gradients too (they move in the image)"""
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in (R, T, K))


_TABLE_CACHE = {}


def _device_map_table(table_host, dev):
    """(M) DbwMapDesc on the device, cached per (layout, device): built once, so that steady-state calls do no H2D.
    Entries are (offset, H, W) or (offset, H, W, reserved) -- reserved != 0: a cell map (scene_ops.cell_map_table)."""
    key = (tuple(table_host), str(dev))
    if key not in _TABLE_CACHE:
        table = (DbwMapDesc * len(table_host))(*[DbwMapDesc(*(int(x) for x in e), *([0] if len(e) == 3 else [])) for e in table_host])
        _TABLE_CACHE[key] = torch.frombuffer(bytearray(bytes(table)), dtype=torch.int32).to(dev)
    return _TABLE_CACHE[key]


def make_settings(B, H, W, K, V, Fn, M, alpha_stride, intr, sigma, blur_radius, z_clip, background, clip_inside=True,
                  perspective_correct=True, clip_barycentric=True, detach_bary=False, verts_are_ndc=False, eps=EPS,
                  n_map_floats=0, maps_are_texels4=False, save_fragment_state=False, alpha_group=1, n_static_faces=0,
                  view_rows=None):
    s = DbwRenderSettings()
    s.n_views, s.height, s.width, s.faces_per_pixel = B, H, W, K
    s.n_verts, s.n_faces, s.n_maps, s.alpha_view_stride = V, Fn, M, alpha_stride
    s.fx, s.fy, s.px, s.py = intr
    s.sigma, s.blur_radius = float(sigma), float(blur_radius)
    s.z_clip = float(z_clip) if z_clip is not None else -1.0
    s.proj_eps = float(eps)
    s.background = (ctypes.c_float * 3)(*[float(c) for c in background])
    s.clip_inside, s.perspective_correct = int(clip_inside), int(perspective_correct)
    s.clip_barycentric, s.detach_bary, s.verts_are_ndc = int(clip_barycentric), int(detach_bary), int(verts_are_ndc)
    s.n_map_floats = int(n_map_floats)
    s.maps_are_texels4 = int(maps_are_texels4)
    s.save_fragment_state = int(save_fragment_state)
    s.alpha_group, s.n_static_faces = int(alpha_group), int(n_static_faces)
    if view_rows is not None:
        if view_rows.dtype != torch.int32 or not view_rows.is_cuda or tuple(view_rows.shape) != (B, 2) or not view_rows.is_contiguous():
            raise DbwError('view_rows must be a contiguous CUDA int32 tensor of shape (B, 2)')
        s.view_rows = view_rows.data_ptr()
        s._view_rows_owner = view_rows            # keeps the device buffer alive as long as the settings
    return s


def _check_cell_maps(table_host, maps, texels4):
    """cell maps (DbwMapDesc.reserved != 0) lie within `maps`, counted in float4 cells (the library only sees the device table)"""
    for e in table_host:
        if len(e) < 4 or not e[3]:
            continue
        o, h, _, r = (int(x) for x in e[:4])
        f, p_left = r & 0xff, r >> 8
        if not texels4 or f not in (2, 4, 8, 16, 32, 64, 128) or h % f or p_left > h or o % 3:
            raise DbwError(f'bad cell map {tuple(e)}: needs maps_are_texels4, a power-of-two f in [2, 128] dividing H, p_left <= H')
        if o // 3 + (h // f) ** 2 > maps.numel() // 4:
            raise DbwError(f'cell map {tuple(e)} reaches past the {maps.numel() // 4} cells of `maps`')


def scene_settings(verts, faces, maps, map_table_host, B, intr, image_size, sigma, faces_per_pixel, z_clip=None,
                   detach_bary=False, clip_inside=True, background=(0., 0., 0.), faces_alpha=None, perspective_correct=True,
                   verts_are_ndc=False, blur_radius=None, maps_are_texels4=False, alpha_group=1, n_static_faces=0, view_rows=None):
    """(DbwRenderSettings, device map table) of one render pass over raw scene tensors.
    alpha_group: faces per opacity entry (faces_alpha then has F / alpha_group [or B * that] entries);
    n_static_faces: leading faces whose vertices are constants (no vertex gradient wanted)."""
    H, W = image_size
    V, Fn = verts.shape[-2], faces.shape[0]
    _check_cell_maps(map_table_host, maps, maps_are_texels4)
    map_table = _device_map_table(map_table_host, verts.device)
    alpha_stride = 0
    if faces_alpha is not None:
        n_alpha = Fn // alpha_group
        if faces_alpha.numel() == B * n_alpha and B > 1:
            alpha_stride = n_alpha
        elif faces_alpha.numel() != n_alpha:
            raise DbwError(f'faces_alpha must have {n_alpha} or B*{n_alpha} entries, got {faces_alpha.numel()}')
    if blur_radius is None:
        blur_radius = np.log(1. / 1e-4 - 1.) * sigma            # renderer.py:51
    cfg = make_settings(B, H, W, faces_per_pixel, V, Fn, len(map_table_host), alpha_stride, intr, sigma, blur_radius,
                        z_clip, background, clip_inside, perspective_correct, True, detach_bary, verts_are_ndc,
                        n_map_floats=(maps.numel() // 4 * 3) if maps_are_texels4 else maps.numel(),
                        # 2: float4 maps with cell maps among them (the backward then spreads their gradient over copies)
                        maps_are_texels4=(2 if any(len(e) > 3 and e[3] for e in map_table_host) else 1) if maps_are_texels4 else 0,
                        # what a backward streams, written only when one may follow: records and colours of the kept
                        # fragments; 2 = a pass without opacities (a hard single-layer one then needs no colours)
                        save_fragment_state=(1 if faces_alpha is not None else 2) if torch.is_grad_enabled() else 0,
                        alpha_group=alpha_group, n_static_faces=n_static_faces,
                        view_rows=view_rows)
    return cfg, map_table


def render_scene(verts, faces, faces_uvs, face_map, maps, map_table_host, R, T, intr, image_size, sigma, faces_per_pixel,
                 z_clip=None, detach_bary=False, clip_inside=True, background=(0., 0., 0.), faces_alpha=None,
                 perspective_correct=True, verts_are_ndc=False, blur_radius=None, return_ids=False, maps_are_texels4=False,
                 face_shade=None, return_dists=False, alpha_group=1, n_static_faces=0, view_rows=None, return_depth=False,
                 return_zbuf=False):
    """Functional form over raw tensors (used by Renderer.forward and by the parity tests).
    verts (V,3) [or (B,V,3) NDC], faces (F,3) int32, faces_uvs (F,3,2), face_map (F) int32, maps flat float buffer,
    map_table_host [(offset,H,W)], R (B,3,3), T (B,3), faces_alpha None | (F,) | (B*F,).
    intr: (fx, fy, px, py) floats shared by every view, or a tensor K (B,4,4) of per-view intrinsics: the world vertices are
    then projected per view on the device (project_verts) and rendered as NDC input; R, T and K receive gradients.
    maps_are_texels4: `maps` is a float4 (RGB+pad) texel atlas from scene_ops.scene_atlases (offsets stay 3*texel).
    return_depth / return_zbuf: also the blended depth (B,1,H,W) -- layered_rgb_blend of the fragments' view-space z with
    background 0, so depth / alpha is the expected depth of the covered part -- and the per-fragment depth (B,K,H,W)
    (PyTorch3D's fragments.zbuf, planar like the ids; -1 in empty slots), appended to the outputs in that order.  Both are
    differentiable, to the same leaves as the image, also with detach_bary; the image is the same bits as without them.
    Not with face_shade or view_rows."""
    if torch.is_tensor(intr):
        if verts_are_ndc or R is None:
            raise DbwError('per-view intrinsics project world vertices: they need R and T, and verts_are_ndc=False')
        if cameras_need_grad(R, T, intr):
            n_static_faces = 0
        verts, R, T, intr, verts_are_ndc = project_verts(verts, R, T, intr), None, None, (1., 1., 0., 0.), True
    dev = verts.device
    B = R.shape[0] if R is not None else verts.shape[0]
    cfg, map_table = scene_settings(verts, faces, maps, map_table_host, B, intr, image_size, sigma, faces_per_pixel, z_clip,
                                    detach_bary, clip_inside, background, faces_alpha, perspective_correct, verts_are_ndc,
                                    blur_radius, maps_are_texels4, alpha_group, n_static_faces, view_rows)
    if R is None:
        R = torch.eye(3, device=dev)[None].expand(B, -1, -1)
        T = torch.zeros(B, 3, device=dev)
    args = (verts, maps, faces_alpha, R, T, faces.to(torch.int32).contiguous(), faces_uvs.contiguous().float(),
            face_map.to(torch.int32).contiguous(), map_table, cfg)
    if return_depth or return_zbuf:
        if face_shade is not None:
            raise NotImplementedError('depth of a lit (flat-shaded) render is not implemented')
        # (rgba, [slot ids], [signed squared distances], [depth], [zbuf])
        return _RenderDepthFn.apply(*args, bool(return_depth), bool(return_zbuf), bool(return_ids), bool(return_dists))
    res = _RenderFn.apply(*args, face_shade, return_dists, return_ids)
    return res                           # rgba | (rgba, slot ids) | (rgba, slot ids, signed squared distances)


VIZ_FACTOR = 4      # VizMeshRenderer's supersampling (renderer.py:56-60)


def _viz_settings(verts, faces, maps, map_table_host, B, intr, image_size, z_clip, detach_bary, clip_inside, background,
                  perspective_correct, verts_are_ndc):
    """settings of a resolving render: the hard pass (K = 1, sigma = 0) on the 4H x 4W sample grid of (H, W) frames"""
    H, W = image_size
    with torch.no_grad():            # no fragment records
        return scene_settings(verts, faces, maps, map_table_host, B, intr, (H * VIZ_FACTOR, W * VIZ_FACTOR), 0.0, 1, z_clip,
                              detach_bary, clip_inside, background, perspective_correct=perspective_correct,
                              verts_are_ndc=verts_are_ndc, blur_radius=0.0)


def viz_bytes(n_verts, n_faces, map_table_host, maps_numel, B, image_size):
    """device bytes of a resolving render of B (H, W) frames: workspace, float RGBA frames and uint8 frames"""
    s = make_settings(B, image_size[0] * VIZ_FACTOR, image_size[1] * VIZ_FACTOR, 1, n_verts, n_faces, len(map_table_host), 0,
                      (1., 1., 0., 0.), 0.0, 0.0, None, (0., 0., 0.), n_map_floats=maps_numel)
    ws = ctypes.c_size_t(0)
    _lib.check(_lib.lib().dbw_viz_workspace_bytes(ctypes.byref(s), VIZ_FACTOR, ctypes.byref(ws)), 'dbw_viz_workspace_bytes')
    return ws.value + B * image_size[0] * image_size[1] * (4 * 4 + 3)


@torch.no_grad()
def render_scene_viz(verts, faces, faces_uvs, face_map, maps, map_table_host, R, T, intr, image_size, z_clip=None,
                     detach_bary=False, clip_inside=True, background=(0., 0., 0.), perspective_correct=True, face_shade=None,
                     bkg=None, frames_u8=False):
    """VizMeshRenderer's frame (renderer.py:56-60,178-183) in one kernel: the hard render at 4H x 4W resolved 4x4 on chip
    (dbw_render_forward_viz), equal bit for bit to avg_pool2d(render_scene(..., (4H, 4W), 0.0, 1, ...), 4).
    Arguments as render_scene; image_size is the (H, W) of the frames.  bkg (3,H,W) or (1 | B,3,H,W): composited under the
    RGB as rec * alpha + (1 - alpha) * bkg.  Returns rgba (B,4,H,W), and with frames_u8 also (B,H,W,3) uint8 frames,
    uint8(trunc(clamp(rgb * 255, 0, 255))) of the same RGB."""
    if torch.is_tensor(intr):
        verts, R, T, intr, verts_are_ndc = project_verts(verts, R, T, intr), None, None, (1., 1., 0., 0.), True
    else:
        verts_are_ndc = False
    dev = verts.device
    if not verts.is_cuda:
        raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
    B = R.shape[0] if R is not None else verts.shape[0]
    H, W = image_size
    cfg, map_table = _viz_settings(verts, faces, maps, map_table_host, B, intr, image_size, z_clip, detach_bary, clip_inside,
                                   background, perspective_correct, verts_are_ndc)
    if R is None:
        R = torch.eye(3, device=dev)[None].expand(B, -1, -1)
        T = torch.zeros(B, 3, device=dev)
    L = _lib.lib()
    ws_bytes = ctypes.c_size_t(0)
    _lib.check(L.dbw_viz_workspace_bytes(ctypes.byref(cfg), VIZ_FACTOR, ctypes.byref(ws_bytes)), 'dbw_viz_workspace_bytes')
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    n_bkg = 0
    if bkg is not None:
        bkg = bkg.to(device=dev, dtype=torch.float32).reshape(-1, 3, H, W).contiguous()
        n_bkg = bkg.shape[0]
    rgba = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)
    rgb8 = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev) if frames_u8 else None
    # converted copies are held until the launch is enqueued: a temporary freed earlier could be handed to the next one
    args = [verts.contiguous().float(), faces.to(torch.int32).contiguous(), faces_uvs.contiguous().float(),
            face_map.to(torch.int32).contiguous(), maps.contiguous().float(), map_table, R.contiguous().float(),
            T.contiguous().float(), None, face_shade.contiguous().float() if face_shade is not None else None]
    _lib.check(L.dbw_render_forward_viz(ctypes.byref(cfg), *[_c(a) for a in args], VIZ_FACTOR, _c(bkg), n_bkg, _c(rgba), _c(rgb8),
                                        _c(ws), ws.numel(), _stream()), 'dbw_render_forward_viz')
    return (rgba, rgb8) if frames_u8 else rgba


# ------------------------------------------------------------------ phong shading
# PyTorch3D's defaults: DirectionalLights / PointLights, AmbientLights (white), Materials (the reference passes none)
LIGHT_DEFAULTS = {'ambient_color': (0.5, 0.5, 0.5), 'diffuse_color': (0.3, 0.3, 0.3), 'specular_color': (0.2, 0.2, 0.2),
                  'direction': (0., 1., 0.), 'location': (0., 1., 0.)}
AMBIENT_LIGHT_COLOR = (1., 1., 1.)
MATERIAL_DEFAULTS = {'ambient_color': (1., 1., 1.), 'diffuse_color': (1., 1., 1.), 'specular_color': (1., 1., 1.), 'shininess': 64.}


def phong_shading(lights=None, materials=None):
    """DbwPhongShading of PyTorch3D lights given as the reference's Renderer takes them ({'name': 'ambient' | 'directional' |
    'point', colours, direction / location}, one light) and of Materials kwargs (ambient_color, diffuse_color, specular_color,
    shininess), each defaulting as in PyTorch3D"""
    lights, materials = dict(lights or {}), dict(materials or {})
    name = lights.pop('name', 'ambient')
    if name not in _lib.LIGHTS:
        raise NotImplementedError(f'lights name={name!r}: only ambient, directional and point lights are implemented')
    vec = lambda v: [float(x) for x in (v.detach().cpu() if torch.is_tensor(v) else torch.tensor(v, dtype=torch.float64)).reshape(-1, 3)[0]]
    sh = DbwPhongShading()
    sh.light = _lib.LIGHTS[name]
    defaults = dict(LIGHT_DEFAULTS, ambient_color=AMBIENT_LIGHT_COLOR) if name == 'ambient' else LIGHT_DEFAULTS
    for k in ('ambient_color', 'diffuse_color', 'specular_color'):
        getattr(sh, k)[:] = vec(lights.get(k, defaults[k])) if name != 'ambient' or k == 'ambient_color' else [0., 0., 0.]
    sh.direction[:] = vec(lights.get('location' if name == 'point' else 'direction', defaults['direction']))
    for field, k in (('ka', 'ambient_color'), ('kd', 'diffuse_color'), ('ks', 'specular_color')):
        getattr(sh, field)[:] = vec(materials.get(k, MATERIAL_DEFAULTS[k]))
    sh.shininess = float(materials.get('shininess', MATERIAL_DEFAULTS['shininess']))
    return sh


def vertex_face_list(faces, n_verts):
    """(vf_end (V), vf_faces (3F)) int32: the faces of vertex v, in ascending order, are vf_faces[vf_end[v-1] : vf_end[v]]
    (dbw_vertex_face_list).  faces (F,3) int32 on the device."""
    faces = faces.to(torch.int32).contiguous()
    vf_end = torch.empty(n_verts, dtype=torch.int32, device=faces.device)
    vf_faces = torch.empty(faces.numel(), dtype=torch.int32, device=faces.device)
    _lib.check(_lib.lib().dbw_vertex_face_list(_c(faces), faces.shape[0], n_verts, _c(vf_end), _c(vf_faces), _stream()),
               'dbw_vertex_face_list')
    return vf_end, vf_faces


@torch.no_grad()
def vertex_normals(verts, faces, vf=None):
    """Meshes.verts_normals_packed of one mesh: (V,3) unit area-weighted vertex normals (eps 1e-6), summed in a fixed order
    (bit-reproducible).  vf: vertex_face_list(faces, V), built here when not given."""
    if not verts.is_cuda:
        raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
    verts, faces = verts.detach().contiguous().float(), faces.to(torch.int32).contiguous()
    vf_end, vf_faces = vertex_face_list(faces, verts.shape[0]) if vf is None else vf
    out = torch.empty_like(verts)
    _lib.check(_lib.lib().dbw_vertex_normals(_c(verts), _c(faces), verts.shape[0], _c(vf_end), _c(vf_faces), _c(out), _stream()),
               'dbw_vertex_normals')
    return out


class _PhongFn(torch.autograd.Function):
    """a phong render (dbw_render_forward_phong) in the autograd graph: its backward refuses, as the flat-shaded one does"""

    @staticmethod
    def forward(ctx, verts, maps, faces_alpha, R, T, run):
        return run()

    @staticmethod
    def backward(ctx, *grads):
        raise NotImplementedError('phong-shaded renders are a visualisation path: no backward')


def render_scene_phong(verts, faces, faces_uvs, face_map, maps, map_table_host, R, T, intr, image_size, shading, factor=1,
                       z_clip=None, detach_bary=False, clip_inside=True, background=(0., 0., 0.), faces_alpha=None,
                       perspective_correct=True, bkg=None, frames_u8=False, normals=None):
    """The hard single-layer render (faces_per_pixel 1, sigma 0) with every pixel Phong-shaded (dbw_render_forward_phong).
    Arguments as render_scene; shading: a DbwPhongShading (phong_shading()); normals: vertex_normals(verts, faces), computed
    here when None.  factor 1: rgba (B,4,H,W) of image_size.  factor 4: render_scene_viz's frames of image_size (the render
    at 4H x 4W resolved 4x4 in the kernel), with bkg and frames_u8 as there.  No gradient: a backward raises."""
    if factor not in (1, 4):
        raise DbwError('factor must be 1 (plain hard render) or 4 (the resolving render)')
    if not verts.is_cuda:
        raise DbwError('the CUDA renderer needs CUDA tensors (there is no CPU fallback)')
    dev = verts.device
    H, W = image_size
    B = R.shape[0]
    normals = vertex_normals(verts, faces) if normals is None else normals

    def run():
        with torch.no_grad():
            vw, Rc, Tc = verts.detach().contiguous().float(), R.detach().contiguous().float(), T.detach().contiguous().float()
            v_in, i_in, ndc = vw, intr, False
            if torch.is_tensor(intr):             # per-view intrinsics: the kernel rasterizes the projected vertices
                v_in, i_in, ndc = project_verts(vw, Rc, Tc, intr).contiguous(), (1., 1., 0., 0.), True
            L = _lib.lib()
            cfg, map_table = scene_settings(v_in, faces, maps, map_table_host, B, i_in, (H * factor, W * factor), 0.0, 1, z_clip,
                                            detach_bary, clip_inside, background, faces_alpha, perspective_correct, ndc,
                                            blur_radius=0.0)
            ws_bytes, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
            if factor == 4:
                _lib.check(L.dbw_viz_workspace_bytes(ctypes.byref(cfg), 4, ctypes.byref(ws_bytes)), 'dbw_viz_workspace_bytes')
            else:
                _lib.check(L.dbw_workspace_bytes(ctypes.byref(cfg), ctypes.byref(ws_bytes), ctypes.byref(bwd)), 'dbw_workspace_bytes')
            ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
            n_bkg, bk = 0, None
            if bkg is not None:
                bk = bkg.to(device=dev, dtype=torch.float32).reshape(-1, 3, H, W).contiguous()
                n_bkg = bk.shape[0]
            rgba = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)
            rgb8 = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev) if frames_u8 else None
            # converted copies are held until the launch is enqueued
            args = [v_in.contiguous().float(), faces.to(torch.int32).contiguous(), faces_uvs.contiguous().float(),
                    face_map.to(torch.int32).contiguous(), maps.contiguous().float(), map_table, Rc, Tc,
                    faces_alpha.detach().contiguous().float() if faces_alpha is not None else None, vw, normals.contiguous().float()]
            _lib.check(L.dbw_render_forward_phong(ctypes.byref(cfg), *[_c(a) for a in args], ctypes.byref(shading), factor, _c(bk),
                                                  n_bkg, _c(rgba), _c(rgb8), _c(ws), ws.numel(), _stream()), 'dbw_render_forward_phong')
            return (rgba, rgb8) if frames_u8 else rgba

    if factor == 1 and (bkg is not None or frames_u8):
        raise DbwError('bkg and frames_u8 belong to the resolving render (factor 4)')
    if frames_u8:
        return run()
    return _PhongFn.apply(verts, maps, faces_alpha, R, T, run)


class Renderer(nn.Module):
    def __init__(self, img_size, **kwargs):
        super().__init__()
        self.img_size = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        self._init_kwargs = deepcopy(kwargs)
        self.init_cameras(**kwargs.pop('cameras', {}))
        self.init_lights(**kwargs.pop('lights', {}))
        self.sigma = kwargs.pop('sigma', 1e-4)
        self.background_color = tuple(kwargs.pop('background_color', (0, 0, 0)))
        self.faces_per_pixel = kwargs.pop('faces_per_pixel', 25)
        p_correct = kwargs.pop('perspective_correct', None)
        self.perspective_correct = True if p_correct is None else bool(p_correct)   # None -> True for perspective cams
        self.z_clip = kwargs.pop('z_clip', None)
        kwargs.pop('debug', False)
        if not kwargs.pop('layered_shader', LAYERED_SHADER):
            raise NotImplementedError('only the LayeredShader path of the reference is implemented')
        self.clip_inside = kwargs.pop('clip_inside', True)
        self.shading_type = kwargs.pop('shading_type', SHADING_TYPE)
        self.detach_bary = kwargs.pop('detach_bary', False)
        assert len(kwargs) == 0, kwargs
        self._vf = None             # (int32 faces, vertex -> face list) of the last phong render's topology
        self.blur_radius = float(np.log(1. / 1e-4 - 1.) * self.sigma)                # renderer.py:51

    def init_cameras(self, **kwargs):
        kwargs = deepcopy(kwargs)
        self.cam_kwargs = kwargs
        self.cameras = _Cameras(**kwargs)

    def init_lights(self, **kwargs):
        self.light_kwargs = deepcopy(kwargs)

    @property
    def init_kwargs(self):
        return deepcopy(self._init_kwargs)

    def update_cameras(self, **kwargs):
        merged = deepcopy(self.cam_kwargs)
        merged.update(kwargs)
        self.cameras = _Cameras(**merged)

    def to(self, device):
        super().to(device)
        self.cameras = self.cameras.to(device)
        return self

    def _flat_shade(self, verts, faces, R):
        """PyTorch3D flat shading with ambient + directional diffuse light, as the reference configures renderer_light
        (dbw.py:139-143): per (view, face) colour multiplier ambient + diffuse * relu(n_f . l_b), the light direction
        being re-expressed per view so that it is fixed relative to the camera (renderer.py:87-89)."""
        lk = self.light_kwargs
        col = lambda k, d: torch.tensor(lk.get(k, d), dtype=torch.float32, device=verts.device).reshape(-1, 3)[0]
        ambient, diffuse = col('ambient_color', [[0.5] * 3]), col('diffuse_color', [[0.3] * 3])
        direction = col('direction', [[0, 1, 0]])
        fv = verts[faces.long()]
        n = torch.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0], dim=-1)
        n = F.normalize(n, dim=-1, eps=1e-6)
        l = F.normalize(direction[None] @ R.transpose(1, 2), dim=-1, eps=1e-6)          # (B,1,3)
        cos = torch.relu((n[None] * l).sum(-1))                                          # (B,F)
        return ambient[None, None] + diffuse[None, None] * cos[..., None]

    def _scene(self, meshes):
        verts, faces = meshes.get_mesh_verts_faces(0)
        fvu, fmap = meshes.textures.scene_arrays()
        maps, table = meshes.textures.packed_maps()
        return verts, faces, fvu, fmap, maps, table

    def _phong_normals(self, verts, faces):
        """vertex_normals of the scene, through a vertex -> face list kept while the faces tensor is unchanged (its storage is
        held with it, so that no other faces can take its address)"""
        key = (faces.data_ptr(), tuple(faces.shape), faces.stride(), faces._version, verts.shape[0], str(faces.device))
        if self._vf is None or self._vf[0] != key:
            f32 = faces.to(torch.int32).contiguous()
            self._vf = (key, faces, f32, vertex_face_list(f32, verts.shape[0]))
        return vertex_normals(verts, self._vf[2], self._vf[3])

    def _phong(self, meshes, R, T, K, factor, faces_alpha=None, bkg=None, frames_u8=False):
        """LayeredShader(shading_type='phong') over the hard single-layer render: render_scene_phong with this renderer's
        lights, PyTorch3D's default materials and the scene's vertex normals"""
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        intr = K if K is not None else self.cameras.intrinsics()
        return render_scene_phong(verts, faces, fvu, fmap, maps, table, R, T, intr, self.img_size, phong_shading(self.light_kwargs),
                                  factor, self.z_clip, self.detach_bary, self.clip_inside, self.background_color, faces_alpha,
                                  self.perspective_correct, bkg=bkg, frames_u8=frames_u8, normals=self._phong_normals(verts, faces))

    def _shade(self, verts, faces, R):
        """the per-(view, face) flat-shading multiplier of a lit renderer, None for the raw one"""
        lit = self.light_kwargs.get('name', 'ambient') == 'directional'
        if self.shading_type == 'gouraud':
            raise NotImplementedError('shading_type=gouraud: PyTorch3D interpolates vertex colours (TexturesVertex), which a '
                                      'texture-mapped scene does not have')
        if self.shading_type not in ('raw', 'flat') or (lit != (self.shading_type == 'flat')):
            raise NotImplementedError(f'shading_type={self.shading_type} with lights={self.light_kwargs.get("name", "ambient")}: '
                                      'only raw+ambient (training) and flat+directional (renderer_light) are implemented')
        return self._flat_shade(verts, faces, R) if lit else None

    def forward(self, meshes, R, T, viz_purpose=False, depth=False, **kwargs):
        """(B,4,H,W) RGBA; with depth=True (rgba, depth): depth (B,1,H,W) is the fragments' view-space z blended with the colour
        weights over a background of 0 (depth / alpha: the expected depth of the covered part), differentiable like the image"""
        faces_alpha, K = kwargs.get('faces_alpha'), kwargs.get('K')
        if depth and (viz_purpose or self.shading_type != 'raw'):
            raise NotImplementedError('depth=True is a training render: raw shading, viz_purpose=False')
        if self.shading_type == 'phong':
            if viz_purpose:          # VizMeshRenderer's frame, resolved in the kernel: the bits of avg_pool2d(render at 4x, 4)
                with torch.no_grad():
                    return self._phong(meshes, R, T, K, 4, faces_alpha)
            if self.sigma != 0 or self.faces_per_pixel != 1:
                raise NotImplementedError(f'soft phong shading (sigma={self.sigma}, faces_per_pixel={self.faces_per_pixel}) is not '
                                          'implemented: phong renders are hard and single-layer (sigma=0, faces_per_pixel=1)')
            return self._phong(meshes, R, T, K, 1, faces_alpha)
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        H, W = self.img_size
        intr = K if K is not None else self.cameras.intrinsics()      # K (B,4,4): each view with its own intrinsics
        shade = self._shade(verts, faces, R)
        if viz_purpose:
            # VizMeshRenderer (renderer.py:56-60,178-183): hard 4x supersampled render, box-filtered, no gradient
            with torch.no_grad():
                out = render_scene(verts, faces, fvu, fmap, maps, table, R, T, intr, (H * 4, W * 4), 0.0, 1, self.z_clip,
                                   self.detach_bary, self.clip_inside, self.background_color, faces_alpha,
                                   self.perspective_correct, face_shade=shade)
                return F.avg_pool2d(out, kernel_size=4, stride=4)
        return render_scene(verts, faces, fvu, fmap, maps, table, R, T, intr, (H, W), self.sigma, self.faces_per_pixel,
                            self.z_clip, self.detach_bary, self.clip_inside, self.background_color, faces_alpha,
                            self.perspective_correct, blur_radius=self.blur_radius, face_shade=shade, return_depth=depth)

    @torch.no_grad()
    def render_viz(self, meshes, R, T, K=None, bkg=None, frames_u8=False):
        """forward(meshes, R, T, viz_purpose=True, K=K) -- the same bits -- in one resolving kernel that never writes the 4x
        supersampled image (render_scene_viz): rgba (B,4,H,W), RGB composited over bkg ((3,H,W) or (1 | B,3,H,W)) when given;
        with frames_u8 also the (B,H,W,3) uint8 frames a video encoder takes.  No gradient."""
        if self.shading_type == 'phong':
            return self._phong(meshes, R, T, K, 4, bkg=bkg, frames_u8=frames_u8)
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        intr = K if K is not None else self.cameras.intrinsics()
        return render_scene_viz(verts, faces, fvu, fmap, maps, table, R, T, intr, self.img_size, self.z_clip, self.detach_bary,
                                self.clip_inside, self.background_color, self.perspective_correct,
                                face_shade=self._shade(verts, faces, R), bkg=bkg, frames_u8=frames_u8)

    def viz_bytes(self, meshes, n_views):
        """device bytes render_viz needs for n_views frames of this renderer"""
        verts, faces = meshes.get_mesh_verts_faces(0)
        maps, table = meshes.textures.packed_maps()
        return viz_bytes(verts.shape[-2], faces.shape[0], table, maps.numel(), n_views, self.img_size)

    # ------------------------------------------------------------------ edge overlays (renderer.py:134-175)
    @torch.no_grad()
    def render_edges(self, meshes, R, T, image_size=None, linewidth=1, return_pix2face=False, faces_per_pixel=1, K=None):
        """mask of the pixels closer than `linewidth` pixels to an edge of the face(s) they see: a hard rasterization whose
        signed squared NDC distances are thresholded at (linewidth * 2 / min(image_size))^2.  K (B,4,4): per-view intrinsics."""
        image_size = tuple(image_size or self.img_size)
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        intr = K if K is not None else self.cameras.intrinsics()
        _, ids, dists = render_scene(verts, faces, fvu, fmap, maps, table, R, T, intr, image_size, 0.0,
                                     faces_per_pixel, self.z_clip, perspective_correct=self.perspective_correct,
                                     return_dists=True)
        mask = (-dists < (linewidth * 2 / min(image_size)) ** 2).float().max(1, keepdim=True)[0]       # (B,1,H,W)
        if return_pix2face:
            Fn = faces.shape[0]
            slot = ids[:, 0].long()
            face = torch.where(slot >= Fn, slot - Fn, slot)                 # second halves of z-clipped quads -> their face
            pix2face = torch.where(slot >= 0, face + torch.arange(len(R), device=slot.device)[:, None, None] * Fn, slot)
            return mask, pix2face                                           # batch-packed ids like fragments.pix_to_face
        return mask

    def draw_edges(self, img, meshes, R=None, T=None, colors=None, linewidth=1, antialias=True, K=None):
        dev = meshes.device
        B = img.shape[0] if isinstance(img, torch.Tensor) and img.dim() == 4 else 1
        if R is None:
            R = torch.eye(3, device=dev)[None].expand(B, -1, -1)
        if T is None:
            T = torch.zeros(1, 3, device=dev).expand(B, -1)
        if colors is None:
            colors = (1, 0, 0)
        assert isinstance(img, torch.Tensor), 'PIL inputs are an export path of the reference: pass a (B,3,H,W) tensor'
        img_size = tuple(img.shape[-2:])
        if antialias:
            img_size, linewidth = (img_size[0] * 4, img_size[1] * 4), linewidth * 4
        if isinstance(colors, (list, tuple)):
            colors = torch.Tensor(colors)
        mask, pix2face = self.render_edges(meshes, R, T, image_size=img_size, linewidth=linewidth, return_pix2face=True, K=K)
        if colors.dim() == 2:
            face_img = colors.to(mask.device)[pix2face].permute(0, 3, 1, 2)               # one colour per (packed) face
        else:
            face_img = colors.to(mask.device)[:, None, None].expand(-1, *mask.shape[2:])[None].expand(len(mask), -1, -1, -1)
        if antialias:
            mask, face_img = [F.avg_pool2d(t, kernel_size=4, stride=4) for t in [mask, face_img]]
        return img * (1 - mask) + mask * face_img
