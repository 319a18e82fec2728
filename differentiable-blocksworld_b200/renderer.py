"""Drop-in for the reference's `Renderer` (src/model/renderer.py:24-132): same constructor kwargs, same
`forward(meshes, R, T, viz_purpose=False, **kwargs) -> (B,4,H,W)`, same `update_cameras(device=, K=)` /
`.cameras.K` probe (src/model/dbw.py:204-208) -- but the whole MeshRasterizer + LayeredShader + layered_rgb_blend
stack behind it is ONE pair of hand-written sm_90a kernels reached through the C-ABI of include/dbw_render.h.
There is no CPU / PyTorch fallback: a missing library or a non-CUDA tensor raises."""
import ctypes
from copy import deepcopy

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import _lib
from ._lib import DbwMapDesc, DbwRenderSettings, DbwError

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
        _lib.check(L.dbw_render_forward_ex(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                           _c(map_table), _c(R), _c(T), _c(fa), _c(out), _c(ids), _c(ws), fwd.value,
                                           _c(shade), _c(dists), _stream()), 'dbw_render_forward_ex')
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
        _lib.check(L.dbw_render_backward(ctypes.byref(s), _c(verts), _c(faces), _c(faces_uvs), _c(face_map), _c(maps),
                                         _c(map_table), _c(R), _c(T), _c(fa), None, _c(ws), ws.numel(), _c(g_out),
                                         _c(g_verts), _c(g_fa), _c(g_maps), _c(scratch), scratch.numel(), _stream()),
                   'dbw_render_backward')
        return g_verts, g_maps, g_fa, None, None, None, None, None, None, None, None, None, None


_TABLE_CACHE = {}


def _device_map_table(table_host, dev):
    """(M) DbwMapDesc on the device, cached per (layout, device): built once, so that steady-state calls do no H2D."""
    key = (tuple(table_host), str(dev))
    if key not in _TABLE_CACHE:
        table = (DbwMapDesc * len(table_host))(*[DbwMapDesc(int(o), int(h), int(w), 0) for o, h, w in table_host])
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


def scene_settings(verts, faces, maps, map_table_host, B, intr, image_size, sigma, faces_per_pixel, z_clip=None,
                   detach_bary=False, clip_inside=True, background=(0., 0., 0.), faces_alpha=None, perspective_correct=True,
                   verts_are_ndc=False, blur_radius=None, maps_are_texels4=False, alpha_group=1, n_static_faces=0, view_rows=None):
    """(DbwRenderSettings, device map table) of one render pass over raw scene tensors.
    alpha_group: faces per opacity entry (faces_alpha then has F / alpha_group [or B * that] entries);
    n_static_faces: leading faces whose vertices are constants (no vertex gradient wanted)."""
    H, W = image_size
    V, Fn = verts.shape[-2], faces.shape[0]
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
                        maps_are_texels4=maps_are_texels4,
                        # what a backward streams: one 16 B record per kept fragment, written only when one may follow
                        save_fragment_state=torch.is_grad_enabled(), alpha_group=alpha_group, n_static_faces=n_static_faces,
                        view_rows=view_rows)
    return cfg, map_table


def render_scene(verts, faces, faces_uvs, face_map, maps, map_table_host, R, T, intr, image_size, sigma, faces_per_pixel,
                 z_clip=None, detach_bary=False, clip_inside=True, background=(0., 0., 0.), faces_alpha=None,
                 perspective_correct=True, verts_are_ndc=False, blur_radius=None, return_ids=False, maps_are_texels4=False,
                 face_shade=None, return_dists=False, alpha_group=1, n_static_faces=0, view_rows=None):
    """Functional form over raw tensors (used by Renderer.forward and by the parity tests).
    verts (V,3) [or (B,V,3) NDC], faces (F,3) int32, faces_uvs (F,3,2), face_map (F) int32, maps flat float buffer,
    map_table_host [(offset,H,W)], R (B,3,3), T (B,3), faces_alpha None | (F,) | (B*F,).
    maps_are_texels4: `maps` is a float4 (RGB+pad) texel atlas from scene_ops.texture_atlas (offsets stay 3*texel)."""
    dev = verts.device
    B = R.shape[0] if R is not None else verts.shape[0]
    cfg, map_table = scene_settings(verts, faces, maps, map_table_host, B, intr, image_size, sigma, faces_per_pixel, z_clip,
                                    detach_bary, clip_inside, background, faces_alpha, perspective_correct, verts_are_ndc,
                                    blur_radius, maps_are_texels4, alpha_group, n_static_faces, view_rows)
    if R is None:
        R = torch.eye(3, device=dev)[None].expand(B, -1, -1)
        T = torch.zeros(B, 3, device=dev)
    res = _RenderFn.apply(verts, maps, faces_alpha, R, T, faces.to(torch.int32).contiguous(),
                          faces_uvs.contiguous().float(), face_map.to(torch.int32).contiguous(), map_table, cfg,
                          face_shade, return_dists, return_ids)
    return res                           # rgba | (rgba, slot ids) | (rgba, slot ids, signed squared distances)


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

    def forward(self, meshes, R, T, viz_purpose=False, **kwargs):
        lit = self.light_kwargs.get('name', 'ambient') == 'directional'
        if self.shading_type not in ('raw', 'flat') or (lit != (self.shading_type == 'flat')):
            raise NotImplementedError(f'shading_type={self.shading_type} with lights={self.light_kwargs.get("name", "ambient")}: '
                                      'only raw+ambient (training) and flat+directional (renderer_light) are implemented')
        faces_alpha = kwargs.get('faces_alpha')
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        H, W = self.img_size
        intr = self.cameras.intrinsics()
        shade = self._flat_shade(verts, faces, R) if lit else None
        if viz_purpose:
            # VizMeshRenderer (renderer.py:56-60,178-183): hard 4x supersampled render, box-filtered, no gradient
            with torch.no_grad():
                out = render_scene(verts, faces, fvu, fmap, maps, table, R, T, intr, (H * 4, W * 4), 0.0, 1, self.z_clip,
                                   self.detach_bary, self.clip_inside, self.background_color, faces_alpha,
                                   self.perspective_correct, face_shade=shade)
                return F.avg_pool2d(out, kernel_size=4, stride=4)
        return render_scene(verts, faces, fvu, fmap, maps, table, R, T, intr, (H, W), self.sigma, self.faces_per_pixel,
                            self.z_clip, self.detach_bary, self.clip_inside, self.background_color, faces_alpha,
                            self.perspective_correct, blur_radius=self.blur_radius, face_shade=shade)

    # ------------------------------------------------------------------ edge overlays (renderer.py:134-175)
    @torch.no_grad()
    def render_edges(self, meshes, R, T, image_size=None, linewidth=1, return_pix2face=False, faces_per_pixel=1):
        """mask of the pixels closer than `linewidth` pixels to an edge of the face(s) they see: a hard rasterization whose
        signed squared NDC distances are thresholded at (linewidth * 2 / min(image_size))^2."""
        image_size = tuple(image_size or self.img_size)
        verts, faces, fvu, fmap, maps, table = self._scene(meshes)
        _, ids, dists = render_scene(verts, faces, fvu, fmap, maps, table, R, T, self.cameras.intrinsics(), image_size, 0.0,
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

    def draw_edges(self, img, meshes, R=None, T=None, colors=None, linewidth=1, antialias=True):
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
        mask, pix2face = self.render_edges(meshes, R, T, image_size=img_size, linewidth=linewidth, return_pix2face=True)
        if colors.dim() == 2:
            face_img = colors.to(mask.device)[pix2face].permute(0, 3, 1, 2)               # one colour per (packed) face
        else:
            face_img = colors.to(mask.device)[:, None, None].expand(-1, *mask.shape[2:])[None].expand(len(mask), -1, -1, -1)
        if antialias:
            mask, face_img = [F.avg_pool2d(t, kernel_size=4, stride=4) for t in [mask, face_img]]
        return img * (1 - mask) + mask * face_img
