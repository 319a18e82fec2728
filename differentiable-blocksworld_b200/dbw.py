"""Scene model of the render hot path: a drop-in for the reference's `DifferentiableBlocksWorld`
(the reference's src/model/dbw.py:38-462) as far as src/trainer.py, src/optimizer.py and configs/*.yml see it --
same constructor kwargs, same parameter / buffer names (checkpoints, the `texture*` Adam group), same
`forward(inp, labels) -> {loss name: tensor}` / `predict(...)` / `build_*` / `get_opacities` surface.

What is different underneath is everything that costs time:
  * leaf parameters -> world-space vertices and float4 texel atlases by two fused kernels (scene_ops.py) instead of
    ~200 eager ops; the background sphere's world vertices are a constant;
  * blocks dropped by the opacity filters stay in the mesh and are DISABLED (face_map = -1): fixed shapes, no host
    synchronisation, so a whole optimisation step replays as one CUDA graph (graph.py);
  * both render passes, compositing and the RGB loss go through the C-ABI kernels (renderer.py).
The reference-shaped `build_bkg / build_ground / build_blocks / build_scene` (returning Meshes) remain for the
visualisation / export call sites (trainer.py:181-198,261-263)."""
import ctypes
from collections import OrderedDict
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, geometry as G, losses as L
from .renderer import Renderer, render_scene, _c, _stream
from .fused_loss import ScenePass, scene_mse
from .scene_ops import (scene_geometry_passes, block_opacities, scene_atlases, scene_texture_cells, atlases_from_cells,
                        cell_map_table)
from .structures import Meshes, TexturesUV, join_meshes_as_scene

# accepted keys and defaults of the config sub-dicts (configs/*/*.yml -> model.{mesh,rend_optim,loss}); unknown keys are
# an error, as in the reference (dbw.py:71,129,157)
MESH_KEYS = dict(n_blocks=1, S_world=1, R_world=(0, 0, 0), T_world=(0., 0., 0.), z_far=10, ratio_block_scene=0.25,
                 txt_size=256, txt_bkg_upscale=1, scale_min=0.2, opacity_init=0.5, T_range=(1, 1, 1), T_init_mode='gauss')
REND_OPTIM_KEYS = dict(opacity_noise=False, decouple_rendering=False, coarse_learning=True, decimate_txt=False,
                       decimate_factor=8, kill_blocks=False)
LOSS_KEYS = dict(rgb_weight=1.0, perceptual_weight=0, parsimony_weight=0, scale_weight=0, tv_weight=0, overlap_weight=0,
                 name='mse', perceptual_name='lpips', tv_type='l2sq')
LIGHT_FOR_SYNTHETIC_VIEWS = {'name': 'directional', 'direction': [[1, 0.25, -1]], 'ambient_color': [[0.7, 0.7, 0.7]],
                             'diffuse_color': [[0.4, 0.4, 0.4]], 'specular_color': [[0., 0., 0.]]}


def _parse(cfg, spec, what):
    cfg = dict(cfg or {})
    out = {k: cfg.pop(k, d) for k, d in spec.items()}
    assert not cfg, f'unknown {what} options: {cfg}'
    return out


class _CompositeMSE(torch.autograd.Function):
    """rec = fg_rgb * fg_a + (1 - fg_a) * env_rgb ; loss = mean((imgs - rec)^2)   (dbw.py:223 + :366-367): one kernel
    forward, one kernel backward (which also folds in a gradient arriving at `rec` from other loss terms)."""

    @staticmethod
    def forward(ctx, fg, env, imgs, n_total_views):
        ctx.set_materialize_grads(False)          # g_rec arrives as None when `rec` is unused: no zero tensors, no sync
        B, _, H, W = fg.shape
        fg, env, imgs = fg.contiguous(), env.contiguous(), imgs.contiguous().float()
        rec = torch.empty(B, 3, H, W, device=fg.device, dtype=torch.float32)
        loss = torch.zeros((), device=fg.device, dtype=torch.float32)
        inv = 1.0 / (float(n_total_views) * 3 * H * W)
        _lib.check(_lib.lib().dbw_composite_mse(B, H, W, _c(fg), _c(env), _c(imgs), ctypes.c_float(inv), _c(rec), _c(loss),
                                                None, None, _stream()), 'dbw_composite_mse')
        ctx.save_for_backward(fg, env, imgs)
        ctx.inv = inv
        return rec, loss

    @staticmethod
    def backward(ctx, g_rec, g_loss):
        fg, env, imgs = ctx.saved_tensors
        B, _, H, W = fg.shape
        g_fg, g_env = torch.empty_like(fg), torch.empty_like(env)
        gl = g_loss.contiguous().float() if g_loss is not None else None
        gr = g_rec.contiguous().float() if g_rec is not None else None
        _lib.check(_lib.lib().dbw_composite_mse_backward(B, H, W, _c(fg), _c(env), _c(imgs), ctypes.c_float(ctx.inv), _c(gl),
                                                         _c(gr), _c(g_fg), _c(g_env), _stream()), 'dbw_composite_mse_backward')
        return g_fg, g_env, None, None


class DifferentiableBlocksWorld(nn.Module):
    name = 'dbw'

    def __init__(self, img_size, **kwargs):
        super().__init__()
        self._init_kwargs = dict(deepcopy(kwargs), img_size=img_size)
        mesh = _parse(kwargs.get('mesh'), MESH_KEYS, 'mesh')
        sched = _parse(kwargs.get('rend_optim'), REND_OPTIM_KEYS, 'rend_optim')
        loss = _parse(kwargs.get('loss'), LOSS_KEYS, 'loss')

        for k in ('n_blocks', 'S_world', 'z_far', 'ratio_block_scene', 'txt_size', 'txt_bkg_upscale', 'scale_min'):
            setattr(self, k, mesh[k])
        self._build_template(mesh['R_world'], mesh['T_world'])
        self._build_parameters(mesh['opacity_init'], mesh['T_range'], mesh['T_init_mode'])
        self._build_renderers(img_size, kwargs.get('renderer', {}))

        # training schedule switches: bool, or the epoch from which the feature is OFF (is_live)
        self.opacity_noise, self.decouple_rendering = sched['opacity_noise'], sched['decouple_rendering']
        self.coarse_learning, self.decimate_txt = sched['coarse_learning'], sched['decimate_txt']
        self.decim_factor, self.kill_blocks = sched['decimate_factor'], sched['kill_blocks']

        weights = {k[:-len('_weight')]: loss[k] for k in ('rgb_weight', 'perceptual_weight', 'parsimony_weight',
                                                          'scale_weight', 'tv_weight', 'overlap_weight')}
        self.loss_weights = {k: w for k, w in weights.items() if w > 0}
        self.loss_names = [f'loss_{k}' for k in self.loss_weights] + ['loss_total']
        self.tv_norm = L.TV_NORMS[loss['tv_type']]
        self.criterion = {'mse': nn.MSELoss, 'l2': nn.MSELoss, 'l1': nn.L1Loss}[loss['name']]()
        if 'perceptual' in self.loss_weights:
            # LPIPS is a VGG16 conv network (cuDNN / tensor cores): outside the render hot path (SURVEY 8a row a13);
            # any callable (imgs, rec) -> scalar can be installed with set_perceptual_loss()
            self.perceptual_loss = _make_perceptual(loss['perceptual_name'])
        self.cur_epoch = 0

        # execution options of this implementation
        self.static_topology = True       # disable filtered blocks via face_map = -1 instead of slicing (no host sync)
        self.fused_scene = True           # scene_ops kernels for mesh build + texture prep
        self.fused_loss = True            # compositing + MSE in the rasterizer's epilogue (fused_loss.py) when nothing else reads rec
        self._passes = None
        self.alpha_group_faces = None     # None: one opacity entry per block (alpha_group = BNF); 1: one per face, as dbw.py:219 packs them
        self.n_total_views = None         # data-parallel context (parallel.py): views of the whole step
        self.grad_sum_point = None        # likewise: parallel.GradSumPoint, sums the scene tensors' gradients over ranks inside the backward
        self.noise_generator = None       # RNG shared by all ranks for opacity noise / overlap samples
        self.opacity_noise_buffer = None  # pre-drawn randn (N,) used instead of drawing inside forward (graph.py)
        self.overlap_samples_buffer = None  # pre-drawn U(0,1) (N,1000,3) for the overlap term, likewise
        self._static = None
        self._reg_state_stale = False

    # ------------------------------------------------------------------ construction
    def _build_template(self, R_world, T_world):
        """static topology: inward-facing background icosphere (level 2, radius z_far), ground plane subdivided 3x,
        N block icospheres (level 1) with seam/pole-fixed spherical UVs padded circularly along u (dbw.py:73-96)"""
        N, TS = self.n_blocks, self.txt_size
        self.register_buffer('R_world', G.euler_world_rotation(*R_world))
        self.register_buffer('T_world', torch.tensor([float(t) for t in T_world])[None])
        sphere_v, sphere_f = G.ico_sphere(2)
        self.bkg = Meshes((sphere_v * self.z_far)[None], sphere_f.flip(1)[None])
        self.register_buffer('bkg_verts_uvs', G.spherical_uv(self.bkg.verts_packed()))
        plane_v, plane_f = G.unit_plane()
        plane_v = plane_v * torch.tensor([self.z_far, 1., self.z_far])
        for _ in range(3):
            plane_v, plane_f = G.subdivide_mesh(plane_v, plane_f)
        self.ground = Meshes(plane_v[None], plane_f[None])
        self.register_buffer('ground_verts_uvs', (plane_v[:, [0, 2]] / self.z_far + 1) / 2)
        unit_v, unit_f = G.ico_sphere(1)
        self.blocks = Meshes((unit_v * self.ratio_block_scene).expand(N, -1, -1).clone(), unit_f.expand(N, -1, -1).clone())
        local = self.blocks.verts_padded() / self.ratio_block_scene
        self.register_buffer('sq_eta', torch.asin(local[..., 1]))
        self.register_buffer('sq_omega', torch.atan2(local[..., 0], local[..., 2]))
        faces_uvs, uvs = G.icosphere_uvs(1)
        u_lo, u_hi = uvs[:, 0].min().item(), uvs[:, 0].max().item()
        pad_left, pad_right = abs(int(np.floor(u_lo * TS))), int(np.ceil((u_hi - 1) * TS))
        self.txt_padding = (pad_left, pad_right)
        self.BNF = len(faces_uvs)
        self.register_buffer('block_faces_uvs', faces_uvs)
        self.register_buffer('block_verts_uvs', torch.stack([(uvs[:, 0] * TS + pad_left) / (TS + pad_left + pad_right), uvs[:, 1]], -1))

    def _build_parameters(self, opacity_init, T_range, T_init_mode):
        """leaf parameters, initialised as dbw.py:84,98-119 (random draws in the same order: S, rotations, T, textures)"""
        N, TS, up = self.n_blocks, self.txt_size, self.txt_bkg_upscale
        T_range = torch.tensor([float(t) for t in T_range])
        self.sq_eps = nn.Parameter(torch.zeros(N, 2))
        self.R_6d_ground = nn.Parameter(torch.tensor([[1., 0., 0., 0., 1., 0.]]))
        self.T_ground = nn.Parameter(torch.tensor([[0., -0.9 * T_range[1].item(), 0.]]))
        self.S = nn.Parameter((torch.rand(N, 3) + 0.5 - self.scale_min).log())
        self.R_6d = nn.Parameter(G.matrix_to_rotation_6d(G.random_rotations(N)))
        if T_init_mode == 'gauss':
            T0 = torch.randn(N, 3) / 2 * T_range
        elif T_init_mode == 'uni':
            T0 = (2 * torch.rand(N, 3) - 1) * T_range
        else:
            raise NotImplementedError(T_init_mode)
        self.T = nn.Parameter(T0)
        self.alpha_logit = nn.Parameter(torch.logit(torch.full((N,), float(opacity_init))) + 1e-3)
        self.texture_bkg = nn.Parameter(torch.randn(1, TS * up, TS * up, 3) / 10)
        self.texture_ground = nn.Parameter(torch.randn(1, TS * up, TS * up, 3) / 10)
        self.textures = nn.Parameter(torch.randn(N, TS, TS, 3) / 10)

    def _build_renderers(self, img_size, cfg):
        """the four renderers of dbw.py:131-143: coarse (config sigma), fine (5e-6), environment (hard, K=1, gradients
        through barycentrics), and the lit flat-shaded one for synthetic-colour views"""
        variants = OrderedDict([
            ('renderer', {}),
            ('renderer_fine', {'sigma': 5e-6}),
            ('renderer_env', {'sigma': 0, 'faces_per_pixel': 1, 'detach_bary': False}),
            ('renderer_light', {'sigma': 0, 'faces_per_pixel': 1, 'detach_bary': False, 'lights': LIGHT_FOR_SYNTHETIC_VIEWS,
                                'shading_type': 'flat', 'background_color': (1, 1, 1)}),
        ])
        for attr, override in variants.items():
            setattr(self, attr, Renderer(img_size, **dict(deepcopy(cfg), **deepcopy(override))))

    def _renderers(self):
        return self.renderer, self.renderer_fine, self.renderer_env, self.renderer_light

    @property
    def init_kwargs(self):
        return deepcopy(self._init_kwargs)

    def set_perceptual_loss(self, fn):
        """fn(imgs, rec) -> scalar: an nn.Module (registered, follows .to() / state_dict) or any callable"""
        if isinstance(getattr(self, 'perceptual_loss', None), nn.Module) and not isinstance(fn, nn.Module):
            del self.perceptual_loss
        self.perceptual_loss = fn

    def cache_perceptual_targets(self, imgs_or_dataset):
        """register the training images with the installed PerceptualTerm(perceptual.LPIPS): later steps read their LPIPS
        taps from a device cache instead of recomputing them, with the same results bit for bit (images not in the cache
        are computed as before).  imgs_or_dataset: an (N,3,H,W) tensor, or an iterable of (3,H,W) / (B,3,H,W) tensors or
        of dicts holding them under 'imgs' (the reference's datasets).  Returns the cache's device bytes.  A GraphedStep
        captured before this call keeps computing its targets: build the step after registering."""
        from .perceptual import LPIPS
        term = getattr(self, 'perceptual_loss', None)
        net = getattr(term, 'loss', None)
        if not (isinstance(term, PerceptualTerm) and isinstance(net, LPIPS)):
            raise TypeError('cache_perceptual_targets: the installed perceptual term is not PerceptualTerm(dbw_b200.perceptual.LPIPS) '
                            f'(got {type(term).__name__}); install one with set_perceptual_loss()')
        if torch.is_tensor(imgs_or_dataset):
            imgs = imgs_or_dataset
        else:
            items = [x['imgs'] if isinstance(x, dict) else x for x in imgs_or_dataset]
            imgs = torch.cat([x.detach().reshape(-1, *x.shape[-3:]).to(net.scaling_layer.shift.device) for x in items])
        net.cache_targets(imgs.detach().to(net.scaling_layer.shift.device), normalize=True)
        return net.target_cache_bytes(imgs.shape[-2], imgs.shape[-1], len(imgs))

    def set_cur_epoch(self, epoch):
        self.cur_epoch = epoch

    def step(self):
        self.cur_epoch += 1

    def is_live(self, name):
        switch = getattr(self, name)
        return switch if isinstance(switch, bool) else self.cur_epoch < switch

    def to(self, device):
        super().to(device)
        self.bkg, self.ground, self.blocks = self.bkg.to(device), self.ground.to(device), self.blocks.to(device)
        for r in self._renderers():
            r.to(device)
        return self

    bkg_n_faces = property(lambda self: int(self.bkg.num_faces_per_mesh().sum()))
    ground_n_faces = property(lambda self: int(self.ground.num_faces_per_mesh().sum()))
    env_n_faces = property(lambda self: self.bkg_n_faces + self.ground_n_faces)
    blocks_n_faces = property(lambda self: int(self.blocks.num_faces_per_mesh().sum()))

    # ------------------------------------------------------------------ one step
    def forward(self, inp, labels=None):
        imgs = inp['imgs']
        if inp.get('rows') is not None and not self._fused_loss_ok(imgs):
            raise NotImplementedError("inp['rows'] (row-band sharding, parallel.py) needs the fused-loss path: decoupled rendering, "
                                      'MSE, no perceptual term')
        if self._fused_loss_ok(imgs):
            return self.compute_losses(imgs, None, rgb_loss=self._scene_mse_fused(inp))
        env_rgba, fg_rgba = self._render_layers(inp)
        n_total = self.n_total_views or len(imgs)
        if fg_rgba is not None and isinstance(self.criterion, nn.MSELoss) and imgs.is_cuda:
            rec, mse = _CompositeMSE.apply(fg_rgba, env_rgba, imgs, n_total)
            return self.compute_losses(imgs, rec, rgb_loss=mse)
        rec = self._composite(env_rgba, fg_rgba)
        return self.compute_losses(imgs, rec, rgb_loss=self.criterion(imgs, rec) * (len(imgs) / float(n_total)))

    def _install_cameras(self, inp):
        """dbw.py:204-208: the first batch's intrinsics become the cameras of all four renderers"""
        if 'K' in inp and self.renderer.cameras.K is None:
            for r in self._renderers():
                r.update_cameras(device=inp['imgs'].device, K=inp['K'][0:1])
                r.cameras.intrinsics()          # the one host read of K happens here, never inside a step

    def _phase(self, filter_transparent=False):
        fine = not self.is_live('coarse_learning')
        return fine, (filter_transparent or fine), (self.renderer_fine if fine else self.renderer)

    def _render_layers(self, inp, filter_transparent=False):
        """(environment RGBA, blocks RGBA) in decoupled mode (every shipped config), (whole-scene RGBA, None) otherwise"""
        B, R, T = len(inp['imgs']), inp['R'], inp['T']
        self._install_cameras(inp)
        fine, hard_filter, renderer = self._phase(filter_transparent)
        if not self.decouple_rendering:
            scene = self.build_scene(filter_transparent=hard_filter)
            alpha = None
            if not hard_filter:
                alpha = torch.cat([torch.ones(self.env_n_faces, device=R.device), self._alpha.repeat_interleave(self.BNF)])
            return renderer(scene.extend(B), R=R, T=T, faces_alpha=alpha), None
        if self._fused_scene_ok(R):
            return self._render_decoupled_fused(R, T, hard_filter, renderer)
        env = join_meshes_as_scene([self.build_bkg(world_coord=True), self.build_ground(world_coord=True)])
        env_rgba = self.renderer_env(env.extend(B), R=R, T=T)
        if self.static_topology:
            verts, faces, fvu, fmap, maps, table = self._blocks_static(hard_filter)
            alpha = None if hard_filter else self._alpha.repeat_interleave(self.BNF)
            return env_rgba, self._raster(renderer, verts, faces, fvu, fmap, maps, table, R, T, alpha, texels4=False)
        blocks = self.build_blocks(filter_transparent=hard_filter, as_scene=True)
        if len(blocks) == 0:
            return env_rgba, torch.zeros_like(env_rgba)
        alpha = None if hard_filter else self._alpha.repeat_interleave(self.BNF)
        return env_rgba, renderer(blocks.extend(B), R=R, T=T, faces_alpha=alpha)

    def _fused_scene_ok(self, ref):
        """the fused scene kernels apply: static topology on the GPU, and a box decimation the texture-prep kernel has
        (factor 8, the value of every shipped config; others go through the eager F.avg_pool2d path of _maps)"""
        decim_live = self.training and self.is_live('decimate_txt')
        return (self.static_topology and self.fused_scene and ref.is_cuda and (not decim_live or self.decim_factor in (1, 8)))

    @staticmethod
    def _raster(r, verts, faces, fvu, fmap, maps, table, R, T, alpha, texels4, alpha_group=1, n_static_faces=0):
        return render_scene(verts, faces, fvu, fmap, maps, table, R, T, r.cameras.intrinsics(), r.img_size, r.sigma,
                            r.faces_per_pixel, r.z_clip, r.detach_bary, r.clip_inside, r.background_color, alpha,
                            r.perspective_correct, blur_radius=r.blur_radius, maps_are_texels4=texels4,
                            alpha_group=alpha_group, n_static_faces=n_static_faces)

    @staticmethod
    def _composite(env_rgba, fg_rgba):
        if fg_rgba is None:
            return env_rgba[:, :3]
        cover = fg_rgba[:, 3:]
        return fg_rgba[:, :3] * cover + (1 - cover) * env_rgba[:, :3]          # dbw.py:223

    # ------------------------------------------------------------------ fused / static scene construction
    def _static_arrays(self):
        """device-side constants of the scene: face / UV / map-index arrays of both passes, the background sphere's
        world vertices, and the constants of the geometry kernel"""
        dev = self.alpha_logit.device
        if self._static is None or self._static['dev'] != dev:
            N, Vb = self.n_blocks, self.sq_eta.shape[1]
            gv, gf = self.ground.get_mesh_verts_faces(0)
            bv, bf = self.bkg.get_mesh_verts_faces(0)
            geom = dict(n_blocks=N, verts_per_block=Vb, n_ground_verts=gv.shape[0], sq_eta=self.sq_eta.contiguous(),
                        sq_omega=self.sq_omega.contiguous(), ground_verts=gv.contiguous().float(),
                        ratio=float(self.ratio_block_scene), scale_min=float(self.scale_min), S_world=float(self.S_world),
                        R_world=[float(x) for x in self.R_world.flatten().cpu()], T_world=[float(x) for x in self.T_world.flatten().cpu()])
            offsets = (torch.arange(N, device=dev) * Vb)[:, None, None]
            self._static = dict(
                dev=dev, geom=geom, bkg_world=self._to_world(bv[None])[0].contiguous(),
                faces_b=(self.blocks.faces_padded() + offsets).reshape(-1, 3).to(torch.int32).contiguous(),
                fvu_b=self.block_verts_uvs[self.block_faces_uvs].expand(N, -1, -1, -1).reshape(-1, 3, 2).contiguous(),
                fmap_b=torch.arange(N, device=dev, dtype=torch.int32).repeat_interleave(self.BNF),
                faces_e=torch.cat([bf, gf + bv.shape[0]]).to(torch.int32).contiguous(),
                fvu_e=torch.cat([self.bkg_verts_uvs[bf], self.ground_verts_uvs[gf]]).contiguous(),
                fmap_e=torch.cat([torch.zeros(len(bf)), torch.ones(len(gf))]).to(dev).to(torch.int32),
                minus_one=torch.full((), -1, dtype=torch.int32, device=dev))
        return self._static

    def _fused_arrays(self):          # name used by tests / scene_ops callers
        return self._static_arrays()

    def _opacities(self, hard_filter, coarse_training):
        """per-block opacities (+ exploration noise while coarse) and the face_map that disables filtered blocks
        (dbw.py:300-316 with static shapes); written for few launches: it runs every step"""
        st = self._static_arrays()
        noisy = bool(self.opacity_noise) and coarse_training
        if self.fused_scene and self.alpha_logit.is_cuda:
            thr = 0.5 if hard_filter else (0.01 if self.kill_blocks else -1.0)
            self._alpha, self._alpha_full, fmap = block_opacities(self.alpha_logit, self._draw_opacity_noise() if noisy else None,
                                                                  float(self.opacity_noise) if noisy else 0.0, thr, st['fmap_b'], self.BNF)
            return fmap
        logit = self.alpha_logit
        if noisy:
            logit = torch.add(logit, self._draw_opacity_noise(), alpha=float(self.opacity_noise))
        self._alpha = torch.sigmoid(logit)
        self._alpha_full = self._alpha
        fmap = st['fmap_b']
        if hard_filter or self.kill_blocks:
            with torch.no_grad():
                keep = torch.sigmoid(self.alpha_logit) > (0.5 if hard_filter else 0.01)
                fmap = torch.where(keep[:, None], fmap.view(self.n_blocks, self.BNF), st['minus_one']).reshape(-1)
            self._alpha_full = self._alpha * keep
        return fmap

    def _draw_opacity_noise(self):
        if self.opacity_noise_buffer is not None:
            return self.opacity_noise_buffer
        if self.noise_generator is not None:
            return torch.randn(self.alpha_logit.shape, generator=self.noise_generator, device=self.alpha_logit.device)
        return torch.randn_like(self.alpha_logit)

    def _scene_tensors(self, hard_filter, cells=False):
        """leaf parameters -> scene kernels -> raw tensors of the two passes:
        (env verts, env atlas, env map table), (block verts, block atlas, block map table, face_map, per-face opacities).
        cells: while both texture stacks are box-decimated 8x, the "atlases" are the float4 CELLS of scene_texture_cells and the
        tables describe cell maps -- the passes sample and scatter at the cells (64x fewer texels, no atlas expansion either
        way); the renders are bit for bit those of the atlases"""
        st = self._static_arrays()
        coarse_training = self.training and self.is_live('coarse_learning')
        decim_env = self.decim_factor if (self.training and self.is_live('decimate_txt')) else 1
        decim_blocks = self.decim_factor if (coarse_training and self.is_live('decimate_txt')) else 1
        # environment vertices = constant background sphere + posed ground; both passes' arrays come out of one launch
        blk_verts, env_verts = scene_geometry_passes(self.sq_eps, self.S, self.R_6d, self.T, self.R_6d_ground, self.T_ground,
                                                     st['geom'], st['bkg_world'])
        fmap = self._opacities(hard_filter, coarse_training)
        alpha = None if hard_filter else self._alpha          # one opacity per block: alpha_group = BNF faces share an entry
        side = self.texture_bkg.shape[1]
        cells = cells and decim_env == 8 and decim_blocks == 8
        if cells or (self.grad_sum_point is not None and decim_env == 8 and decim_blocks == 8):
            cells_env, cells_blk = scene_texture_cells(self.texture_bkg, self.texture_ground, self.textures, decim_env, decim_blocks,
                                                       texels4=cells)
            if self.grad_sum_point is not None:
                # data parallel: everything the two raster passes differentiate goes through ONE gradient-sum point, textures
                # as their decimated cells (parallel.GradSumPoint); what lies before it turns summed gradients into leaf gradients
                summed = self.grad_sum_point(blk_verts, env_verts, cells_env, cells_blk, *([alpha] if alpha is not None else []))
                blk_verts, env_verts, cells_env, cells_blk = summed[:4]
                alpha = summed[4] if alpha is not None else None
            if cells:
                env_atlas, atlas = cells_env, cells_blk
                env_table = cell_map_table(2, side, decim_env)
                table = cell_map_table(self.n_blocks, self.textures.shape[1], decim_blocks, *self.txt_padding)
                self._reg_state_stale = True
                return (env_verts, env_atlas.reshape(-1, 4), env_table), (blk_verts, atlas.reshape(-1, 4), table, fmap,
                                                                         self._per_face_alpha(alpha))
            env_atlas, atlas = atlases_from_cells(cells_env, cells_blk, self.txt_padding, decim_env, decim_blocks)
        else:
            env_atlas, atlas = scene_atlases(self.texture_bkg, self.texture_ground, self.textures, self.txt_padding, decim_env, decim_blocks)
        env_atlas = env_atlas.reshape(-1, 4)
        env_table = [(0, side, side), (side * side * 3, side, side)]
        rows, cols = atlas.shape[1], atlas.shape[2]
        table = [(i * rows * cols * 3, rows, cols) for i in range(self.n_blocks)]
        self._reg_state_stale = True          # compute_losses() rebuilds what the regularisers read, if they are on
        return (env_verts, env_atlas, env_table), (blk_verts, atlas.reshape(-1, 4), table, fmap, self._per_face_alpha(alpha))

    def _per_face_alpha(self, alpha):
        if alpha is not None and self.alpha_group_faces == 1:
            alpha = alpha[:, None].expand(-1, self.BNF).reshape(-1)
        return alpha

    def _render_decoupled_fused(self, R, T, hard_filter, renderer):
        """environment pass + blocks pass over the fused scene tensors -> (env RGBA, blocks RGBA)"""
        st = self._static_arrays()
        (env_verts, env_atlas, env_table), (blk_verts, atlas, table, fmap, alpha) = self._scene_tensors(hard_filter)
        env_rgba = self._raster(self.renderer_env, env_verts, st['faces_e'], st['fvu_e'], st['fmap_e'], env_atlas, env_table,
                                R, T, None, texels4=True, n_static_faces=self.bkg_n_faces)
        fg_rgba = self._raster(renderer, blk_verts, st['faces_b'], st['fvu_b'], fmap, atlas, table, R, T, alpha, texels4=True,
                               alpha_group=self.alpha_group_faces or self.BNF)
        return env_rgba, fg_rgba

    def _fused_loss_ok(self, imgs):
        """the loss epilogue of the rasterizer applies: decoupled static scene on the GPU, plain MSE, nothing else reads `rec`"""
        return (self.fused_loss and self.decouple_rendering and self._fused_scene_ok(imgs)
                and isinstance(self.criterion, nn.MSELoss) and 'rgb' in self.loss_weights
                and not ('perceptual' in self.loss_weights and self.perceptual_loss is not None))

    def _scene_mse_fused(self, inp):
        """render both layers, composite and take the MSE inside the rasterizer (fused_loss.scene_mse)"""
        self._install_cameras(inp)
        _, hard_filter, renderer = self._phase()
        st = self._static_arrays()
        (env_verts, env_atlas, env_table), (blk_verts, atlas, table, fmap, alpha) = self._scene_tensors(hard_filter, cells=True)
        key = (id(renderer), id(st['faces_b']), tuple(env_table), tuple(table))
        if self._passes is None or self._passes[0] != key:
            self._passes = (key, ScenePass(st['faces_e'], st['fvu_e'], st['fmap_e'], env_table, self.renderer_env,
                                           n_static_faces=self.bkg_n_faces),
                            ScenePass(st['faces_b'], st['fvu_b'], st['fmap_b'], table, renderer, alpha_group=self.alpha_group_faces or self.BNF))
        # data parallel with pose gradients: the poses are this rank's slices of pose leaves that went through the sum point
        R, T = self.grad_sum_point.cameras(inp) if self.grad_sum_point is not None else (inp['R'], inp['T'])
        return scene_mse(env_verts, env_atlas, blk_verts, atlas, alpha, R, T, inp['imgs'], self._passes[1],
                         self._passes[2], fmap, n_total_views=self.n_total_views or len(inp['imgs']), view_rows=inp.get('rows'))

    def can_sum_gradients_at_scene_tensors(self, imgs):
        """the step's gradients may be summed over data-parallel ranks at the scene tensors (vertices, opacities, texture CELLS)
        instead of at the leaves: fused-loss path, and both texture stacks box-decimated (the cells are then 64x smaller than
        the texture parameters; undecimated they are as large and the leaf all-reduce is used)"""
        return (self._fused_loss_ok(imgs) and self.training and self.is_live('decimate_txt') and self.is_live('coarse_learning')
                and self.decim_factor == 8)

    def grad_sum_floats(self):
        """floats a parallel.GradSumPoint moves per step (vertices of both passes, decimated cells of all maps, opacities)"""
        f = self.decim_factor
        ts, side = self.textures.shape[1], self.texture_bkg.shape[1]
        cells = (self.n_blocks * (ts // f) ** 2 + 2 * (side // f) ** 2) * 4          # float4 cells (scene_texture_cells(texels4=True))
        verts = (self.n_blocks * self.sq_eta.shape[1] + self.bkg.verts_packed().shape[0] + self.ground.verts_packed().shape[0]) * 3
        return cells + verts + self.n_blocks + 8

    def _blocks_static(self, hard_filter):
        """eager (PyTorch ops) construction of the blocks scene with fixed shapes -- the reference's arithmetic
        (dbw.py:299-344) minus the slicing: filtered blocks are disabled through face_map"""
        st = self._static_arrays()
        coarse_training = self.training and self.is_live('coarse_learning')
        fmap = self._opacities(hard_filter, coarse_training)
        S, R, T = self._pose()
        verts = self._to_world(torch.bmm(self.get_blocks_verts() * S[:, None], R) + T[:, None]).reshape(-1, 3)
        maps = self._maps(self.textures, decimate=coarse_training and self.is_live('decimate_txt'), pad=self.txt_padding)
        self._blocks_maps, self._blocks_SRT = torch.sigmoid(self.textures), (S, R, T)
        rows, cols = maps.shape[1], maps.shape[2]
        table = [(i * rows * cols * 3, rows, cols) for i in range(self.n_blocks)]
        return verts, st['faces_b'], st['fvu_b'], fmap, maps.reshape(-1), table

    # ------------------------------------------------------------------ reference-shaped builders (Meshes objects)
    def _pose(self):
        return self.S.exp() + self.scale_min, G.rotation_6d_to_matrix(self.R_6d), self.T

    def _to_world(self, verts):
        return (verts * self.S_world) @ self.R_world + self.T_world[:, None]

    def _maps(self, logits, decimate=False, pad=(0, 0), synthetic=None):
        """sigmoid -> optional box decimation (avg-pool + nearest upsample, dbw.py:331-334) -> circular u padding"""
        maps = torch.sigmoid(logits) if synthetic is None else synthetic
        if decimate:
            f = self.decim_factor
            maps = F.interpolate(F.avg_pool2d(maps.permute(0, 3, 1, 2), f, f), scale_factor=f).permute(0, 2, 3, 1)
        if pad[0] or pad[1]:
            maps = F.pad(maps.permute(0, 3, 1, 2), pad=(pad[0], pad[1], 0, 0), mode='circular').permute(0, 2, 3, 1)
        return maps.contiguous()

    def get_blocks_verts(self):
        eps = self.sq_eps.sigmoid() * 1.8 + 0.1
        self._blocks_eps = eps[:, :1], eps[:, 1:]
        return G.superquadric_points(self.sq_eta, self.sq_omega, *self._blocks_eps) * self.ratio_block_scene

    def _env_part(self, mesh, verts_uvs, logits, verts, world_coord, synthetic_colors):
        faces = mesh.get_mesh_verts_faces(0)[1][None]
        if world_coord:
            verts = self._to_world(verts)
        synthetic = torch.ones_like(logits) if synthetic_colors else None
        maps = self._maps(logits, decimate=self.training and self.is_live('decimate_txt'), synthetic=synthetic)
        return Meshes(verts, faces, textures=TexturesUV(maps, faces, verts_uvs[None], align_corners=True))

    def build_bkg(self, reduced=False, world_coord=False, synthetic_colors=False):
        verts = self.bkg.get_mesh_verts_faces(0)[0][None]
        if reduced:
            verts = verts * 3 / self.z_far
        self._bkg_maps = torch.sigmoid(self.texture_bkg)
        return self._env_part(self.bkg, self.bkg_verts_uvs, self.texture_bkg, verts, world_coord, synthetic_colors)

    def build_ground(self, reduced=False, world_coord=False, synthetic_colors=False):
        verts = self.ground.get_mesh_verts_faces(0)[0][None]
        if reduced:
            verts = verts * torch.tensor([3 / self.z_far, 1, 3 / self.z_far], device=verts.device)
        verts = verts @ G.rotation_6d_to_matrix(self.R_6d_ground) + self.T_ground[:, None]
        self._ground_maps = torch.sigmoid(self.texture_ground)
        return self._env_part(self.ground, self.ground_verts_uvs, self.texture_ground, verts, world_coord, synthetic_colors)

    def build_blocks(self, filter_transparent=False, world_coord=False, as_scene=False, synthetic_colors=False):
        """Meshes of the (kept) blocks, sliced like the reference (dbw.py:297-346): host-synchronising, used by the
        visualisation / export call sites; the training step goes through _render_decoupled_fused / _blocks_static"""
        coarse_training = self.training and self.is_live('coarse_learning')
        self._opacities(False, coarse_training)
        S, R, T = self._pose()
        verts = torch.bmm(self.get_blocks_verts() * S[:, None], R) + T[:, None]
        faces = self.blocks.faces_padded()
        synthetic = None
        if synthetic_colors:
            shades = G.fancy_cmap()(torch.linspace(0, 1, self.n_blocks + 1)[1:].numpy())
            synthetic = torch.from_numpy(shades).float().to(verts.device)[:, None, None].expand(-1, self.txt_size, self.txt_size, -1)
        logits = self.textures
        self._blocks_maps, self._blocks_SRT = torch.sigmoid(self.textures), (S, R, T)
        n_kept = self.n_blocks
        if filter_transparent or self.kill_blocks:
            keep = torch.sigmoid(self.alpha_logit) > (0.5 if filter_transparent else 0.01)
            self._alpha_full = self._alpha_full * keep
            n_kept = int(keep.sum())
            if n_kept == 0:
                return Meshes([], [])
            verts, faces, logits, self._alpha = verts[keep], faces[keep], logits[keep], self._alpha[keep]
            synthetic = synthetic[keep] if synthetic is not None else None
        maps = self._maps(logits, decimate=coarse_training and self.is_live('decimate_txt'), pad=self.txt_padding, synthetic=synthetic)
        if world_coord or as_scene:
            verts = self._to_world(verts)
        txt = TexturesUV(maps, self.block_faces_uvs.expand(n_kept, -1, -1), self.block_verts_uvs.expand(n_kept, -1, -1), align_corners=True)
        blocks = Meshes(verts, faces, textures=txt)
        return join_meshes_as_scene(blocks) if as_scene else blocks

    def build_scene(self, filter_transparent=False, w_bkg=True, reduce_ground=False, synthetic_colors=False):
        parts = [self.build_bkg(synthetic_colors=synthetic_colors)] if w_bkg else []
        parts.append(self.build_ground(reduced=reduce_ground, synthetic_colors=synthetic_colors))
        blocks = self.build_blocks(filter_transparent, synthetic_colors=synthetic_colors)
        if len(blocks) > 0:
            parts.append(blocks)
        scene = join_meshes_as_scene(parts)
        verts, faces = scene.get_mesh_verts_faces(0)
        return Meshes(self._to_world(verts[None]), faces[None], scene.textures)

    # ------------------------------------------------------------------ prediction / visualisation
    def predict(self, inp, labels=None, w_edges=False, filter_transparent=False):
        rec = self._composite(*self._render_layers(inp, filter_transparent))
        if w_edges:                                   # dbw.py:234-238: coloured face edges drawn over the reconstruction
            B = len(inp['imgs'])
            _, hard_filter, renderer = self._phase(filter_transparent)
            parts = [self.build_bkg(world_coord=True), self.build_ground(world_coord=True)]
            blocks = self.build_blocks(filter_transparent=hard_filter, as_scene=True)
            if len(blocks) > 0:
                parts.append(blocks)
            colors = self.get_scene_face_colors(filter_transparent=hard_filter).repeat(B, 1)
            rec = renderer.draw_edges(rec, join_meshes_as_scene(parts).extend(B), inp['R'], inp['T'], colors=colors)
        return rec

    def predict_synthetic(self, inp, labels=None):
        """flat-shaded render of the opaque blocks with one synthetic colour per block (dbw.py:241-248)"""
        self._install_cameras(inp)
        blocks = self.build_blocks(filter_transparent=True, synthetic_colors=True, as_scene=True)
        if len(blocks) == 0:
            return torch.ones_like(inp['imgs'])
        return self.renderer_light(blocks.extend(len(inp['imgs'])), R=inp['R'], T=inp['T'], viz_purpose=True)[:, :3]

    @torch.no_grad()
    def get_scene_face_colors(self, filter_transparent=False, w_env=True):
        """one colour per scene face: environment faces the map's first colour, block k the colour at (k+1)/N (dbw.py:420-431)"""
        values = torch.linspace(0, 1, self.n_blocks + 1)[1:]
        if filter_transparent or self.kill_blocks:
            values = values[self.get_opacities().cpu() > (0.5 if filter_transparent else 0.01)]
        values = torch.cat([torch.zeros(self.env_n_faces if w_env else 0), values.repeat_interleave(self.BNF)])
        return torch.from_numpy(G.fancy_cmap()(values.numpy())).float().to(self.bkg.device)

    @torch.no_grad()
    def get_arranged_block_txt(self):
        """the block textures tiled 5 per row, (1,3,rows*TS,5*TS) (dbw.py:433-438)"""
        maps = torch.sigmoid(self.textures).permute(0, 3, 1, 2)
        rows = [torch.cat(list(maps[5 * i:5 * i + 5]), dim=2) for i in range(len(maps) // 5)]
        return torch.cat(rows, dim=1)[None]

    def get_opacities(self):
        alpha = torch.sigmoid(self.alpha_logit)
        return alpha * (alpha > 0.01) if self.kill_blocks else alpha

    @torch.no_grad()
    def get_nb_opaque_blocks(self):
        return int((self.get_opacities() > 0.5).sum())

    # ------------------------------------------------------------------ objective (dbw.py:361-408)
    def _refresh_reg_state(self):
        if self._reg_state_stale:
            self._blocks_maps = torch.sigmoid(self.textures)
            self._bkg_maps, self._ground_maps = torch.sigmoid(self.texture_bkg), torch.sigmoid(self.texture_ground)
            self._blocks_SRT = self._pose()
            eps = self.sq_eps.sigmoid() * 1.8 + 0.1
            self._blocks_eps = eps[:, :1], eps[:, 1:]
            self._reg_state_stale = False

    def compute_losses(self, imgs, rec, rgb_loss=None):
        coarse = self.is_live('coarse_learning')
        w = self.loss_weights
        if 'tv' in w or 'overlap' in w:
            self._refresh_reg_state()
        terms = {}
        if 'rgb' in w:
            rgb = rgb_loss if rgb_loss is not None else self.criterion(imgs, rec)
            terms['rgb'] = rgb if w['rgb'] == 1 else w['rgb'] * rgb
        if 'perceptual' in w and self.perceptual_loss is not None:
            terms['perceptual'] = w['perceptual'] * (1 if coarse else 0.1) * self.perceptual_loss(imgs, rec)
        if 'parsimony' in w:
            terms['parsimony'] = w['parsimony'] * L.parsimony(self._alpha_full, coarse)
        if 'tv' in w:
            terms['tv'] = w['tv'] * L.total_variation(self._bkg_maps, self._ground_maps, self._blocks_maps, self.tv_norm, coarse)
        if 'overlap' in w:
            S, R, T = self._blocks_SRT
            terms['overlap'] = w['overlap'] * L.overlap(S, R, T, *self._blocks_eps, self._alpha_full, self.ratio_block_scene,
                                                        coarse, generator=self.noise_generator, unit_samples=self.overlap_samples_buffer)
        vals = list(terms.values())
        total = vals[0] if vals else torch.zeros((), device=imgs.device)
        for v in vals[1:]:
            total = total + v
        for k in w:                                   # weights whose term is not produced (perceptual without a network)
            terms.setdefault(k, torch.zeros((), device=imgs.device))
        terms['total'] = total
        return terms

    # ------------------------------------------------------------------ checkpoints / evaluation
    @torch.no_grad()
    def load_state_dict(self, state_dict, **_unused):
        """tolerant loading as dbw.py:440-455: DDP prefixes stripped, `spq_` keys of old checkpoints renamed"""
        own = self.state_dict()
        unknown = []
        for key, value in state_dict.items():
            key = key.replace('module.', '').replace('spq_', 'sq_')
            if key in own:
                own[key].copy_(value.data if isinstance(value, nn.Parameter) else value)
            else:
                unknown.append(key)
        if unknown:
            print(f'load_state_dict: {unknown} not found')

    @torch.no_grad()
    def quantitative_eval(self, loader, device, hard_inference=True):
        """the columns of final_scores.tsv (dbw.py:464-493): n_blocks, L_tot, L_rec, PSNR, SSIM, LPIPS, alpha_k -- hard 4x
        supersampled renders of the opaque blocks over a loader.  LPIPS is NaN when no perceptual network is installed, or
        when the installed term is the VGG feature loss (perceptual.PerceptualLoss), which is not an LPIPS score."""
        from .perceptual import PerceptualLoss
        self.eval()
        opacities = self.get_opacities()
        scene = self.build_scene(filter_transparent=True)
        perceptual = getattr(self, 'perceptual_loss', None)
        if isinstance(perceptual, PerceptualLoss):
            perceptual = None
        sums, count = dict(L_tot=0.0, L_rec=0.0, PSNR=0.0, SSIM=0.0, LPIPS=0.0), 0
        for inp, labels in loader:
            inp = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in inp.items()}
            self._install_cameras(inp)
            imgs, n = inp['imgs'], len(inp['imgs'])
            rec = (self.renderer(scene.extend(n), inp['R'], inp['T'], viz_purpose=True)[:, :3] if hard_inference
                   else self.predict(inp, labels, filter_transparent=True))
            losses = self.compute_losses(imgs, rec)
            sums['L_tot'] += float(losses['total']) * n
            sums['L_rec'] += float(sum(losses[k] for k in ('rgb', 'perceptual') if k in losses)) * n
            sums['PSNR'] += float(-10.0 * torch.log10(F.mse_loss(imgs, rec))) * n
            sums['SSIM'] += float(L.ssim(imgs, rec).mean()) * n
            sums['LPIPS'] += (float(perceptual(imgs, rec)) if perceptual is not None else float('nan')) * n
            count += n
        return OrderedDict([('n_blocks', int((opacities > 0.5).sum()))] + [(k, v / max(count, 1)) for k, v in sums.items()]
                           + [(f'alpha{k}', a.item()) for k, a in enumerate(opacities)])

    @torch.no_grad()
    def qualitative_eval(self, loader, device, path=None, NV=240, n_inputs=10):
        """the still images and meshes of dbw.py:495-554: texture maps, the scene as OBJ (with and without background), and
        per input view the hard reconstruction, its block-coloured edge overlays and the lit synthetic-colour render.
        The reference's mp4 trajectories (NV frames through imageio / ffmpeg) and the ground-truth point-cloud PLY are
        export paths outside the render hot path and are not written."""
        from pathlib import Path
        path = Path(path) if path is not None else Path('.')
        path.mkdir(parents=True, exist_ok=True)
        self.eval()
        (path / 'textures').mkdir(exist_ok=True)
        _save_png(torch.sigmoid(self.texture_bkg).permute(0, 3, 1, 2)[0], path / 'textures' / 'bkg.png')
        _save_png(torch.sigmoid(self.texture_ground).permute(0, 3, 1, 2)[0], path / 'textures' / 'ground.png')
        for k, img in enumerate(torch.sigmoid(self.textures).permute(0, 3, 1, 2)):
            _save_png(img, path / 'textures' / f'block_{str(k).zfill(2)}.png')
        meshes = self.build_scene(filter_transparent=True)
        _save_obj(meshes, path / 'mesh_full.obj')
        _save_obj(self.build_scene(filter_transparent=True, w_bkg=False, reduce_ground=True), path / 'mesh.obj')
        syn_blocks = self.build_blocks(filter_transparent=True, synthetic_colors=True, as_scene=True)
        if len(syn_blocks) == 0:
            return None
        colors = self.get_scene_face_colors(filter_transparent=True, w_env=False)
        count, n_zeros = 0, int(np.log10(max(n_inputs - 1, 1))) + 1
        for inp, labels in loader:
            if count >= n_inputs:
                break
            inp = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in inp.items()}
            self._install_cameras(inp)
            for k in range(min(len(inp['imgs']), n_inputs - count)):
                tag = str(count).zfill(n_zeros)
                img, R, T = inp['imgs'][k:k + 1], inp['R'][k:k + 1], inp['T'][k:k + 1]
                _save_png(img[0], path / f'{tag}_inp.png')
                rec = self.renderer(meshes, R, T, viz_purpose=True)[:, :3]
                _save_png(rec[0], path / f'{tag}_rec.png')
                _save_png(self.renderer.draw_edges(rec, syn_blocks, R, T, colors)[0], path / f'{tag}_rec_col.png')
                _save_png(self.renderer.draw_edges(img, syn_blocks, R, T, colors)[0], path / f'{tag}_rec_col_inp.png')
                syn = self.renderer_light(syn_blocks, R, T, viz_purpose=True)[:, :3]
                _save_png(syn[0], path / f'{tag}_rec_syn_nobkg.png')
                _save_png(self.renderer_light.draw_edges(syn, syn_blocks, R, T, linewidth=0.7, colors=(0.3, 0.3, 0.3))[0],
                          path / f'{tag}_rec_syn_nobkg_edged.png')
                count += 1
        return count


def _save_png(chw, path):
    from PIL import Image
    arr = (chw.detach().float().clamp(0, 1) * 255).permute(1, 2, 0).cpu().numpy().astype(np.uint8)
    Image.fromarray(arr).convert('RGB').save(path)


def _save_obj(meshes, path):
    """geometry-only Wavefront OBJ of the first mesh (the reference's textured export goes through PyTorch3D's save_obj)"""
    verts, faces = meshes.get_mesh_verts_faces(0)
    with open(path, 'w') as fh:
        for v in verts.detach().cpu().tolist():
            fh.write('v {:.6f} {:.6f} {:.6f}\n'.format(*v))
        for f in (faces.detach().cpu() + 1).tolist():
            fh.write('f {} {} {}\n'.format(*f))


class PerceptualTerm(nn.Module):
    """`LPIPSLoss` of the reference (src/model/loss.py:32-40): a FROZEN LPIPS network as a registered submodule (moved by
    .to(), present in the state_dict as `perceptual_loss.*`), called as net(imgs, rec, normalize=True).mean().  The network
    itself is a VGG16 conv stack (cuDNN / tensor cores): outside the render hot path (SURVEY 8a row a13)."""

    def __init__(self, net):
        super().__init__()
        self.loss = net
        for p in self.loss.parameters():
            p.requires_grad_(False)

    def forward(self, imgs, rec):
        return self.loss(imgs, rec, normalize=True).mean()


def _make_perceptual(name):
    """the perceptual term's network, or None (with a LOUD warning: every shipped config weighs it 0.1) when `lpips` and its
    VGG weights are not available -- set_perceptual_loss() installs any callable / module instead.  'perceptual' builds
    perceptual.PerceptualLoss from torchvision's hub cache file (the file the reference's vgg16(weights=IMAGENET1K_V1)
    loads); it never downloads.  It is called as perceptual_loss(imgs, rec), as in the reference, so it is not wrapped."""
    if name == 'perceptual':
        import os
        from .perceptual import PerceptualLoss
        path = os.path.join(torch.hub.get_dir(), 'checkpoints', 'vgg16-397923af.pth')
        if os.path.exists(path):
            return PerceptualLoss.from_files(path)
        import warnings
        warnings.warn(f'[dbw_b200] perceptual_weight > 0 but the VGG16 weights are unavailable ({path} not found; nothing is '
                      f'downloaded): the perceptual term is DROPPED from the objective (reported as 0) until '
                      f'set_perceptual_loss() installs one', RuntimeWarning)
        return None
    if name != 'lpips':
        raise NotImplementedError(name)
    try:
        import lpips
        return PerceptualTerm(lpips.LPIPS(net='vgg', verbose=False))
    except (ImportError, NotImplementedError, OSError) as exc:
        import warnings
        warnings.warn(f'[dbw_b200] perceptual_weight > 0 but the LPIPS network is unavailable ({exc}): the perceptual term is '
                      f'DROPPED from the objective (reported as 0) until set_perceptual_loss() installs one', RuntimeWarning)
        return None


def create_model(cfg, img_size, **kwargs):
    """model factory with the reference's signature (src/model/__init__.py:12-17)"""
    kwargs = deepcopy(cfg['model'])
    name = kwargs.pop('name')
    assert name == 'dbw', name
    return DifferentiableBlocksWorld(img_size, **kwargs)
