"""autograd seams over the fused scene-construction kernels (dbw_scene_geometry_*, dbw_texture_prep_*): the
superquadric mesh build and the texture preparation of src/model/dbw.py:267-352 as ONE kernel each way instead of
~200 eager ops, with no host synchronisation (CUDA-graph friendly)."""
import ctypes

import torch

from . import _lib
from ._lib import DbwSceneGeometry, DbwTexJob
from .renderer import _c, _stream


def _geom_struct(static, sq_eps, S, R6, T, R6g, Tg):
    g = DbwSceneGeometry()
    g.n_blocks, g.verts_per_block, g.n_ground_verts = static['n_blocks'], static['verts_per_block'], static['n_ground_verts']
    g.sq_eta, g.sq_omega = static['sq_eta'].data_ptr(), static['sq_omega'].data_ptr()
    g.sq_eps, g.S, g.R_6d, g.T = sq_eps.data_ptr(), S.data_ptr(), R6.data_ptr(), T.data_ptr()
    g.ground_verts = static['ground_verts'].data_ptr()
    g.R_6d_ground, g.T_ground = R6g.data_ptr(), Tg.data_ptr()
    g.ratio_block_scene, g.scale_min, g.S_world = static['ratio'], static['scale_min'], static['S_world']
    g.R_world = (ctypes.c_float * 9)(*static['R_world'])
    g.T_world = (ctypes.c_float * 3)(*static['T_world'])
    return g


class _SceneGeometryEnvFn(torch.autograd.Function):
    """dbw_scene_geometry_forward / _backward: both passes' vertex arrays out of one launch and one buffer
    (static environment vertices | ground | blocks), their gradients taken where autograd hands them over -- no
    concatenation either way, no zero-fill (the backward kernel writes every leaf gradient)."""

    @staticmethod
    def forward(ctx, sq_eps, S, R6, T, R6g, Tg, static, env_static):
        args = [t.detach().contiguous().float() for t in (sq_eps, S, R6, T, R6g, Tg)]
        g = _geom_struct(static, *args)
        n_static, n_ground = env_static.shape[0], static['n_ground_verts']
        nb = static['n_blocks'] * static['verts_per_block']
        out = torch.empty(n_static + n_ground + nb, 3, device=sq_eps.device, dtype=torch.float32)
        _lib.check(_lib.lib().dbw_scene_geometry_forward(ctypes.byref(g), _c(env_static), n_static, _c(out), _stream()),
                   'dbw_scene_geometry_forward')
        ctx.save_for_backward(*args)
        ctx.static, ctx.n_static = static, n_static
        return out[n_static + n_ground:], out[:n_static + n_ground]

    @staticmethod
    def backward(ctx, g_blocks, g_env):
        args = ctx.saved_tensors
        g = _geom_struct(ctx.static, *args)
        g_blocks = g_blocks.reshape(-1, 3).contiguous().float()
        g_ground = g_env.reshape(-1, 3)[ctx.n_static:].contiguous().float()
        fill = torch.empty if ctx.static['n_ground_verts'] > 0 else torch.zeros      # without a ground its two gradients stay unwritten
        flat = fill(sum(t.numel() for t in args), device=g_blocks.device, dtype=torch.float32)
        grads, o = [], 0
        for t in args:
            grads.append(flat[o:o + t.numel()].view_as(t))
            o += t.numel()
        _lib.check(_lib.lib().dbw_scene_geometry_backward(ctypes.byref(g), _c(g_blocks), _c(g_ground), *[_c(t) for t in grads],
                                                          _stream()), 'dbw_scene_geometry_backward')
        return (*grads, None, None)


def scene_geometry_passes(sq_eps, S, R_6d, T, R_6d_ground, T_ground, static, env_static_verts):
    """(block vertices (N*Vb, 3), environment vertices (n_static + Vg, 3) = `env_static_verts` then the posed ground) in world
    space: the vertex arrays of the blocks pass and of the environment pass, from one kernel launch."""
    return _SceneGeometryEnvFn.apply(sq_eps, S, R_6d, T, R_6d_ground, T_ground, static, env_static_verts.contiguous().float())


class _OpacityFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logit, noise, noise_scale, keep_threshold, face_map, faces_per_block):
        lg = logit.detach().contiguous().float()
        nz = noise.detach().contiguous().float() if noise is not None else None
        N = lg.numel()
        out = torch.empty(2, N, device=lg.device, dtype=torch.float32)
        filtered = keep_threshold >= 0
        fmap = torch.empty_like(face_map) if filtered else face_map
        _lib.check(_lib.lib().dbw_opacity_forward(_c(lg), _c(nz), float(noise_scale), float(keep_threshold), _c(face_map), N,
                                                  int(faces_per_block), _c(out[0]), _c(out[1]), _c(fmap) if filtered else None,
                                                  _stream()), 'dbw_opacity_forward')
        ctx.save_for_backward(lg, nz)
        ctx.cfg = (float(noise_scale), float(keep_threshold))
        ctx.mark_non_differentiable(fmap)
        ctx.set_materialize_grads(False)
        return out[0], out[1], fmap

    @staticmethod
    def backward(ctx, g_alpha, g_kept, _g_fmap):
        lg, nz = ctx.saved_tensors
        if g_alpha is None and g_kept is None:
            return None, None, None, None, None, None
        ga = g_alpha.contiguous().float() if g_alpha is not None else None
        gk = g_kept.contiguous().float() if g_kept is not None else None
        g = torch.empty_like(lg)
        _lib.check(_lib.lib().dbw_opacity_backward(_c(lg), _c(nz), ctx.cfg[0], ctx.cfg[1], _c(ga), _c(gk), lg.numel(), _c(g), _stream()),
                   'dbw_opacity_backward')
        return g, None, None, None, None, None


def block_opacities(alpha_logit, noise, noise_scale, keep_threshold, face_map, faces_per_block):
    """(alpha (N,), alpha_kept (N,), face_map (N*faces_per_block,) int32) in one launch -- src/model/dbw.py:300-316 with static
    shapes: alpha = sigmoid(logit + noise_scale * noise); with keep_threshold >= 0 the blocks whose noise-free opacity is not
    above it are zeroed in alpha_kept and disabled (-1) in the returned face map (keep_threshold < 0: nothing is filtered and
    `face_map` is returned as it is)."""
    return _OpacityFn.apply(alpha_logit, noise, noise_scale, keep_threshold, face_map, faces_per_block)


class _SceneAtlasesFn(torch.autograd.Function):
    """the three texture stacks of a step -- background, ground, blocks (src/model/dbw.py:276-279,291-294,307,331-341) -- to
    the two float4 atlases the passes sample, in ONE launch each way: (env atlas = background then ground, blocks atlas)"""

    @staticmethod
    def forward(ctx, tex_bkg, tex_ground, tex_blocks, pad, decim_env, decim_blocks):
        tb, tg, tk = (t.detach().contiguous().float() for t in (tex_bkg, tex_ground, tex_blocks))
        se, N, TS = tb.shape[1], tk.shape[0], tk.shape[1]
        assert tb.shape == tg.shape and tb.shape[0] == 1
        env = torch.empty(2, se, se, 4, device=tb.device, dtype=torch.float32)
        blk = torch.empty(N, TS, TS + pad[0] + pad[1], 4, device=tb.device, dtype=torch.float32)
        jobs = (DbwTexJob * 3)(DbwTexJob(tb.data_ptr(), env[0].data_ptr(), None, 1, se, 0, 0, decim_env, 0),
                               DbwTexJob(tg.data_ptr(), env[1].data_ptr(), None, 1, se, 0, 0, decim_env, 0),
                               DbwTexJob(tk.data_ptr(), blk.data_ptr(), None, N, TS, pad[0], pad[1], decim_blocks, 0))
        _lib.check(_lib.lib().dbw_texture_prep_forward_multi(jobs, 3, _stream()), 'dbw_texture_prep_forward_multi')
        ctx.save_for_backward(tb, tg, tk)
        ctx.cfg = (pad, decim_env, decim_blocks)
        return env, blk

    @staticmethod
    def backward(ctx, g_env, g_blk):
        tb, tg, tk = ctx.saved_tensors
        pad, decim_env, decim_blocks = ctx.cfg
        se, N, TS = tb.shape[1], tk.shape[0], tk.shape[1]
        g_env, g_blk = g_env.contiguous().float(), g_blk.contiguous().float()
        flat = torch.empty(tb.numel() + tg.numel() + tk.numel(), device=tb.device, dtype=torch.float32)
        gb, gg, gk = flat[:tb.numel()].view_as(tb), flat[tb.numel():tb.numel() + tg.numel()].view_as(tg), flat[tb.numel() + tg.numel():].view_as(tk)
        jobs = (DbwTexJob * 3)(DbwTexJob(tb.data_ptr(), g_env[0].data_ptr(), gb.data_ptr(), 1, se, 0, 0, decim_env, 0),
                               DbwTexJob(tg.data_ptr(), g_env[1].data_ptr(), gg.data_ptr(), 1, se, 0, 0, decim_env, 0),
                               DbwTexJob(tk.data_ptr(), g_blk.data_ptr(), gk.data_ptr(), N, TS, pad[0], pad[1], decim_blocks, 0))
        _lib.check(_lib.lib().dbw_texture_prep_backward_multi(jobs, 3, _stream()), 'dbw_texture_prep_backward_multi')
        return gb, gg, gk, None, None, None


STAGE_FUSED, STAGE_CELLS, STAGE_EXPAND, STAGE_CELLS4 = 0, 1, 2, 3          # DBW_TEX_STAGE_* of include/dbw_render.h


def _tex_launch(jobs, backward):
    fn = _lib.lib().dbw_texture_prep_backward_multi if backward else _lib.lib().dbw_texture_prep_forward_multi
    _lib.check(fn((DbwTexJob * len(jobs))(*jobs), len(jobs), _stream()), 'dbw_texture_prep_*_multi')


class _SceneCellsFn(torch.autograd.Function):
    """first half of the texture preparation (DBW_TEX_STAGE_CELLS): the three texture stacks -> their CELL colours
    box_mean(sigmoid(logits)): (2, se/f_env, se/f_env, C) for background + ground, (N, TS/f_blk, TS/f_blk, C) for the blocks;
    C = 3, or 4 (RGB + 0, DBW_TEX_STAGE_CELLS4: the float4 cells the raster passes sample as cell maps)"""

    @staticmethod
    def forward(ctx, tex_bkg, tex_ground, tex_blocks, decim_env, decim_blocks, texels4):
        tb, tg, tk = (t.detach().contiguous().float() for t in (tex_bkg, tex_ground, tex_blocks))
        se, N, TS = tb.shape[1], tk.shape[0], tk.shape[1]
        assert tb.shape == tg.shape and tb.shape[0] == 1
        ce, ck, C = se // decim_env, TS // decim_blocks, 4 if texels4 else 3
        stage = STAGE_CELLS4 if texels4 else STAGE_CELLS
        env = torch.empty(2, ce, ce, C, device=tb.device, dtype=torch.float32)
        blk = torch.empty(N, ck, ck, C, device=tb.device, dtype=torch.float32)
        _tex_launch([DbwTexJob(tb.data_ptr(), env[0].data_ptr(), None, 1, se, 0, 0, decim_env, stage),
                     DbwTexJob(tg.data_ptr(), env[1].data_ptr(), None, 1, se, 0, 0, decim_env, stage),
                     DbwTexJob(tk.data_ptr(), blk.data_ptr(), None, N, TS, 0, 0, decim_blocks, stage)], False)
        ctx.save_for_backward(tb, tg, tk)
        ctx.cfg = (decim_env, decim_blocks, stage)
        return env, blk

    @staticmethod
    def backward(ctx, g_env, g_blk):
        tb, tg, tk = ctx.saved_tensors
        decim_env, decim_blocks, stage = ctx.cfg
        se, N, TS = tb.shape[1], tk.shape[0], tk.shape[1]
        g_env, g_blk = g_env.contiguous().float(), g_blk.contiguous().float()
        flat = torch.empty(tb.numel() + tg.numel() + tk.numel(), device=tb.device, dtype=torch.float32)
        gb, gg, gk = flat[:tb.numel()].view_as(tb), flat[tb.numel():tb.numel() + tg.numel()].view_as(tg), flat[tb.numel() + tg.numel():].view_as(tk)
        _tex_launch([DbwTexJob(tb.data_ptr(), g_env[0].data_ptr(), gb.data_ptr(), 1, se, 0, 0, decim_env, stage),
                     DbwTexJob(tg.data_ptr(), g_env[1].data_ptr(), gg.data_ptr(), 1, se, 0, 0, decim_env, stage),
                     DbwTexJob(tk.data_ptr(), g_blk.data_ptr(), gk.data_ptr(), N, TS, 0, 0, decim_blocks, stage)], True)
        return gb, gg, gk, None, None, None


class _AtlasesFromCellsFn(torch.autograd.Function):
    """second half (DBW_TEX_STAGE_EXPAND): cell colours -> the two float4 atlases the passes sample (nearest upsampling by the
    decimation factor, circular u padding of the blocks' maps); backward: atlas gradients -> cell gradients (sums)"""

    @staticmethod
    def forward(ctx, cells_env, cells_blk, pad, decim_env, decim_blocks):
        ce, ck = cells_env.detach().contiguous().float(), cells_blk.detach().contiguous().float()
        se, N, TS = ce.shape[1] * decim_env, ck.shape[0], ck.shape[1] * decim_blocks
        env = torch.empty(2, se, se, 4, device=ce.device, dtype=torch.float32)
        blk = torch.empty(N, TS, TS + pad[0] + pad[1], 4, device=ce.device, dtype=torch.float32)
        _tex_launch([DbwTexJob(ce.data_ptr(), env.data_ptr(), None, 2, se, 0, 0, decim_env, STAGE_EXPAND),
                     DbwTexJob(ck.data_ptr(), blk.data_ptr(), None, N, TS, pad[0], pad[1], decim_blocks, STAGE_EXPAND)], False)
        ctx.shapes = (ce.shape, ck.shape, se, N, TS, pad, decim_env, decim_blocks)
        return env, blk

    @staticmethod
    def backward(ctx, g_env, g_blk):
        ce_shape, ck_shape, se, N, TS, pad, decim_env, decim_blocks = ctx.shapes
        g_env, g_blk = g_env.contiguous().float(), g_blk.contiguous().float()
        n_e = ce_shape.numel()
        flat = torch.empty(n_e + ck_shape.numel(), device=g_env.device, dtype=torch.float32)
        ge, gk = flat[:n_e].view(ce_shape), flat[n_e:].view(ck_shape)
        # `textures` is not read by this stage's backward: any valid device pointer
        _tex_launch([DbwTexJob(g_env.data_ptr(), g_env.data_ptr(), ge.data_ptr(), 2, se, 0, 0, decim_env, STAGE_EXPAND),
                     DbwTexJob(g_blk.data_ptr(), g_blk.data_ptr(), gk.data_ptr(), N, TS, pad[0], pad[1], decim_blocks, STAGE_EXPAND)], True)
        return ge, gk, None, None, None


def scene_texture_cells(texture_bkg, texture_ground, textures, decim_env=1, decim_blocks=1, texels4=False):
    """(environment cells (2, se/f, se/f, 3), block cells (N, TS/f, TS/f, 3)): sigmoid + box mean of the three texture stacks, one
    launch.  With atlases_from_cells() it equals scene_atlases() bit for bit; the cells are where a data-parallel step sums its
    texture gradients (64x fewer values than the parameters while textures are decimated).  texels4: float4 cells (last dim 4,
    RGB + 0), which the raster passes sample directly through cell_map_table() -- no atlas in between."""
    return _SceneCellsFn.apply(texture_bkg, texture_ground, textures, int(decim_env), int(decim_blocks), bool(texels4))


def cell_map_table(n_maps, txt_size, decimate, p_left=0, p_right=0):
    """map table [(offset, H, W, reserved)] of `n_maps` float4 cell maps stored back to back (scene_texture_cells(...,
    texels4=True)): each samples as the (txt_size, p_left + txt_size + p_right) atlas that atlases_from_cells() would expand it
    to (DbwMapDesc / DBW_MAP_CELLS in include/dbw_render.h)"""
    cs = txt_size // decimate
    return [(i * cs * cs * 3, txt_size, txt_size + p_left + p_right, (p_left << 8) | decimate) for i in range(n_maps)]


def atlases_from_cells(cells_env, cells_blk, pad, decim_env=1, decim_blocks=1):
    """the two float4 atlases of scene_atlases() from the cell colours of scene_texture_cells(), one launch"""
    return _AtlasesFromCellsFn.apply(cells_env, cells_blk, (int(pad[0]), int(pad[1])), int(decim_env), int(decim_blocks))


def scene_atlases(texture_bkg, texture_ground, textures, pad, decim_env=1, decim_blocks=1):
    """(env atlas (2, S, S, 4): background then ground; blocks atlas (N, TS, p_left + TS + p_right, 4)) from the three texture
    parameters in one launch (and one for all three gradients): sigmoid, optional 8x8 box decimation, circular padding along
    u, as float4 texels -- the layout the rasterizer samples directly (render_scene(..., maps_are_texels4=True))"""
    return _SceneAtlasesFn.apply(texture_bkg, texture_ground, textures, (int(pad[0]), int(pad[1])), int(decim_env), int(decim_blocks))
