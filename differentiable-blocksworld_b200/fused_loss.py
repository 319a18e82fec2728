"""Decoupled render + compositing + RGB loss as ONE autograd node (SURVEY 8f rank 3, "MSE fused into blend"):

    env  = render(environment)                      src/model/dbw.py:219      (renderer_env, K=1)
    fg   = render(blocks)                           src/model/dbw.py:220-221  (renderer / renderer_fine, K=10)
    rec  = fg_rgb * fg_a + (1 - fg_a) * env_rgb     src/model/dbw.py:223
    loss = mean((imgs - rec)^2)                     src/model/dbw.py:366-367  (nn.MSELoss)

The blocks pass runs with the loss epilogue of include/dbw_render.h (dbw_render_forward_loss): compositing, squared error
and the MSE gradients w.r.t. both layers happen per pixel inside the rasterizer while the blended colour is in registers.
Neither `fg` nor `rec` nor the two image-sized gradient round trips of a separate composite kernel ever touch HBM; the
backward is the two raster backward kernels reading those gradients, scaled on the fly by the upstream gradient of the loss
(dbw_render_backward's grad_scale).  When the blocks pass is detach_bary over cell maps (the coarse phase) and a gradient is wanted,
it goes further: the blocks forward kernel also runs the pass's backward while the per-pixel fragment lists are still on chip
(dbw_render_forward_loss_grad), so neither its fragment records nor d loss / d blocks RGBA are written, and the backward only
folds the accumulated gradients, times the upstream gradient (dbw_render_backward_deferred).  Not usable when another loss consumes `rec` with gradient (LPIPS): the model then keeps
the separate composite kernel (dbw._CompositeMSE), which accepts a gradient on `rec`."""
import ctypes

import torch

from . import _lib
from ._lib import DbwLossEpilogue
from .renderer import _c, _stream, scene_settings, project_verts, view_intrinsics, cameras_need_grad

N_PARTIALS = 1024
GRAD_VERTS, GRAD_MAPS, GRAD_ALPHA = 1, 2, 4          # grad_mask bits of dbw_render_forward_loss_grad (DBW_GRAD_*)
# run the two passes' backward kernels concurrently (the environment's on a side stream: parallel branches of the step's CUDA
# graph).  One GPU, 49 views: no gain (the kernels fill the machine by themselves); 8 GPUs, ~6 views each: the launches are
# short and one kernel's ramp-up hides the other's tail -- bench.py --overlap-bwd measures it
OVERLAP_BACKWARD_PASSES = False
# differentiate the blocks pass inside its loss-epilogue forward kernel where it can (see above); False: the two-kernel path
FUSE_BLOCKS_BACKWARD = True
_side_stream = None


class ScenePass:
    """static description of one render pass: topology, UVs, map layout and the renderer's shading options"""

    def __init__(self, faces, faces_uvs, face_map, map_table_host, renderer, alpha_group=1, n_static_faces=0):
        self.faces = faces.to(torch.int32).contiguous()
        self.faces_uvs = faces_uvs.contiguous().float()
        self.face_map = face_map.to(torch.int32).contiguous()
        self.map_table_host, self.r = map_table_host, renderer
        self.alpha_group, self.n_static_faces = alpha_group, n_static_faces

    def settings(self, verts, maps, B, faces_alpha, view_rows=None, ndc=False, static_faces=True):
        """ndc: `verts` are per-view projected (B,V,3) NDC vertices (per-view intrinsics); static_faces=False: differentiate the
        static faces too (a render whose cameras take a gradient)"""
        r = self.r
        intr = (1., 1., 0., 0.) if ndc else r.cameras.intrinsics()
        return scene_settings(verts, self.faces, maps, self.map_table_host, B, intr, r.img_size, r.sigma,
                              r.faces_per_pixel, r.z_clip, r.detach_bary, r.clip_inside, r.background_color, faces_alpha,
                              r.perspective_correct, ndc, r.blur_radius, True, self.alpha_group,
                              self.n_static_faces if static_faces else 0, view_rows)


def _workspace(cfg, dev):
    fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(_lib.lib().dbw_workspace_bytes(ctypes.byref(cfg), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
    return torch.empty(fwd.value, dtype=torch.uint8, device=dev), bwd.value


class _SceneMSEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, env_verts, env_maps, blk_verts, blk_maps, blk_alpha, R, T, imgs, env_pass, blk_pass, blk_face_map,
                cfgs, inv_count, want_rec):
        L = _lib.lib()
        dev = blk_verts.device
        B, _, H, W = imgs.shape
        f32 = lambda t: t.detach().contiguous().float() if t is not None else None      # R, T: None when verts are NDC
        env_verts, env_maps, blk_verts, blk_maps = f32(env_verts), f32(env_maps), f32(blk_verts), f32(blk_maps)
        R, T, imgs = f32(R), f32(T), f32(imgs)
        fa = f32(blk_alpha) if blk_alpha is not None else None
        fmap_b = blk_face_map.to(torch.int32).contiguous()
        (cfg_e, table_e), (cfg_b, table_b) = cfgs
        need = ctx.needs_input_grad
        # grad mode is off in here: the settings, made outside, say whether a backward may follow (save_fragment_state)
        fused = (FUSE_BLOCKS_BACKWARD and bool(cfg_b.save_fragment_state) and bool(cfg_b.detach_bary)
                 and cfg_b.maps_are_texels4 == 2 and any(need[2:7]))
        if fused:
            cfg_b = _lib.DbwRenderSettings.from_buffer_copy(cfg_b)
            cfg_b.save_fragment_state = 0                                     # the fused kernel writes no fragment records
        ws_e, bwd_e = _workspace(cfg_e, dev)
        ws_b, bwd_b = _workspace(cfg_b, dev)
        env_rgba = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)
        _lib.check(L.dbw_render_forward(ctypes.byref(cfg_e), _c(env_verts), _c(env_pass.faces), _c(env_pass.faces_uvs),
                                        _c(env_pass.face_map), _c(env_maps), _c(table_e), _c(R), _c(T), None, _c(env_rgba),
                                        None, _c(ws_e), ws_e.numel(), None, None, _stream()), 'dbw_render_forward')
        g_env = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)      # d loss / d env RGBA (unscaled)
        partials = torch.empty(N_PARTIALS, dtype=torch.float32, device=dev)
        rec = torch.empty(B, 3, H, W, dtype=torch.float32, device=dev) if want_rec else None
        ep = DbwLossEpilogue()
        ep.env_rgba, ep.target, ep.g_env = env_rgba.data_ptr(), imgs.data_ptr(), g_env.data_ptr()
        ep.rec = rec.data_ptr() if rec is not None else None
        ep.loss_partials, ep.n_partials, ep.inv_count = partials.data_ptr(), N_PARTIALS, float(inv_count)
        # the environment renders without opacities; when it is also hard, its backward has neither an opacity nor a distance
        # path and never reads the alpha plane of g_env (its only reader), so the epilogue does not write it
        ep.env_alpha_unread = int(cfg_e.sigma == 0.0)
        g_fg = scratch_b = None
        if fused:
            mask = ((GRAD_VERTS if need[2] or need[5] or need[6] else 0) | (GRAD_MAPS if need[3] else 0)
                    | (GRAD_ALPHA if need[4] and fa is not None else 0))
            scratch_b = torch.empty(bwd_b, dtype=torch.uint8, device=dev)    # unscaled gradients, folded by the backward
            _lib.check(L.dbw_render_forward_loss_grad(ctypes.byref(cfg_b), _c(blk_verts), _c(blk_pass.faces), _c(blk_pass.faces_uvs),
                                                      _c(fmap_b), _c(blk_maps), _c(table_b), _c(R), _c(T), _c(fa), _c(ws_b),
                                                      ws_b.numel(), ctypes.byref(ep), mask, _c(scratch_b), scratch_b.numel(),
                                                      _stream()), 'dbw_render_forward_loss_grad')
        else:
            g_fg = torch.empty(B, 4, H, W, dtype=torch.float32, device=dev)   # d loss / d blocks RGBA (unscaled)
            _lib.check(L.dbw_render_forward_loss(ctypes.byref(cfg_b), _c(blk_verts), _c(blk_pass.faces), _c(blk_pass.faces_uvs),
                                                 _c(fmap_b), _c(blk_maps), _c(table_b), _c(R), _c(T), _c(fa), _c(g_fg), None,
                                                 _c(ws_b), ws_b.numel(), ctypes.byref(ep), _stream()), 'dbw_render_forward_loss')
        loss = partials.sum()
        ctx.save_for_backward(env_verts, env_maps, blk_verts, blk_maps, fa, R, T, fmap_b, table_e, table_b, ws_e, ws_b, g_fg, g_env,
                              scratch_b)
        ctx.meta = (env_pass, blk_pass, cfg_e, cfg_b, bwd_e, bwd_b)
        if want_rec:
            ctx.mark_non_differentiable(rec)
            return loss, rec
        return loss

    @staticmethod
    def backward(ctx, g_loss, _g_rec=None):
        env_verts, env_maps, blk_verts, blk_maps, fa, R, T, fmap_b, table_e, table_b, ws_e, ws_b, g_fg, g_env, scratch_b = ctx.saved_tensors
        env_pass, blk_pass, cfg_e, cfg_b, bwd_e, bwd_b = ctx.meta
        L = _lib.lib()
        dev = blk_verts.device
        gl = g_loss.detach().contiguous().float()
        need = ctx.needs_input_grad

        # every gradient buffer of both passes (and the kernels' scratch, which they expect zeroed... they zero it themselves)
        # comes out of ONE zero-filled arena: one fill launch per step instead of five
        wants = [('gm_b', blk_maps, need[3]), ('gm_e', env_maps, need[1]), ('gv_b', blk_verts, need[2]), ('gv_e', env_verts, need[0]),
                 ('ga_b', fa, need[4] and fa is not None), ('g_R', R, need[5]), ('g_T', T, need[6])]
        total = sum((t.numel() + 3) // 4 * 4 for _, t, on in wants if on)
        arena = torch.zeros(total, device=dev, dtype=torch.float32)
        g, off = {}, 0
        for name, t, on in wants:
            g[name] = None
            if on:
                g[name] = arena[off:off + t.numel()].view_as(t)
                off += (t.numel() + 3) // 4 * 4                      # float4 texel atlases stay 16-byte aligned

        g_R, g_T = g['g_R'], g['g_T']          # both passes accumulate into them (include/dbw_render.h)

        def run(cfg, p, fmap, verts, maps, table, alpha, ws, grad, bwd_bytes, g_verts, g_maps, g_alpha):
            if g_verts is None and g_maps is None and g_alpha is None and g_R is None and g_T is None:
                return
            scratch = torch.empty(bwd_bytes, dtype=torch.uint8, device=dev)
            _lib.check(L.dbw_render_backward(ctypes.byref(cfg), _c(verts), _c(p.faces), _c(p.faces_uvs), _c(fmap), _c(maps), _c(table),
                                             _c(R), _c(T), _c(alpha), _c(ws), ws.numel(), _c(grad), _c(gl), _c(g_verts), _c(g_alpha),
                                             _c(g_maps), _c(g_R), _c(g_T), _c(scratch), scratch.numel(), _stream()),
                       'dbw_render_backward')

        def run_blocks():
            if scratch_b is None:
                run(cfg_b, blk_pass, fmap_b, blk_verts, blk_maps, table_b, fa, ws_b, g_fg, bwd_b, g['gv_b'], g['gm_b'], g['ga_b'])
                return
            # the blocks pass was differentiated by its forward kernel: fold its scratch into the gradients, times g_loss
            _lib.check(L.dbw_render_backward_deferred(ctypes.byref(cfg_b), _c(blk_verts), _c(blk_pass.faces), _c(R), _c(T), _c(ws_b),
                                                      ws_b.numel(), _c(gl), _c(g['gv_b']), _c(g['ga_b']), _c(g['gm_b']), _c(g_R),
                                                      _c(g_T), _c(scratch_b), scratch_b.numel(), _stream()),
                       'dbw_render_backward_deferred')

        if OVERLAP_BACKWARD_PASSES:
            global _side_stream
            cur = torch.cuda.current_stream()
            if _side_stream is None or _side_stream.device != dev:
                _side_stream = torch.cuda.Stream(device=dev)
            _side_stream.wait_stream(cur)
            with torch.cuda.stream(_side_stream):
                run(cfg_e, env_pass, env_pass.face_map, env_verts, env_maps, table_e, None, ws_e, g_env, bwd_e, g['gv_e'], g['gm_e'], None)
            run_blocks()
            cur.wait_stream(_side_stream)
        else:
            run_blocks()
            run(cfg_e, env_pass, env_pass.face_map, env_verts, env_maps, table_e, None, ws_e, g_env, bwd_e, g['gv_e'], g['gm_e'], None)
        gv_e, gm_e, gv_b, gm_b, ga_b = g['gv_e'], g['gm_e'], g['gv_b'], g['gm_b'], g['ga_b']
        return gv_e, gm_e, gv_b, gm_b, ga_b, g_R, g_T, None, None, None, None, None, None, None


def scene_mse(env_verts, env_atlas, blk_verts, blk_atlas, blk_alpha, R, T, imgs, env_pass, blk_pass, blk_face_map,
              n_total_views=None, return_rec=False, view_rows=None, K=None):
    """MSE between `imgs` (B,3,H,W) and the blocks composited over the environment, both rendered from raw scene tensors
    (float4 texel atlases from scene_ops.scene_atlases).  `n_total_views`: size of the GLOBAL batch the mean runs over
    (view-sharded data parallelism); `view_rows` (B,2) int32: the [row_begin, row_end) of each view this rank owns.
    K (B,4,4): per-view intrinsics -- both passes' vertices are projected per view (renderer.project_verts) and rendered as NDC
    input, and R, T and K receive gradients through the projection.  Returns the loss, or (loss, rec) with a non-differentiable `rec`."""
    B, _, H, W = imgs.shape
    inv = 1.0 / (float(n_total_views or B) * 3 * H * W)
    if K is not None:
        static = not cameras_need_grad(R, T, K)
        intr = view_intrinsics(K, B)                          # read out of K once for both passes
        env_verts, blk_verts = project_verts(env_verts, R, T, intr=intr), project_verts(blk_verts, R, T, intr=intr)
        cfgs = (env_pass.settings(env_verts, env_atlas, B, None, view_rows, ndc=True, static_faces=static),
                blk_pass.settings(blk_verts, blk_atlas, B, blk_alpha, view_rows, ndc=True, static_faces=static))
        return _SceneMSEFn.apply(env_verts, env_atlas, blk_verts, blk_atlas, blk_alpha, None, None, imgs, env_pass, blk_pass,
                                 blk_face_map, cfgs, inv, bool(return_rec))
    # settings are made out here: inside Function.forward grad mode is off and the passes would not save fragment state
    cfgs = (env_pass.settings(env_verts, env_atlas, B, None, view_rows), blk_pass.settings(blk_verts, blk_atlas, B, blk_alpha, view_rows))
    return _SceneMSEFn.apply(env_verts, env_atlas, blk_verts, blk_atlas, blk_alpha, R, T, imgs, env_pass, blk_pass,
                             blk_face_map, cfgs, inv, bool(return_rec))
