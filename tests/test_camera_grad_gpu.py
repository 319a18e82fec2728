"""GPU: gradients of the camera poses R and T (dbw_render_backward's g_R / g_T, include/dbw_render.h).

Parity with the float64 oracle, whose d/dR and d/dT are torch autograd through oracle.pt3d.world_to_ndc and the rasterizer
(itself checked against central differences in tests/test_camera_grad_host.py).  Tolerances are those of
tests/test_raster_matrix_gpu.py: pixels whose kept faces differ between fp32 and fp64 are excluded on both sides; the pose
gradients must then agree to 1e-3 relative L2 plus an element-wise bound of 2e-3 of the largest magnitude.  Then the C-ABI
contract (a camera gradient adds one launch; the other gradients do not move; row bands sum), the model's
paths, the refusals, the launch count, and a pose recovery."""
import ctypes

import pytest
import torch

from oracle import dbw_path as D
from tests.helpers import decision_mask, intrinsics
from tests.test_model_gpu import _inputs as _model_inputs, _model_and_oracle
from tests.test_raster_matrix_gpu import (BANDS, _alpha, _away_views, _blocks, _cams, _close_to_cuda, _close_to_oracle,
                                          _dev_alpha, _dev_scene, _leaf, _oracle, _rel, _render)

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _env_scene(seed=9):
    """the environment pass of the model: background sphere (static faces) + ground, seen from inside the sphere with a
    wide lens; faces of the sphere straddle the camera plane and are z-clipped"""
    tpl = D.SceneTemplate(n_blocks=2, txt_size=16)
    p = D.init_params(2, 16, seed=seed, dtype=torch.float64)
    R, T, K = _cams(2, seed=seed)
    K = K.clone(); K[0, 0] = K[1, 1] = 1.2
    return tpl, _leaf(tpl.build_env(p)), R, T, K


def _camera_parity(tag, scene, R, T, K, size, sigma, Kf, d, fa_ref=None, fa_dev=None, group=1, n_static_faces=0, seed=0,
                   max_ambiguous=2e-3, conditioning=False, zero_views=(), **opts):
    """CUDA d/dR, d/dT of a weighted sum of the image against the float64 oracle's.  conditioning: the bound is at least 3x the
    error of the oracle's own float32 evaluation against its float64 one (the z-clipped environment: vertices just behind
    the camera have huge NDC coordinates, test_raster_matrix_gpu.test_z_clipped_scene_with_and_without_perspective_correction)"""
    dev = _dev()
    Rl, Tl = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    ref, frags = _oracle(scene, Rl, Tl, K, size, sigma, Kf, fa=fa_ref, **opts)
    Rd = R.detach().float().to(dev).requires_grad_(True)
    Td = T.detach().float().to(dev).requires_grad_(True)
    out, ids = _render(d, Rd, Td, K, size, sigma, Kf, fa=fa_dev, alpha_group=group, n_static_faces=n_static_faces, **opts)
    B, _, H, W = ref.shape
    mask = decision_mask(ids, frags, scene['faces'].shape[0])
    amb = 1 - mask.mean().item()
    print(f'\n{tag}: ambiguous pixels {amb * 100:.3f}%')
    assert amb <= max(max_ambiguous, 1.5 / (B * H * W))
    wgt = torch.rand(B, 4, H, W, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * mask
    ref_R, ref_T = torch.autograd.grad((ref * wgt).sum(), [Rl, Tl], retain_graph=conditioning)
    g_R, g_T = torch.autograd.grad(out, [Rd, Td], grad_outputs=wgt.to(dev).float())
    rel, elem = 1e-3, 2e-3
    if conditioning:
        s32 = dict(scene, verts=scene['verts'].detach().float(), maps=[m.detach().float() for m in scene['maps']],
                   faces_verts_uvs=scene['faces_verts_uvs'].float())
        R32, T32 = R.float().requires_grad_(True), T.float().requires_grad_(True)
        ref32, frags32 = _oracle(s32, R32, T32, K.float(), size, sigma, Kf, fa=fa_ref, **opts)
        m = (frags32.clipped_idx == frags.clipped_idx).all(-1)[:, None].double() * mask
        r64 = torch.autograd.grad((ref * wgt * m).sum(), [Rl, Tl])
        r32 = torch.autograd.grad((ref32 * (wgt * m).float()).sum(), [R32, T32])
        for a, b in zip(r32, r64):
            rel = max(rel, 3 * _rel(a.double(), b))
            elem = max(elem, 3 * (a.double() - b).abs().max().item() / b.abs().max().item())
        print(f'{tag}: float32 oracle rel err R {_rel(r32[0].double(), r64[0]):.3e} T {_rel(r32[1].double(), r64[1]):.3e}')
    print(f'{tag}: g_R rel err {_rel(g_R.cpu().double(), ref_R):.3e}, g_T rel err {_rel(g_T.cpu().double(), ref_T):.3e} (bound {rel:.1e})')
    assert ref_R.abs().max() > 0 and ref_T.abs().max() > 0
    _close_to_oracle(g_R, ref_R, f'{tag} g_R', rel, elem)
    _close_to_oracle(g_T, ref_T, f'{tag} g_T', rel, elem)
    for v in zero_views:
        assert torch.isfinite(g_R[v]).all() and g_R[v].abs().max() == 0 and g_T[v].abs().max() == 0, v
    return g_R, g_T


# ------------------------------------------------------------------------------------------------ parity: blocks
# (tag, faces per pixel, sigma, detach_bary, clip_inside, opacity layout, image size)
BLOCK_CASES = [
    ('coarse', 10, 1e-4, False, True, 'block', (48, 64)),
    ('fine', 10, 5e-6, False, True, 'block', (48, 64)),
    ('sigmoid', 10, 1e-4, False, False, 'face', (48, 64)),
    ('detach_bary', 10, 1e-4, True, True, 'batch', (48, 64)),
    ('k1', 1, 1e-4, False, True, 'face', (40, 56)),
    ('k25', 25, 1e-4, False, True, 'batch_face', (40, 56)),
    ('tall', 10, 1e-4, True, True, None, (72, 40)),
]


@pytest.mark.parametrize('tag,Kf,sigma,detach,clip_inside,alpha,size', BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_blocks_camera_gradients_match_oracle(tag, Kf, sigma, detach, clip_inside, alpha, size):
    dev = _dev()
    tpl, _, scene = _blocks(6, seed=21)
    R, T, K = _cams(3, seed=21)
    fa_leaf, fa_ref, group = _alpha(alpha, 3, scene['faces'].shape[0], tpl.BNF, seed=Kf)
    d = _dev_scene(scene, dev, texels4=True)
    _camera_parity(tag, scene, R, T, K, size, sigma, Kf, d, fa_ref=fa_ref, fa_dev=_dev_alpha(fa_leaf, dev), group=group, seed=Kf,
                   detach=detach, clip_inside=clip_inside)


@pytest.mark.parametrize('Kf,sigma', [(10, 1e-4), (1, 0.0)])
def test_views_that_see_nothing_get_zero(Kf, sigma):
    """a view turned away from the scene and one whose frustum misses it: exactly zero (finite) pose gradient"""
    dev = _dev()
    tpl, _, scene = _blocks(4, seed=16)
    R, T, K = _cams(3, seed=16)
    R, T = _away_views(R, T)
    d = _dev_scene(scene, dev)
    _camera_parity(f'away K={Kf}', scene, R, T, K, (32, 40), sigma, Kf, d, seed=3, zero_views=(3, 4))


# ------------------------------------------------------------------------------------------------ parity: environment
@pytest.mark.parametrize('generic', [False, True], ids=['hard_kernel', 'generic_kernel'])
def test_environment_camera_gradients_match_oracle(generic):
    """hard single-layer environment pass (sigma = 0, K = 1) with n_static_faces = the background sphere: the sphere moves in
    the image with the camera, so its barycentric path must reach g_R / g_T"""
    from dbw_b200 import _lib
    dev = _dev()
    tpl, scene, R, T, K = _env_scene()
    n_bkg = tpl.bkg_faces.shape[0]
    d = _dev_scene(scene, dev, texels4=True)
    L = _lib.lib()
    L.dbw_debug_generic_kernel_only(1 if generic else 0)
    try:
        _, frags = _oracle(scene, R, T, K, (40, 48), 0.0, 1)
        assert frags.unclipped_to_clipped is not None, 'no face is z-clipped'
        f0 = frags.pix_to_face[..., 0]
        assert ((f0 >= 0) & (f0 % scene['faces'].shape[0] < n_bkg)).float().mean() > 0.1, 'the sphere is hardly seen'
        _camera_parity(f'env generic={generic}', scene, R, T, K, (40, 48), 0.0, 1, d, n_static_faces=n_bkg, seed=5,
                       max_ambiguous=1e-2, conditioning=True)
    finally:
        L.dbw_debug_generic_kernel_only(0)


def test_environment_soft_camera_gradients_match_oracle():
    """the same scene at sigma > 0 (distance gradients of the halo, the generic forward)"""
    dev = _dev()
    tpl, scene, R, T, K = _env_scene(seed=10)
    d = _dev_scene(scene, dev, texels4=True)
    _camera_parity('env soft', scene, R, T, K, (40, 48), 1e-4, 1, d, n_static_faces=tpl.bkg_faces.shape[0], seed=6,
                   max_ambiguous=1e-2, conditioning=True)


# ------------------------------------------------------------------------------------------------ the C-ABI contract
def _abi(d, R, T, K, size, sigma, Kf, fa=None, group=1, n_static_faces=0, detach=False):
    """forward once through the C-ABI; returns backward(want_cams) -> (g_verts, g_maps, g_fa, g_R, g_T)"""
    from dbw_b200 import _lib
    from dbw_b200.renderer import _c, _stream, scene_settings
    dev = _dev()
    L = _lib.lib()
    B = R.shape[0]
    verts, maps = d['verts'].detach(), d['maps'].detach()
    R, T = R.float().to(dev).contiguous(), T.float().to(dev).contiguous()
    cfg, table = scene_settings(verts, d['faces'], maps, d['table'], B, intrinsics(K), size, sigma, Kf, z_clip=0.001,
                                detach_bary=detach, faces_alpha=fa, maps_are_texels4=d['texels4'], alpha_group=group,
                                n_static_faces=n_static_faces)
    assert cfg.save_fragment_state
    fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(L.dbw_workspace_bytes(ctypes.byref(cfg), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
    ws = torch.empty(fwd.value, dtype=torch.uint8, device=dev)
    out = torch.empty(B, 4, *size, device=dev)
    _lib.check(L.dbw_render_forward(ctypes.byref(cfg), _c(verts), _c(d['faces']), _c(d['fvu']), _c(d['fmap']), _c(maps), _c(table),
                                    _c(R), _c(T), _c(fa), _c(out), None, _c(ws), ws.numel(), None, None, _stream()),
               'dbw_render_forward')
    grad = torch.rand(B, 4, *size, generator=torch.Generator().manual_seed(4)).to(dev)

    def backward(cams):
        g = [torch.zeros_like(verts), torch.zeros_like(maps), torch.zeros_like(fa) if fa is not None else None,
             torch.zeros(B, 3, 3, device=dev) if cams else None, torch.zeros(B, 3, device=dev) if cams else None]
        scratch = torch.empty(bwd.value, dtype=torch.uint8, device=dev)
        _lib.check(L.dbw_render_backward(ctypes.byref(cfg), _c(verts), _c(d['faces']), _c(d['fvu']), _c(d['fmap']), _c(maps), _c(table),
                                         _c(R), _c(T), _c(fa), _c(ws), ws.numel(), _c(grad), None, _c(g[0]), _c(g[2]), _c(g[1]),
                                         _c(g[3]), _c(g[4]), _c(scratch), scratch.numel(), _stream()), 'dbw_render_backward')
        torch.cuda.synchronize()
        return g
    return backward


def _abi_cases():
    dev = _dev()
    tpl, _, scene = _blocks(5, seed=12)
    R, T, K = _cams(2, seed=12)
    fa_leaf, _, group = _alpha('batch', 2, scene['faces'].shape[0], tpl.BNF, seed=3)
    yield 'blocks', _abi(_dev_scene(scene, dev, texels4=True), R, T, K, (40, 56), 1e-4, 10, fa=fa_leaf.float().to(dev), group=group), 0
    tpl, env, R, T, K = _env_scene()
    n_bkg = tpl.bkg_faces.shape[0]
    yield 'env', _abi(_dev_scene(env, dev, texels4=True), R, T, K, (40, 48), 0.0, 1, n_static_faces=n_bkg), env['faces'][:n_bkg]


def test_camera_gradients_leave_the_other_gradients_alone():
    """with cameras on, g_maps, g_faces_alpha and the rows of g_verts that no static face touches are those of the camera-less
    call (g_R = g_T = NULL; to the atomics' order); the static faces' vertices now get gradient too, and one reduction launch
    is added"""
    from dbw_b200 import _lib
    for name, backward, static_faces in _abi_cases():
        ref = backward(False)
        n0 = _lib.launch_count()
        got = backward(True)
        n1 = _lib.launch_count()
        backward(False)
        assert (n1 - n0) - (_lib.launch_count() - n1) == 1, name
        V = ref[0].shape[0]
        static_v = torch.zeros(V, dtype=torch.bool)
        if torch.is_tensor(static_faces) and static_faces.numel():
            static_v[static_faces.reshape(-1)] = True
            assert got[0][static_v.to(got[0].device)].abs().max() > 0, f'{name}: the static vertices got no gradient'
        keep = (~static_v).to(got[0].device)
        for x, y, what in ((got[0][keep], ref[0][keep], 'verts'), (got[1], ref[1], 'maps'), (got[2], ref[2], 'alpha')):
            if y is None:
                continue
            assert y.abs().max() > 0, f'{name} {what}'
            assert (x - y).norm() <= 1e-6 * y.norm(), f'{name} {what}: {((x - y).norm() / y.norm()).item():.3e}'
        assert got[3].abs().max() > 0 and got[4].abs().max() > 0


@pytest.mark.parametrize('Kf,sigma,detach', [(1, 0.0, False), (3, 1e-4, False), (10, 1e-4, True)])
def test_row_bands_sum_to_the_full_camera_gradient(Kf, sigma, detach):
    dev = _dev()
    tpl, _, scene = _blocks(5, seed=12)
    R, T, K = _cams(2, seed=12)
    H, W = 72, 40
    d = _dev_scene(scene, dev)
    wgt = torch.rand(2, 4, H, W, generator=torch.Generator().manual_seed(8)).to(dev)

    def run(rows):
        Rd, Td = R.float().to(dev).requires_grad_(True), T.float().to(dev).requires_grad_(True)
        vr = None if rows is None else torch.tensor(rows, dtype=torch.int32, device=dev)
        out, _ = _render(d, Rd, Td, K, (H, W), sigma, Kf, detach=detach, view_rows=vr)
        return torch.autograd.grad(out, [Rd, Td], grad_outputs=wgt)

    full, full2 = run(None), run(None)
    total = [torch.zeros_like(g) for g in full]
    for rows in BANDS:
        total = [s + g for s, g in zip(total, run(rows))]
    for a, b, b2, what in zip(total, full, full2, ('g_R', 'g_T')):
        assert b.abs().max() > 0
        _close_to_cuda(a, b, b2, f'band sum {what}', floor=1e-5)


def test_fused_loss_camera_gradients_equal_the_composite_path():
    """scene_mse (loss epilogue, both passes accumulating into one g_R / g_T) against render -> dbw_composite_mse"""
    from tests.test_raster_matrix_gpu import _two_passes
    from dbw_b200 import render_scene
    from dbw_b200.dbw import _CompositeMSE
    from dbw_b200.fused_loss import scene_mse
    dev = _dev()
    x, env_pass, blk_pass = _two_passes(dev, 10, 40, 56)

    def rend(p, verts, maps, fa, fmap, R, T):
        r = p.r
        return render_scene(verts, p.faces, p.faces_uvs, fmap, maps, p.map_table_host, R, T, r.cameras.intrinsics(), r.img_size,
                            r.sigma, r.faces_per_pixel, r.z_clip, r.detach_bary, r.clip_inside, r.background_color, fa,
                            r.perspective_correct, blur_radius=r.blur_radius, maps_are_texels4=True, alpha_group=p.alpha_group,
                            n_static_faces=p.n_static_faces)
    grads = []
    for fused in (True, False):
        R, T = x['R'].detach().requires_grad_(True), x['T'].detach().requires_grad_(True)
        if fused:
            loss = scene_mse(x['ev'], x['em'], x['bv'], x['bm'], x['ba'], R, T, x['imgs'], env_pass, blk_pass, x['fmap'])
        else:
            env = rend(env_pass, x['ev'], x['em'], None, env_pass.face_map, R, T)
            fg = rend(blk_pass, x['bv'], x['bm'], x['ba'], x['fmap'], R, T)
            loss = _CompositeMSE.apply(fg, env, x['imgs'], x['imgs'].shape[0])[1]
        grads.append(torch.autograd.grad(loss, [R, T]))
    for a, b, what in zip(*grads, ('g_R', 'g_T')):
        assert b.abs().max() > 0, what
        assert (a - b).norm() <= 1e-4 * b.norm(), (what, ((a - b).norm() / b.norm()).item())


# ------------------------------------------------------------------------------------------------ the model
def _pose_inputs(dev, B=3):
    """model inputs whose R and T are computed from leaves (a correction on top of the dataset poses)"""
    inp, imgs, R, T, K = _model_inputs(dev, B=B)
    dR = torch.zeros(B, 3, 3, device=dev, requires_grad=True)
    dT = torch.zeros(B, 3, device=dev, requires_grad=True)
    return inp, imgs, R, T, K, dR, dT


def _pose_step(model, inp, dR, dT, R0, T0):
    step = dict(inp, R=R0 + dR, T=T0 + dT)
    losses = model(step, None)
    return torch.autograd.grad(losses['total'], [dR, dT])


def test_model_paths_give_the_oracle_pose_gradients():
    """model(inp) with poses computed from leaves: the fused-loss path, fused_loss = False (_CompositeMSE), the eager
    static-topology path and the Meshes path all reach the leaves with the gradient of the oracle's predict + mse_loss"""
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.01
    Rl, Tl = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    rec_ref = D.predict(tpl, p, Rl, Tl, K, (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, keep=keep, decimate=8)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)
    print(f'decision-masked pixels: {bad.double().mean().item() * 100:.4f}%')
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    ref = torch.autograd.grad(D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref), [Rl, Tl])
    R0, T0 = inp['R'], inp['T']
    paths = {'fused_loss': {}, 'composite': dict(fused_loss=False), 'eager_static': dict(fused_loss=False, fused_scene=False),
             'meshes': dict(fused_loss=False, fused_scene=False, static_topology=False)}
    got = {}
    for name, attrs in paths.items():
        model.fused_loss, model.fused_scene, model.static_topology = True, True, True
        for k, v in attrs.items():
            setattr(model, k, v)
        if name == 'fused_loss':
            assert model._fused_loss_ok(inp['imgs'])
        got[name] = _pose_step(model, inp, dR, dT, R0, T0)
        for g, r, what in zip(got[name], ref, ('R', 'T')):
            rel = _rel(g.cpu().double(), r)
            print(f'{name} d/d{what}: rel err {rel:.3e}')
            assert rel < 1e-3, f'{name} d/d{what}: rel err {rel:.3e}'
    for name in ('composite', 'eager_static', 'meshes'):
        for a, b in zip(got[name], got['fused_loss']):
            assert (a - b).norm() <= 1e-4 * b.norm(), name


def test_joint_render_mode_reaches_the_pose_leaves():
    from copy import deepcopy
    from tests.test_model_gpu import CFG
    from dbw_b200.dbw import DifferentiableBlocksWorld
    dev = _dev()
    torch.manual_seed(5)
    cfg = deepcopy(CFG)
    cfg['rend_optim'].update(decouple_rendering=False, kill_blocks=False)
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev).train()
    model.loss_weights = {'rgb': 1.0}
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    tpl = D.SceneTemplate(n_blocks=5, txt_size=32)
    p = {k: v.detach().cpu().double() for k, v in model.named_parameters()}
    Rl, Tl = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    rec_ref = D.predict_joint(tpl, p, Rl, Tl, K, (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, decimate=8)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    ref = torch.autograd.grad(D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref), [Rl, Tl])
    got = _pose_step(model, inp, dR, dT, inp['R'], inp['T'])
    for g, r, what in zip(got, ref, ('R', 'T')):
        rel = _rel(g.cpu().double(), r)
        print(f'joint d/d{what}: rel err {rel:.3e}')
        assert rel < 2e-3, f'joint d/d{what}: rel err {rel:.3e}'        # the bound of test_joint_render_mode_matches_oracle


def test_pose_gradients_with_the_lpips_term():
    """with a (random-weight) LPIPS term installed the model takes the composite path; the pose leaves still get gradient,
    and the term changes it"""
    from dbw_b200.dbw import PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    from oracle import lpips as OL
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    model.set_perceptual_loss(PerceptualTerm(LPIPS.from_state_dict(OL.random_state_dict(2))).to(dev))
    model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
    model.eval()                                  # no dropout: the two steps below differ only by the term
    assert not model._fused_loss_ok(inp['imgs'])
    with_term = _pose_step(model, inp, dR, dT, inp['R'], inp['T'])
    model.loss_weights = {'rgb': 1.0}
    without = _pose_step(model, inp, dR, dT, inp['R'], inp['T'])
    for a, b, what in zip(with_term, without, ('R', 'T')):
        assert torch.isfinite(a).all() and a.abs().max() > 0, what
        assert (a - b).norm() > 1e-3 * b.norm(), f'{what}: the perceptual term does not reach the pose'


def test_launch_count_adds_only_the_reductions():
    """a step without pose gradients launches what it did before (no reduction); with them, one reduction per pass"""
    from dbw_b200 import _lib
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    for fused in (True, False):
        model.fused_loss = fused

        def count(with_pose):
            model.zero_grad(set_to_none=True)
            step = dict(inp, R=R0 + dR, T=T0 + dT) if with_pose else inp
            n = _lib.launch_count()
            model(step, None)['total'].backward()
            torch.cuda.synchronize()
            return _lib.launch_count() - n

        R0, T0 = inp['R'], inp['T']
        count(False); count(True)                                 # warm-up: lazy state
        plain, posed, plain2 = count(False), count(True), count(False)
        assert plain == plain2 and posed - plain == 2, (fused, plain, posed)


def test_sharded_and_graphed_steps_refuse_pose_gradients():
    from dbw_b200.graph import GraphedStep, PipelinedGraphedStep
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    vp = ViewParallel(model, seed=5)
    for key, leaf in (('R', dR), ('T', dT)):
        posed = dict(inp, **{key: inp[key] + leaf})
        with pytest.raises(RuntimeError, match='requires grad'):
            vp.forward_backward(posed)
        with pytest.raises(RuntimeError, match='requires grad'):
            GraphedStep(vp, posed, len(imgs))
        with pytest.raises(RuntimeError, match='requires grad'):
            PipelinedGraphedStep(vp, posed, len(imgs))
    assert dR.grad is None and dT.grad is None


# ------------------------------------------------------------------------------------------------ pose recovery
def _rotation_error_deg(Ra, Rb):
    c = ((Ra.transpose(1, 2) @ Rb).diagonal(dim1=1, dim2=2).sum(-1) - 1) / 2
    return torch.rad2deg(torch.acos(c.clamp(-1, 1)))


POSE_STEPS = 300
POSE_LR = 4e-3


def test_pose_recovery_from_perturbed_cameras():
    """a fixed scene and targets rendered from the true cameras; each view's pose perturbed in its camera frame by a 3-5
    degree rotation about the camera centre and a translation of 3-5 % of |T|; Adam on a camera-frame 6-D rotation and
    translation delta per view (X_view = (X R_init + T_init) Rot(r6) + dt; the scene frozen: a camera-only backward) must
    bring the mean rotation and translation errors below a quarter of their initial values.  The scene has smooth,
    high-contrast textures (4 x 4 random logits of amplitude 3, upsampled) so that the images constrain the pose.  A pose
    perturbed about the world origin instead (R_init = R_true Rot, as first tried) mostly orbits the scene: rotation and
    translation then trade off against each other and 200 steps left the rotation error where it started.  Measured on an
    H100 80GB HBM3 with these seeds: 3.82 -> 0.68 degrees and 0.202 -> 0.0054 in 300 steps (the bound is 1/4: 0.96 degrees
    and 0.051); the step count and learning rate come from that run."""
    from copy import deepcopy
    from dbw_b200 import geometry as G
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from tests.test_model_gpu import CFG
    dev = _dev()
    torch.manual_seed(5)
    model = DifferentiableBlocksWorld((96, 128), **deepcopy(CFG)).to(dev).eval()      # eval: no texture decimation
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for t in (model.textures, model.texture_bkg, model.texture_ground):
            low = 3 * torch.randn(t.shape[0], 3, 4, 4, generator=g)
            t.copy_(torch.nn.functional.interpolate(low, size=t.shape[1:3], mode='bilinear', align_corners=True).permute(0, 2, 3, 1))
    for q in model.parameters():
        q.requires_grad_(False)
    model.loss_weights = {'rgb': 1.0}
    inp, *_ = _model_inputs(dev, B=4, size=(96, 128), seed=11)
    R_true, T_true = inp['R'], inp['T']
    with torch.no_grad():
        inp['imgs'] = model.predict(inp).clamp(0, 1)
    axis = torch.nn.functional.normalize(torch.randn(4, 3, generator=g), dim=-1)
    angle = torch.deg2rad(3 + 2 * torch.rand(4, 1, generator=g))
    Rp = _axis_angle(axis * angle).to(dev)
    dirs = torch.nn.functional.normalize(torch.randn(4, 3, generator=g), dim=-1).to(dev)
    R_init = R_true @ Rp
    T_init = (T_true[:, None] @ Rp)[:, 0] + dirs * T_true.norm(dim=-1, keepdim=True) * (0.03 + 0.02 * torch.rand(4, 1, generator=g)).to(dev)
    r6 = torch.tensor([1., 0., 0., 0., 1., 0.], device=dev).repeat(4, 1).requires_grad_(True)
    dt = torch.zeros(4, 3, device=dev, requires_grad=True)
    opt = torch.optim.Adam([r6, dt], lr=POSE_LR)
    sched = torch.optim.lr_scheduler.StepLR(opt, POSE_STEPS // 3, 0.5)

    def pose():
        Rot = G.rotation_6d_to_matrix(r6)
        return R_init @ Rot, (T_init[:, None] @ Rot)[:, 0] + dt

    def errors():
        with torch.no_grad():
            R, T = pose()
            return _rotation_error_deg(R, R_true).mean().item(), (T - T_true).norm(dim=-1).mean().item()

    e0 = errors()
    for it in range(POSE_STEPS):
        opt.zero_grad(set_to_none=True)
        R, T = pose()
        loss = model(dict(inp, R=R, T=T), None)['total']
        loss.backward()
        opt.step()
        sched.step()
        if it % 25 == 0 or it == POSE_STEPS - 1:
            e = errors()
            print(f'step {it}: loss {loss.item():.4e}, rotation {e[0]:.3f} deg, translation {e[1]:.4f}')
    e1 = errors()
    print(f'initial errors {e0[0]:.3f} deg / {e0[1]:.4f}, final {e1[0]:.3f} deg / {e1[1]:.4f}')
    assert e1[0] < e0[0] / 4 and e1[1] < e0[1] / 4


def _axis_angle(v):
    """Rodrigues: (N,3) axis * angle -> (N,3,3)"""
    theta = v.norm(dim=-1, keepdim=True)[..., None]
    k = v / v.norm(dim=-1, keepdim=True)
    Kx = torch.zeros(len(v), 3, 3)
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 0] = -k[:, 2], k[:, 1], k[:, 2]
    Kx[:, 1, 2], Kx[:, 2, 0], Kx[:, 2, 1] = -k[:, 0], -k[:, 1], k[:, 0]
    return torch.eye(3)[None] + torch.sin(theta) * Kx + (1 - torch.cos(theta)) * Kx @ Kx
