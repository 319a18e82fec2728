"""GPU: the depth outputs of render_scene (return_depth / return_zbuf, dbw_render_forward_depth / dbw_render_backward_depth)
and of the scene model (DifferentiableBlocksWorld.predict(with_depth=True), predict_depth) against the float64 oracle:
zbuf = oracle.pt3d.rasterize_meshes' zbuf, depth = oracle.dbw_path.layered_rgb_blend of that zbuf as a one-channel colour over
a background of 0 (composited D_fg + (1 - alpha_fg) D_env over the oracle's predict passes for the model), and their gradients
(with the image's) by torch autograd -- to the vertices, opacities, maps, R, T and per-view intrinsics, and for the model to
every leaf parameter.  Block scenes and the environment scene (background sphere as static faces, ground; the hard and the
split single-layer backward, with and without camera gradients).  Pixels whose kept faces differ between fp32 and fp64 (a
different discrete decision) are excluded, as in tests/test_raster_matrix_gpu.py, whose bars these are: zbuf within 1e-4 of
the scene's depth range, the blended depth within 1e-4 of its largest depth (its weights carry the image's error, times z),
gradients at 1e-3 relative.  Also: the image is the same bits with and without depth, a backward that reads no depth gives the
depth-free gradients up to the atomics' order, and two forwards give the same depth bits."""
import pytest
import torch

from oracle import dbw_path as D
from tests.helpers import decision_mask
from tests.test_raster_matrix_gpu import (_alpha, _blocks, _cams, _close_to_cuda, _close_to_oracle, _dev, _dev_alpha, _dev_scene,
                                          _leaf, _oracle, _render, _split_maps)

pytestmark = pytest.mark.gpu

SIZE = (48, 64)


def _oracle_depth(frags, sigma, clip_inside, fa_ref, B, n_faces):
    fa = fa_ref
    if fa is not None and fa.numel() == n_faces:
        fa = fa.repeat(B)
    z = frags.zbuf
    return D.layered_rgb_blend(z[..., None].expand(*z.shape, 3), frags.pix_to_face, frags.dists, sigma, (0., 0., 0.), clip_inside,
                               fa)[:, :1]


CASES = [  # (K, sigma, detach_bary, opacity layout, clip_inside, z_clip, perspective_correct)
    (1, 0.0, True, None, True, 0.001, True),
    (1, 0.0, False, 'batch', True, None, True),
    (1, 5e-6, False, 'face', True, 0.001, False),
    (10, 1e-4, True, 'block', True, 0.001, True),
    (10, 5e-6, False, None, False, None, True),
    (10, 0.0, True, 'face', True, 0.001, True),
    (25, 1e-4, False, 'batch', False, 0.001, False),
    (25, 1e-4, True, None, True, 0.001, True),
]


@pytest.mark.parametrize('Kf,sigma,detach,alpha,clip_inside,z_clip,persp', CASES)
def test_depth_against_the_oracle(Kf, sigma, detach, alpha, clip_inside, z_clip, persp):
    dev = _dev()
    tpl, _, scene = _blocks(7, seed=3)
    R, T, K = _cams(2, seed=3, dist=1.6)              # close cameras: views that straddle the clip plane
    B, nf = 2, scene['faces'].shape[0]
    fa_leaf, fa_ref, group = _alpha(alpha, B, nf, tpl.BNF, seed=Kf)
    d = _dev_scene(scene, dev)
    fa_dev = _dev_alpha(fa_leaf, dev)
    R_dev = R.float().to(dev).requires_grad_(True)
    T_dev = T.float().to(dev).requires_grad_(True)
    R64, T64 = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    ref, frags = _oracle(scene, R64, T64, K, SIZE, sigma, Kf, z_clip=z_clip, detach=detach, fa=fa_ref, clip_inside=clip_inside,
                         perspective_correct=persp)
    ref_d = _oracle_depth(frags, sigma, clip_inside, fa_ref, B, nf)
    from dbw_b200 import render_scene
    from tests.helpers import intrinsics
    out, ids, dep, zb = render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R_dev, T_dev, intrinsics(K),
                                     SIZE, sigma, Kf, z_clip=z_clip, detach_bary=detach, clip_inside=clip_inside, faces_alpha=fa_dev,
                                     perspective_correct=persp, return_ids=True, alpha_group=group, return_depth=True,
                                     return_zbuf=True)
    mask = decision_mask(ids, frags, nf)                                    # (B,1,H,W) pixels with the oracle's decisions
    assert 1 - mask.mean().item() <= 2e-3
    zr, valid = _compare_outputs(zb, dep, frags, ref_d, mask)
    _check_grads(scene, d, ref, ref_d, zr, out, dep, zb, mask, valid, [R64, T64], [R_dev, T_dev], fa_leaf, fa_dev,
                 f'K={Kf} sigma={sigma}')


def _check_grads(scene, d, ref, ref_d, zr, out, dep, zb, mask, valid, cams_ref, cams_dev, fa_leaf, fa_dev, tag):
    """one loss over the image, the depth and the zbuf; gradients to the vertices, the maps, the cameras given and the opacities"""
    g = torch.Generator().manual_seed(7)
    w_rgba = torch.rand(out.shape, generator=g, dtype=torch.float64) * mask
    w_d = torch.rand(dep.shape, generator=g, dtype=torch.float64) * mask
    w_z = torch.rand(zb.shape, generator=g, dtype=torch.float64) * mask * valid
    n_maps = len(scene['maps'])
    leaves_ref = [scene['verts'], *scene['maps'], *cams_ref] + ([fa_leaf] if fa_leaf is not None else [])
    leaves_dev = [d['verts'], d['maps'], *cams_dev] + ([fa_dev] if fa_dev is not None else [])
    loss_ref = (ref * w_rgba).sum() + (ref_d * w_d).sum() + (zr * w_z).sum()
    g_ref = list(torch.autograd.grad(loss_ref, leaves_ref, allow_unused=True))
    g_dev = torch.autograd.grad([out, dep, zb], leaves_dev, grad_outputs=[w_rgba.to(out.device).float(), w_d.to(out.device).float(),
                                                                           w_z.to(out.device).float()])
    zero = lambda r, leaf: r if r is not None else torch.zeros(leaf.shape, dtype=torch.float64)
    _close_to_oracle(g_dev[0], zero(g_ref[0], leaves_ref[0]), f'{tag} verts')
    for j, gm in enumerate(_split_maps(g_dev[1], d['table'], d['texels4'])):
        _close_to_oracle(gm, zero(g_ref[1 + j], leaves_ref[1 + j]), f'{tag} maps[{j}]')
    names = ['R', 'T'][:len(cams_dev)] + (['alpha'] if fa_dev is not None else [])
    for name, a, b, leaf in zip(names, g_dev[2:], g_ref[1 + n_maps:], leaves_ref[1 + n_maps:]):
        _close_to_oracle(a, zero(b, leaf), f'{tag} {name}')


def _compare_outputs(zb, dep, frags, ref_d, mask):
    zr = frags.zbuf.permute(0, 3, 1, 2)                                     # (B,K,H,W)
    valid = zr > 0
    assert valid.any()
    zrange = (zr[valid].max() - zr[valid].min()).item()
    err_z = ((zb.detach().cpu().double() - zr).abs() * mask).max().item()
    assert err_z <= 1e-4 * zrange, f'zbuf err {err_z:.3e} (range {zrange:.3e})'
    m = mask.bool().expand_as(valid)
    assert torch.equal((zb.detach().cpu() == -1) & m, ~valid & m), 'empty slots are -1'
    # depth = sum_k w_k z_k: the weights carry the image's error (its 1e-4 bar, absolute on colours in [0, 1]) multiplied by z,
    # so the depth's bar is 1e-4 of the largest depth, not of the range
    err_d = ((dep.detach().cpu().double() - ref_d).abs() * mask).max().item()
    zmax = zr[valid].max().item()
    assert err_d <= 1e-4 * zmax, f'depth err {err_d:.3e} (max depth {zmax:.3e})'
    return zr, valid


@pytest.mark.parametrize('detach,cams', [(False, False), (False, True), (True, False), (True, True)])
def test_environment_scene_depth(detach, cams):
    """the environment pass: hard single layer, background sphere as static faces (no vertex gradient unless the cameras are
    differentiated, which makes every face move), the ground's depth reaching its vertices; not detached = the split backward
    (depth_backward_kernel, then raster_bary_backward_kernel for the colour's barycentrics, both into the slot gradients)"""
    dev = _dev()
    tpl = D.SceneTemplate(n_blocks=2, txt_size=16)
    p = D.init_params(2, 16, seed=9, dtype=torch.float64)
    R, T, K = _cams(2, seed=9)
    K = K.clone(); K[0, 0] = K[1, 1] = 1.2            # wide enough to see the horizon: background sphere and ground
    scene = _leaf(tpl.build_env(p))
    n_bkg_f, n_bkg_v = tpl.bkg_faces.shape[0], tpl.bkg_verts.shape[0]
    R64, T64 = R.clone().requires_grad_(cams), T.clone().requires_grad_(cams)
    scene_o = scene
    if not cams:        # the oracle has no notion of static faces: the background vertices reach it as constants
        keep = torch.ones(scene['verts'].shape[0], 1, dtype=torch.float64)
        keep[:n_bkg_v] = 0
        scene_o = dict(scene, verts=scene['verts'] * keep + scene['verts'].detach() * (1 - keep))
    ref, frags = _oracle(scene_o, R64, T64, K, SIZE, 0.0, 1, detach=detach)
    nf = scene['faces'].shape[0]
    assert (frags.pix_to_face[..., 0] % nf >= n_bkg_f).any() and (frags.pix_to_face[..., 0] % nf < n_bkg_f).any()
    ref_d = _oracle_depth(frags, 0.0, True, None, 2, nf)
    d = _dev_scene(scene, dev)
    R_dev, T_dev = R.float().to(dev).requires_grad_(cams), T.float().to(dev).requires_grad_(cams)
    from dbw_b200 import render_scene
    from tests.helpers import intrinsics
    out, ids, dep, zb = render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R_dev, T_dev, intrinsics(K),
                                     SIZE, 0.0, 1, z_clip=0.001, detach_bary=detach, return_ids=True, n_static_faces=n_bkg_f,
                                     return_depth=True, return_zbuf=True)
    mask = decision_mask(ids, frags, nf)
    assert 1 - mask.mean().item() <= 2e-3
    zr, valid = _compare_outputs(zb, dep, frags, ref_d, mask)
    _check_grads(scene, d, ref, ref_d, zr, out, dep, zb, mask, valid, [R64, T64] if cams else [], [R_dev, T_dev] if cams else [],
                 None, None, f'env detach={detach} cams={cams}')


def test_depth_gradient_to_per_view_intrinsics():
    dev = _dev()
    _, _, scene = _blocks(5, seed=5)
    R, T, K = _cams(2, seed=5)
    Kv = K.reshape(1, 4, 4).repeat(2, 1, 1).clone()
    Kv[1, 0, 0] *= 1.1
    Kv64 = Kv.clone().requires_grad_(True)
    from oracle import pt3d
    ndc = torch.cat([pt3d.world_to_ndc(scene['verts'], R[b:b + 1], T[b:b + 1], Kv64[b]) for b in range(2)])     # one K per view
    fr = pt3d.rasterize_meshes(ndc, scene['faces'], SIZE, blur_radius=D.blur_radius_from_sigma(1e-4), faces_per_pixel=10,
                               z_clip_value=0.001)
    ref_d = _oracle_depth(fr, 1e-4, True, None, 2, scene['faces'].shape[0])
    d = _dev_scene(scene, dev)
    Kd = Kv.float().to(dev).requires_grad_(True)
    from dbw_b200 import render_scene
    out, ids, dep = render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R.float().to(dev),
                                 T.float().to(dev), Kd, SIZE, 1e-4, 10, z_clip=0.001, return_ids=True, return_depth=True)
    mask = decision_mask(ids, fr, scene['faces'].shape[0])
    w = torch.rand(dep.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * mask
    g_ref, = torch.autograd.grad((ref_d * w).sum(), [Kv64])
    g_dev, = torch.autograd.grad(dep, [Kd], grad_outputs=w.to(dev).float())
    sel = torch.zeros(4, 4, dtype=torch.bool)
    sel[0, 0] = sel[1, 1] = sel[0, 2] = sel[1, 2] = True
    _close_to_oracle(g_dev[:, sel], g_ref[:, sel], 'intrinsics')


def test_rgba_unchanged_and_repeatable():
    dev = _dev()
    tpl, _, scene = _blocks(7, seed=3)
    R, T, K = _cams(2, seed=3)
    for Kf, sigma, detach in ((10, 1e-4, True), (1, 0.0, False), (25, 1e-4, False)):
        d = _dev_scene(scene, dev)
        fa = torch.rand(2 * scene['faces'].shape[0] // tpl.BNF, generator=torch.Generator().manual_seed(1)).to(dev) * 0.7 + 0.3
        fa.requires_grad_(True)
        kw = dict(detach=detach, fa=fa, alpha_group=tpl.BNF)
        out0, _ = _render(d, R, T, K, SIZE, sigma, Kf, **kw)
        g0 = torch.rand_like(out0)
        base = torch.autograd.grad(out0, [d['verts'], d['maps'], fa], grad_outputs=g0)
        out1, _ = _render(d, R, T, K, SIZE, sigma, Kf, **kw)
        spread = torch.autograd.grad(out1, [d['verts'], d['maps'], fa], grad_outputs=g0)
        from dbw_b200 import render_scene
        from tests.helpers import intrinsics
        res = [render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R.float().to(dev), T.float().to(dev),
                            intrinsics(K), SIZE, sigma, Kf, z_clip=0.001, detach_bary=detach, faces_alpha=fa, alpha_group=tpl.BNF,
                            return_depth=True) for _ in range(2)]
        assert torch.equal(res[0][0], out0), 'the image changed when depth was asked for'
        assert torch.equal(res[0][1], res[1][1]), 'two forwards gave different depth bits'
        got = torch.autograd.grad(res[0][0], [d['verts'], d['maps'], fa], grad_outputs=g0)        # nothing reads the depth
        for a, b, c, n in zip(got, base, spread, ('verts', 'maps', 'alpha')):
            _close_to_cuda(a, b, c, f'K={Kf} {n}')


# ------------------------------------------------------------------------------------------------ the scene model
def _oracle_pass_depth(scene, R, T, K, sigma, Kf, detach, fa):
    out, frags = D.render(scene, R, T, K, SIZE, sigma=sigma, faces_per_pixel=Kf, z_clip=0.001, detach_bary=detach, faces_alpha=fa,
                          return_fragments=True)
    return out, _oracle_depth(frags, sigma, True, fa, R.shape[0], scene['faces'].shape[0])


def _oracle_predict_depth(tpl, p, R, T, K, sigma, fine, keep, decimate):
    """oracle.dbw_path.predict's two passes with their depths: (rec, D_fg + (1 - alpha_fg) D_env)"""
    env = tpl.build_env(p, decimate=decimate)
    out_e, d_env = _oracle_pass_depth(env, R, T, K, 0.0, 1, False, None)
    blocks, alpha = tpl.build_blocks(p, keep=keep, decimate=decimate)
    fa = None if fine else alpha.repeat_interleave(tpl.BNF).repeat(R.shape[0])
    out_f, d_fg = _oracle_pass_depth(blocks, R, T, K, sigma, 10, True, fa)
    a = out_f[:, 3:]
    return out_f[:, :3] * a + (1 - a) * out_e[:, :3], d_fg + (1 - a) * d_env


@pytest.mark.parametrize('fine', [False, True])
def test_model_predict_with_depth(fine):
    """predict(inp, with_depth=True) against the oracle's predict passes, and the gradients of a depth + RGB loss to every
    leaf parameter and to the poses; predict_depth is its depth"""
    from tests.test_model_gpu import CFG, _inputs, _model_and_oracle
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    inp, imgs, R, T, K = _inputs(dev)
    keep = torch.sigmoid(p['alpha_logit'].detach()) > (0.5 if fine else 0.01)
    assert CFG['rend_optim']['kill_blocks']
    sigma = 5e-6 if fine else 1e-4
    R64, T64 = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    rec_ref, dep_ref = _oracle_predict_depth(tpl, p, R64, T64, K, sigma, fine, keep, 0 if fine else 8)
    inp['R'].requires_grad_(True)
    inp['T'].requires_grad_(True)
    rec, dep = model.predict(inp, with_depth=True)
    assert rec.shape == (3, 3, *SIZE) and dep.shape == (3, 1, *SIZE)
    assert torch.equal(rec, model.predict(inp)), 'with_depth changed the reconstruction'
    assert torch.equal(dep, model.predict_depth(inp))
    err = (rec.detach().cpu().double() - rec_ref.detach()).abs()
    good = ~(err > 1e-4).any(1, keepdim=True)                         # pixels where fp32 takes the oracle's discrete decisions
    assert 1 - good.double().mean().item() < 2e-3
    zmax = dep_ref.max().item()
    err_d = ((dep.detach().cpu().double() - dep_ref.detach()).abs() * good).max().item()
    assert err_d <= 1e-4 * zmax, f'depth err {err_d:.3e} (max depth {zmax:.3e})'
    g = torch.Generator().manual_seed(11)
    w_rec = torch.rand(rec.shape, generator=g, dtype=torch.float64) * good
    w_d = torch.rand(dep.shape, generator=g, dtype=torch.float64) * good
    ((rec_ref * w_rec).sum() + (dep_ref * w_d).sum()).backward()
    torch.autograd.backward([rec, dep], [w_rec.float().to(dev), w_d.float().to(dev)])
    checked = 0
    cams = {'camera R': (inp['R'], R64), 'camera T': (inp['T'], T64)}          # (the model has parameters named R and T)
    for name, prm in list(model.named_parameters()) + [(k, v[0]) for k, v in cams.items()]:
        g_ref = cams[name][1].grad if name in cams else p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            assert prm.grad is None or prm.grad.abs().max().item() < 1e-12, name
            continue
        rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        assert rel < 1e-3, f'{name}: rel grad err {rel:.3e}'
        checked += 1
    assert checked >= 6
