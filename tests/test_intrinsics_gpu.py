"""GPU: rendering each view with its own intrinsics, and their gradient (dbw_camera_project{,_backward},
renderer.project_verts, model.set_per_view_intrinsics).

1. Parity with the float64 oracle, which projects each view with its own K (oracle.pt3d.world_to_ndc, one call per view:
   the oracle takes one K per call, and rendering one view at a time with its own K is the intended per-view reference;
   tests/test_intrinsics_model_gpu.py does the same with the model-level oracle) and differentiates K, R, T and the leaves by
   autograd: distinct K per view (+-5 % focal, shifted principal points) at
   K = 1 / 10 / 25 faces per pixel, the z-clipped environment with its static faces, row bands.  Tolerances are those of
   tests/test_raster_matrix_gpu.py: images 1e-4; gradients 1e-3 relative L2 plus an element bound, over the pixels whose
   kept faces agree between fp32 and fp64.
2. Every view's K equal to K[0]: images, loss terms and NDC vertices equal the single-camera path bit for bit; gradients
   agree to within the atomics' summation order.
3. The model and the step objects: a focal-scale leaf gets the eager gradient through GraphedStep (with and without
   BucketAdam) and ViewParallel; a replay with a new K renders with it; the refusals."""
import pytest
import torch

from oracle import dbw_path as D
from tests.helpers import decision_mask, intrinsics
from tests.test_camera_grad_gpu import _env_scene
from tests.test_model_gpu import _inputs as _model_inputs, _model_and_oracle
from tests.test_raster_matrix_gpu import BANDS, _blocks, _cams, _close_to_oracle, _dev_scene, _oracle, _rel

pytestmark = pytest.mark.gpu
SAME_RESULTS = 1e-6          # gradients of two summation orders: of each array's largest magnitude


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _per_view_K(K, B, seed):
    """(B,4,4) float64: K with +-5 % focal lengths and principal points shifted by up to 0.1 per view"""
    g = torch.Generator().manual_seed(seed)
    Ks = K.reshape(4, 4)[None].repeat(B, 1, 1)
    Ks[:, 0, 0] *= 1 + 0.05 * (2 * torch.rand(B, generator=g, dtype=torch.float64) - 1)
    Ks[:, 1, 1] *= 1 + 0.05 * (2 * torch.rand(B, generator=g, dtype=torch.float64) - 1)
    Ks[:, 0, 2] += 0.1 * (2 * torch.rand(B, generator=g, dtype=torch.float64) - 1)
    Ks[:, 1, 2] += 0.1 * (2 * torch.rand(B, generator=g, dtype=torch.float64) - 1)
    return Ks


def _oracle_views(scene, R, T, Ks, size, sigma, Kf, **opts):
    """float64 render of each view with its own K -> ((B,4,H,W), per-view fragments)"""
    outs = [_oracle(scene, R[b:b + 1], T[b:b + 1], Ks[b], size, sigma, Kf, **opts) for b in range(R.shape[0])]
    return torch.cat([o for o, _ in outs]), [f for _, f in outs]


def _render_views(d, R, T, Ks, size, sigma, Kf, n_static_faces=0, view_rows=None, **opts):
    from dbw_b200 import render_scene
    return render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R, T, Ks, size, sigma, Kf,
                        z_clip=opts.get('z_clip', 0.001), detach_bary=opts.get('detach', False), return_ids=True,
                        maps_are_texels4=d['texels4'], n_static_faces=n_static_faces, view_rows=view_rows)


def _parity(tag, scene, R, T, Ks, size, sigma, Kf, n_static_faces=0, seed=0, rel=1e-3, elem=2e-3, max_ambiguous=2e-3, **opts):
    dev = _dev()
    Rl, Tl, Kl = (t.clone().requires_grad_(True) for t in (R, T, Ks))
    ref, frags = _oracle_views(scene, Rl, Tl, Kl, size, sigma, Kf, **opts)
    d = _dev_scene(scene, dev)
    Rd, Td, Kd = (t.detach().float().to(dev).requires_grad_(True) for t in (R, T, Ks))
    out, ids = _render_views(d, Rd, Td, Kd, size, sigma, Kf, n_static_faces=n_static_faces, **opts)
    B, _, H, W = ref.shape
    mask = torch.cat([decision_mask(ids[b:b + 1], frags[b], scene['faces'].shape[0]) for b in range(B)])
    amb = 1 - mask.mean().item()
    print(f'\n{tag}: ambiguous pixels {amb * 100:.3f}%')
    assert amb <= max(max_ambiguous, 1.5 / (B * H * W))
    img_err = ((out.detach().cpu().double() - ref.detach()).abs() * mask).max().item()
    print(f'{tag}: image max err {img_err:.3e}')
    assert img_err < 1e-4, img_err
    wgt = torch.rand(B, 4, H, W, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * mask
    leaves = [Rl, Tl, Kl, scene['verts']]
    ref_g = torch.autograd.grad((ref * wgt).sum(), leaves)
    got = torch.autograd.grad(out, [Rd, Td, Kd, d['verts']], grad_outputs=wgt.to(dev).float())
    idx = ((0, 0), (1, 1), (0, 2), (1, 2))
    for name, g, r in zip(('g_R', 'g_T', 'g_K', 'g_verts'), got, ref_g):
        if name == 'g_K':              # the product reads four entries of K; the oracle's full-matrix product touches all 16
            g = torch.stack([g[:, i, j] for i, j in idx], -1)
            r = torch.stack([r[:, i, j] for i, j in idx], -1)
            assert g.detach().abs().min() > 0, f'{tag}: an intrinsic got no gradient'
        print(f'{tag}: {name} rel err {_rel(g.detach().cpu().double(), r):.3e}')
        _close_to_oracle(g, r, f'{tag} {name}', rel, elem)
    return out


@pytest.mark.parametrize('Kf,sigma', [(1, 0.0), (10, 1e-4), (25, 1e-4)])
def test_blocks_rendered_with_per_view_intrinsics_match_oracle(Kf, sigma):
    tpl, _, scene = _blocks(6, seed=21)
    R, T, K = _cams(3, seed=21)
    _parity(f'blocks K={Kf}', scene, R, T, _per_view_K(K, 3, seed=Kf), (48, 64), sigma, Kf, seed=Kf)


def test_z_clipped_environment_with_per_view_intrinsics_matches_oracle():
    """the hard single-layer environment pass seen from inside the sphere: the static faces take the camera gradient"""
    tpl, scene, R, T, K = _env_scene()
    out = _parity('environment', scene, R, T, _per_view_K(K, 2, seed=4), (40, 56), 0.0, 1, n_static_faces=scene['faces'].shape[0] // 2)
    assert out.shape[0] == 2


def test_row_band_shares_sum_to_the_whole_gradient():
    dev = _dev()
    tpl, _, scene = _blocks(5, seed=12)
    R, T, K = _cams(2, seed=12)
    Ks = _per_view_K(K, 2, seed=12)
    d = _dev_scene(scene, dev)
    H, W = 72, 40
    wgt = torch.rand(2, 4, H, W, generator=torch.Generator().manual_seed(2)).to(dev)
    Rd, Td, Kd = (t.detach().float().to(dev).requires_grad_(True) for t in (R, T, Ks))
    full, _ = _render_views(d, Rd, Td, Kd, (H, W), 1e-4, 10)
    whole = torch.autograd.grad((full * wgt).sum(), [Rd, Td, Kd, d['verts']])
    acc = [torch.zeros_like(g) for g in whole]
    for rows in BANDS:
        vr = torch.tensor(rows, dtype=torch.int32, device=dev)
        part, _ = _render_views(d, Rd, Td, Kd, (H, W), 1e-4, 10, view_rows=vr)
        for a, g in zip(acc, torch.autograd.grad((part * wgt).sum(), [Rd, Td, Kd, d['verts']])):
            a += g
    for name, a, w in zip(('g_R', 'g_T', 'g_K', 'g_verts'), acc, whole):
        err = (a - w).abs().max().item() / w.abs().max().item()
        print(f'row bands {name}: {err:.3e}')
        assert err <= 1e-5, (name, err)


def test_equal_intrinsics_reproduce_the_single_camera_path():
    """every view's K = K[0]: NDC vertices, images bit for bit; gradients within the atomics' order"""
    from dbw_b200 import render_scene
    from dbw_b200.renderer import project_verts
    dev = _dev()
    tpl, _, scene = _blocks(6, seed=21)
    R, T, K = _cams(3, seed=21)
    d = _dev_scene(scene, dev, texels4=True)
    Rd, Td = (t.float().to(dev).requires_grad_(True) for t in (R, T))
    Ks = K.float().reshape(1, 4, 4).repeat(3, 1, 1).to(dev).requires_grad_(True)
    wgt = torch.rand(3, 4, 48, 64, generator=torch.Generator().manual_seed(0)).to(dev)
    worst = 0.0
    for Kf, sigma in ((1, 0.0), (10, 1e-4), (25, 1e-4)):
        args = (d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], Rd, Td)
        kw = dict(z_clip=0.001, maps_are_texels4=True)
        a = render_scene(*args, intrinsics(K), (48, 64), sigma, Kf, **kw)
        b = render_scene(*args, Ks, (48, 64), sigma, Kf, **kw)
        assert torch.equal(a, b), Kf
        ga = torch.autograd.grad((a * wgt).sum(), [d['verts'], d['maps'], Rd, Td])
        gb = torch.autograd.grad((b * wgt).sum(), [d['verts'], d['maps'], Rd, Td])
        for name, x, y in zip(('verts', 'maps', 'R', 'T'), ga, gb):
            err = (x - y).abs().max().item() / y.abs().max().item()
            worst = max(worst, err)
            assert err <= SAME_RESULTS, (Kf, name, err)
    print(f'\nequal intrinsics: largest gradient difference {worst:.2e} of the array maxima')
    # the NDC vertices themselves: rendering from project_verts' output as NDC input gives the same image bit for bit
    ndc = project_verts(d['verts'].detach(), Rd.detach(), Td.detach(), Ks.detach())
    c = render_scene(ndc, d['faces'], d['fvu'], d['fmap'], d['maps'].detach(), d['table'], None, None, intrinsics(K), (48, 64),
                     1e-4, 10, z_clip=0.001, maps_are_texels4=True, verts_are_ndc=True)
    with torch.no_grad():
        a = render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], Rd, Td, intrinsics(K), (48, 64),
                         1e-4, 10, z_clip=0.001, maps_are_texels4=True)
    assert torch.equal(a, c.detach())


# ------------------------------------------------------------------------------------------------ the model and its steps
def _model_case(B=3):
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K = _model_inputs(dev, B=B)
    model.loss_weights = {'rgb': 1.0}
    Ks = _per_view_K(K, B, seed=1).float().to(dev)
    return model, dev, inp, Ks


def _scaled(Ks, scale):
    """Ks with fx, fy scaled per view (the principal point untouched)"""
    f = torch.stack([scale, scale, torch.ones_like(scale), torch.ones_like(scale)], -1)
    return Ks * torch.diag_embed(f) + Ks * (1 - torch.eye(4, device=Ks.device))


def _eager_focal(model, inp, Ks, scale):
    params = [p for p in model.parameters() if p.requires_grad]
    s = scale.detach().clone().requires_grad_(True)
    total = model(dict(inp, K=_scaled(Ks, s)))['total']
    *gp, gs = torch.autograd.grad(total, params + [s], allow_unused=True)
    return total.detach(), gs, torch.cat([(g if g is not None else torch.zeros_like(p)).reshape(-1) for g, p in zip(gp, params)])


def test_model_per_view_switch_equal_K_is_bit_identical():
    model, dev, inp, _ = _model_case()
    base = {k: v.detach() for k, v in model(inp).items()}
    model.set_per_view_intrinsics(True)
    per = {k: v.detach() for k, v in model(inp).items()}
    for k in base:
        assert torch.equal(base[k], per[k]), k
    model.eval()
    with torch.no_grad():
        a = model.predict(inp)
        model.set_per_view_intrinsics(False)
        assert torch.equal(a, model.predict(inp))


def test_model_renders_each_view_with_its_own_K():
    """a view's render depends on its own K only: per-view rendering equals the single-camera render of that view alone"""
    model, dev, inp, Ks = _model_case()
    model.eval()
    model.set_per_view_intrinsics(True)
    with torch.no_grad():
        rec = model.predict(dict(inp, K=Ks))
        for b in range(3):
            one = {'imgs': inp['imgs'][b:b + 1], 'R': inp['R'][b:b + 1], 'T': inp['T'][b:b + 1], 'K': Ks[b:b + 1]}
            assert torch.equal(rec[b:b + 1], model.predict(one)), b
        assert not torch.equal(rec, model.predict(inp))
        syn = model.predict_synthetic(dict(inp, K=Ks))
        assert syn.shape == inp['imgs'].shape


def test_focal_scale_gradient_eager_graphed_and_view_parallel():
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import BucketAdam
    from dbw_b200.parallel import ViewParallel
    model, dev, inp, Ks = _model_case()
    scale = (1 + 0.02 * torch.randn(3, generator=torch.Generator().manual_seed(9))).to(dev)
    total, gs, gp = _eager_focal(model, inp, Ks, scale)
    assert gs.abs().min() > 0, gs
    # K that requires grad takes the per-view path without the switch
    assert not model.per_view_intrinsics
    vp = ViewParallel(model, seed=5, max_pose_views=3, intrinsics=True)
    s = scale.clone().requires_grad_(True)
    vp.forward_backward(dict(inp, K=_scaled(Ks, s)))
    assert _rel(s.grad, gs) <= 1e-5, _rel(s.grad, gs)
    for opt in (None, BucketAdam):
        model2, _, _, _ = _model_case()
        vp2 = ViewParallel(model2, seed=5, max_pose_views=3, intrinsics=True)
        optimizer = opt([p for p in model2.parameters() if p.requires_grad], lr=0.0) if opt is not None else None
        s0 = scale.clone().requires_grad_(True)
        step = GraphedStep(vp2, dict(inp, K=_scaled(Ks, s0)), 3, warmup=1, optimizer=optimizer)
        s1 = scale.clone().requires_grad_(True)
        losses = step.run(dict(inp, K=_scaled(Ks, s1)))
        torch.cuda.synchronize()
        assert _rel(s1.grad, gs) <= 1e-5, (opt, _rel(s1.grad, gs))
        assert abs(losses['total'].item() - total.item()) <= 1e-6 * abs(total.item())
        with pytest.raises(RuntimeError, match='requires_grad'):
            step.run(dict(inp, K=_scaled(Ks, scale)))                    # K captured with grad, given without


def test_graphed_replay_renders_a_new_K():
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, dev, inp, Ks = _model_case()
    model.set_per_view_intrinsics(True)
    step = GraphedStep(ViewParallel(model, seed=5), dict(inp, K=Ks), 3, warmup=1)
    Ks2 = Ks.clone()
    Ks2[:, 0, 0] *= 1.03
    Ks2[:, 1, 2] -= 0.02
    got = step.run(dict(inp, K=Ks2))['total'].item()
    want = model(dict(inp, K=Ks2))['total'].item()
    first = model(dict(inp, K=Ks))['total'].item()
    assert abs(got - want) <= 1e-6 * abs(want) and abs(got - first) > 1e-5 * abs(first), (got, want, first)


def test_steps_refuse_intrinsics_gradients_they_were_not_built_for():
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, dev, inp, Ks = _model_case()
    Kg = Ks.clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match=r"inp\['K'\] requires grad"):
        ViewParallel(model, seed=5).forward_backward(dict(inp, K=Kg))
    with pytest.raises(RuntimeError, match='intrinsics=True'):
        GraphedStep(ViewParallel(model, seed=5, max_pose_views=3), dict(inp, K=Kg), 3, warmup=1)
    step = GraphedStep(ViewParallel(model, seed=5, max_pose_views=3, intrinsics=True), dict(inp, K=Ks), 3, warmup=1)
    with pytest.raises(RuntimeError):
        step.run(dict(inp, K=Kg))
    lit = model.renderer_light
    blocks = model.build_blocks(filter_transparent=False, as_scene=True)
    out = lit(blocks.extend(3), R=inp['R'], T=inp['T'], K=Kg)
    with pytest.raises(NotImplementedError):
        out.sum().backward()
