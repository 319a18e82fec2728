"""GPU: the VGG16 feature-reconstruction loss (perceptual.PerceptualLoss on dbw_vgg_loss_* of csrc/dbw_lpips.cu) against the
float64 restatement of tests/_vgg_oracle.py and the reference's own forward frozen in tests/golden/vgg_perceptual.npz; the
LPIPS kernels it shares still give the bits of the build before it (tests/golden/lpips_bits.npz); and the term inside the
model's eager, graph-captured and view-parallel steps."""
import json
import math
import os

import numpy as np
import pytest
import torch

from tests import _vgg_oracle as OV

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# the whole-term bounds of tests/test_lpips_gpu.py: value (max relative) and gradient (relative L2), against the
# TF32-emulated oracle and against exact float64
TOL = dict(tf32=dict(value=1e-4, grad=6e-2), exact=dict(value=1e-2, grad=1e-1))
# images whose deepest requested level is a few pixels (2x17x23 at relu3_3 is 4x5; the smallest legal images are 1x1 there)
# average the TF32 roundings that an fp32 ulp flips over too few terms for 1e-4: measured on an H100 80GB HBM3 at 700 W,
# up to 1.2e-3 (value) and 1.5e-2 (gradient) against the emulated oracle.  These shapes take the per-tap bounds of
# tests/test_lpips_gpu.py (2e-3, 1.5e-1), which cover the same regime; against exact float64 the whole-term bounds hold.
TOL_FEW_PIXELS = dict(tf32=dict(value=2e-3, grad=1.5e-1), exact=TOL['exact'])


@pytest.fixture(scope='module')
def sd():
    return OV.random_state_dict(0)


def _module(sd, **kw):
    from dbw_b200.perceptual import PerceptualLoss
    return PerceptualLoss.from_state_dict(sd, **kw).to(DEV)


def _images(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g)
    return a, (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)


def _run(m, a, b, grad_value):
    x = b.to(DEV).requires_grad_(True)
    v = m.per_image(a.to(DEV), x)
    (v * grad_value.to(DEV)).sum().backward()
    return v.detach().cpu().double(), x.grad.cpu().double()


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _check(m, sd, o, a, b, gv, what, tol=TOL):
    v, g = _run(m, a, b, gv)
    assert torch.isfinite(v).all() and torch.isfinite(g).all(), what
    for mode in ('tf32', 'exact'):
        wv, wg = OV.value_and_grad(sd, a.to(DEV), b.to(DEV), **o, mode=mode, grad_value=gv.to(DEV))
        wv, wg = wv.cpu(), wg.cpu()
        ev, eg = float(((v - wv).abs() / wv.abs()).max()), _rel(g, wg)
        print(f'{what} {mode}: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
        assert ev < tol[mode]['value'] and eg < tol[mode]['grad'], (what, mode, ev, eg)


def _min_size(o):
    return 2 ** (max(o['levels']) - 1)


SHAPES = [(1, 300, 400), (4, 300, 400), (2, 64, 96), (2, 17, 23), 'min3', 'min5']


@pytest.mark.parametrize('shape', SHAPES, ids=[s if isinstance(s, str) else 'x'.join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize('name', list(OV.OPTION_SETS))
def test_whole_term_against_oracle(sd, name, shape):
    kw = OV.OPTION_SETS[name]
    o = OV.options(**kw)
    if isinstance(shape, str):                      # the smallest legal image for the deepest level 3, or 5
        deepest = int(shape[-1])
        if max(o['levels']) > deepest:
            pytest.skip('the option set needs a larger image')
        if deepest == 5:
            o = dict(o, levels=tuple(sorted(set(o['levels']) | {5})))
            kw = dict(kw, feature_levels=list(o['levels']))
        s = _min_size(dict(o, levels=(deepest,)))
        shape = (2, s, s + 1)
    B, H, W = shape
    a, b = _images(B, H, W, H + W + B)
    few = (H >> (max(o['levels']) - 1)) * (W >> (max(o['levels']) - 1)) < 64
    _check(_module(sd, **kw), sd, o, a, b, torch.linspace(0.5, 1.5, B), f'{name} {B}x{H}x{W}', TOL_FEW_PIXELS if few else TOL)


@pytest.mark.parametrize('shape', [0, 1])
@pytest.mark.parametrize('name', list(OV.OPTION_SETS))
def test_against_the_references_forward(name, shape):
    z = np.load(os.path.join(GOLDEN, 'vgg_perceptual.npz'))
    sd = OV.random_state_dict(json.loads(str(z['meta']))['weight_seed'])
    a, b = (torch.from_numpy(z[f's{shape}__{k}']) for k in ('imgs', 'rec'))
    m = _module(sd, **OV.OPTION_SETS[name])
    x = b.to(DEV).requires_grad_(True)
    v = m(a.to(DEV), x)
    assert v.dim() == 0
    v.backward()
    want_v, want_g = float(z[f's{shape}__{name}__value']), torch.from_numpy(z[f's{shape}__{name}__grad']).double()
    ev, eg = abs(v.item() - want_v) / abs(want_v), _rel(x.grad.cpu().double(), want_g)
    print(f'{name} shape {shape}: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
    assert ev < TOL['exact']['value'] and eg < TOL['exact']['grad']


@pytest.mark.parametrize('normalize_features', [True, False])
@pytest.mark.parametrize('level', [1, 2, 3, 4, 5])
def test_each_level_alone_against_oracle(sd, level, normalize_features):
    """one level at a time: a wrong head or a missing level cannot hide inside the sum.  The bounds of
    tests/test_lpips_gpu.py's per-tap check (a deep level alone averages over few pixels after up to 12 TF32 layers)"""
    o = OV.options(feature_levels=[level], normalize_features=normalize_features)
    a, b = _images(2, 64, 96, 31 + level)
    m = _module(sd, feature_levels=[level], normalize_features=normalize_features)
    v, g = _run(m, a, b, torch.tensor([0.7, 1.3]))
    wv, wg = OV.value_and_grad(sd, a.to(DEV), b.to(DEV), **o, mode='tf32', grad_value=torch.tensor([0.7, 1.3], device=DEV))
    ev, eg = float(((v - wv.cpu()).abs() / wv.cpu().abs()).max()), _rel(g, wg.cpu())
    print(f'level {level} normalize_features={normalize_features}: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
    assert ev < 2e-3 and eg < 1.5e-1, (level, ev, eg)


def test_value_bits_repeat_and_black_images_stay_finite(sd):
    a, b = _images(3, 75, 101, 3)
    for kw in ({}, dict(feature_levels=[1, 2, 3, 4, 5], sum_channels=True), dict(normalize_features=False, normalize_input=False)):
        m = _module(sd, **kw)
        with torch.no_grad():
            v0, v1 = m.per_image(a.to(DEV), b.to(DEV)), m.per_image(a.to(DEV), b.to(DEV))
        v2, _ = _run(m, a, b, torch.ones(3))
        assert torch.equal(v0, v1) and torch.equal(v0.cpu().double(), v2), kw     # with or without the saved activations
        # all-black images: with normalize_input=False every feature vector is relu(bias) or zero; with the ImageNet
        # transform a constant image; either way the forward and backward leave no NaN or Inf
        z = torch.zeros(2, 3, 32, 48)
        v, g = _run(m, z, z, torch.ones(2))
        assert torch.isfinite(v).all() and torch.isfinite(g).all(), kw


def test_all_zero_features_are_finite(sd):
    """zero weights and biases: every feature vector is 0, so the normalisation divides 0 by 1e-10 and its gradient term
    is dropped (as the oracle's _SafeSqrt does)"""
    zero = {k: (torch.zeros_like(v) if k.startswith('slice') else v) for k, v in sd.items()}
    m = _module(zero, feature_levels=[1, 3])
    a, b = _images(2, 32, 40, 8)
    v, g = _run(m, a, b, torch.ones(2))
    assert torch.equal(v, torch.zeros(2, dtype=torch.float64)) and torch.equal(g, torch.zeros_like(g))


def test_lpips_is_unchanged_bit_for_bit():
    """perceptual.LPIPS on the inputs of tests/golden/make_lpips_bits_golden.py gives the values and gradients the build
    before the VGG feature loss gave, bit for bit"""
    from tests.golden.make_lpips_bits_golden import CASES, lpips_bits
    z = np.load(os.path.join(GOLDEN, 'lpips_bits.npz'))
    got = lpips_bits()
    assert len(got) == 2 * len(CASES)
    for k, v in got.items():
        assert np.array_equal(v.view(np.uint32), z[k].view(np.uint32)), k


def test_weight_changes_re_prepare(sd):
    m = _module(sd)
    a, b = _images(1, 32, 32, 4)
    with torch.no_grad():
        v0 = m(a.to(DEV), b.to(DEV))
        getattr(m.slice2, '5').weight.mul_(0.5)
        v1 = m(a.to(DEV), b.to(DEV))
        want = _module(dict(m.state_dict()))(a.to(DEV), b.to(DEV))
    assert not torch.equal(v0, v1) and torch.equal(v1, want)


# ------------------------------------------------------------------------------------------------ model paths
def _model(fine):
    from tests.test_model_gpu import _model_and_oracle
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    sd = OV.random_state_dict(2)
    model.set_perceptual_loss(_module(sd))
    model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
    model.train()
    return model, tpl, p, sd


@pytest.mark.parametrize('fine', [False, True])
def test_model_step_with_the_term(fine):
    from oracle import dbw_path as D
    from tests.test_model_gpu import _inputs
    model, tpl, p, sd = _model(fine)
    dev = model.alpha_logit.device
    inp, imgs, R, T, K = _inputs(dev)
    assert not model._fused_loss_ok(inp['imgs'])
    decim = 0 if fine else 8
    keep = torch.sigmoid(p['alpha_logit'].detach()) > (0.5 if fine else 0.01)
    rec_ref = D.predict(tpl, p, R, T, K, (48, 64), sigma=5e-6 if fine else 1e-4, faces_per_pixel=10, z_clip=0.001, fine=fine,
                        keep=keep, decimate=decim)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)           # pixels whose top-K decisions differ
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    imgs_ref = torch.where(bad, rec_ref.detach(), imgs)
    losses = model(inp, None)
    factor = 0.1 * (0.1 if fine else 1.0)
    ref_p = factor * OV.vgg_perceptual(sd, imgs_ref, rec_ref[:, :3], mode='tf32').mean()
    err_p = abs(losses['perceptual'].item() - ref_p.item()) / abs(ref_p.item())
    print(f'fine={fine}: perceptual {losses["perceptual"].item():.6e} vs {ref_p.item():.6e} (rel {err_p:.2e})')
    assert err_p < 1e-4
    (D.mse_loss(imgs_ref, rec_ref) + ref_p).backward()
    losses['total'].backward()
    n = 0
    for name, prm in model.named_parameters():
        if not prm.requires_grad:
            assert prm.grad is None and name.startswith('perceptual_loss.'), name
            continue
        g_ref = p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            continue
        rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        print(f'fine={fine} {name}: rel grad err {rel:.3e}')
        assert rel < 1e-1, f'{name}: rel grad err {rel:.3e}'                # the bound of tests/test_lpips_model_gpu.py
        n += 1
    assert n >= 3
    g_with = model.textures.grad.clone()
    model.zero_grad(set_to_none=True)
    model.loss_weights = {'rgb': 1.0}
    model(inp, None)['total'].backward()
    # the term reaches the leaves: 0.01 x the term is 7e-4 of the texture gradient in the fine phase, 1e-5 the renderer's
    # run-to-run spread
    assert (model.textures.grad - g_with).norm() > 1e-4 * g_with.norm()


def test_graphed_and_view_parallel_steps_equal_the_eager_step():
    """a GraphedStep replay and a ViewParallel step give the eager step's perceptual loss bit for bit (the renders are the
    same and the term's reduction is fixed), and its other losses and gradients up to the renderer's atomics: the RGB loss
    is summed with one atomicAdd per CTA (composite_mse_kernel), so its last bits follow the CTAs' order.  The graph is
    captured first, as in tests/test_model_gpu.py: gradients an eager step left on the default stream cannot be
    accumulated into inside a capture"""
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from tests.test_model_gpu import _inputs
    model, *_ = _model(False)
    model.opacity_noise = False                       # every step then renders the same images
    inp, *_ = _inputs(model.alpha_logit.device)
    vp = ViewParallel(model, seed=5)
    graphed = GraphedStep(vp, inp, len(inp['imgs']))
    replay = {k: v.detach().clone() for k, v in graphed.run().items()}
    g_graph = vp.bucket.grads_flat().clone()
    model.zero_grad(set_to_none=False)
    step = vp.forward_backward(inp)
    torch.cuda.synchronize()
    g_step = vp.bucket.grads_flat().clone()
    for q in model.parameters():
        q.grad = None
    eager = model(inp, None)
    eager['total'].backward()
    g_eager = torch.cat([q.grad.flatten() for q in model.parameters() if q.requires_grad])
    for got in (replay, step):
        assert torch.equal(got['perceptual'].detach(), eager['perceptual'].detach())
        for k in ('rgb', 'total'):
            assert abs(got[k].item() - eager[k].item()) <= 1e-6 * abs(eager[k].item()), k
    for g in (g_graph, g_step):
        assert (g - g_eager).norm() <= 1e-4 * g_eager.norm()


def test_quantitative_eval_reports_no_lpips_with_this_term():
    from tests.test_model_gpu import _inputs
    model, *_ = _model(True)
    inp, *_ = _inputs(model.alpha_logit.device, B=4)
    loader = [({k: v[:2].cpu() for k, v in inp.items()}, {}), ({k: v[2:].cpu() for k, v in inp.items()}, {})]
    scores = model.quantitative_eval(loader, model.alpha_logit.device, hard_inference=True)
    assert math.isnan(scores['LPIPS']) and scores['L_rec'] > 0
