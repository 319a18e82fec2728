"""GPU: the image-score kernel (csrc/dbw_metrics.cu, dbw_b200.metrics) against the float64 oracle (oracle/image_scores.py)
and the reference's own float32 scores (tests/golden/image_scores.npz), and `quantitative_eval` against a restatement of the
reference's loop (src/model/dbw.py:464-493) that renders through forward(viz_purpose=True) and scores with the oracle."""
import math

import numpy as np
import pytest
import torch

from oracle import image_scores as O
from tests.golden.make_image_scores_golden import CASES, pairs
from tests.test_image_scores_host import GOLDEN, NEAR_CONSTANT

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
SSIM_ATOL, SE_RTOL = 1e-5, 1e-6


def _pair(B, H, W, seed, correlated):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, H, W, generator=g)
    y = (x + 0.1 * (torch.rand(B, 3, H, W, generator=g) - 0.5)).clamp(0, 1) if correlated else torch.rand(B, 3, H, W, generator=g)
    return x, y


# 11x11 (one output pixel per channel), odd sizes, outputs of exactly one 32 x 32 tile and of one pixel more, sizes that are
# not a multiple of the tile, and the evaluation's 300x400, 400x400 and 576x768
SIZES = [(1, 11, 11), (8, 11, 11), (3, 13, 17), (2, 42, 42), (5, 43, 43), (4, 75, 107), (7, 97, 61), (6, 41, 300),
         (2, 300, 400), (1, 400, 400), (4, 400, 400), (4, 576, 768), (1, 576, 768)]


@pytest.mark.parametrize('correlated', [False, True])
@pytest.mark.parametrize('B,H,W', SIZES)
def test_kernel_matches_the_float64_oracle(B, H, W, correlated):
    from dbw_b200 import metrics
    x, y = _pair(B, H, W, 100 * B + H + W, correlated)
    se, ss = metrics.image_scores(x.to(DEV), y.to(DEV))
    want_ss, want_se = O.ssim(x, y), O.se_sum(x, y)
    err_ss = (ss.cpu().double() - want_ss).abs().max().item()
    err_se = ((se.cpu().double() - want_se).abs() / want_se).max().item()
    print(f'{B}x{H}x{W} correlated={correlated}: |ssim - oracle| {err_ss:.2e}, se_sum rel {err_se:.2e}')
    assert err_ss <= SSIM_ATOL and err_se <= SE_RTOL, (err_ss, err_se)
    # the module's other entry points are the same numbers
    assert torch.equal(metrics.ssim(x.to(DEV), y.to(DEV)), ss)
    assert abs(metrics.psnr(x.to(DEV), y.to(DEV)).item() - O.psnr(x, y).item()) <= 1e-5


def test_two_calls_give_the_same_bits():
    from dbw_b200 import metrics
    x, y = (t.to(DEV) for t in _pair(4, 576, 768, 3, True))
    a, b = metrics.image_scores(x, y), metrics.image_scores(x, y)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_non_contiguous_render_slices_are_scored_like_copies():
    from dbw_b200 import metrics
    x, y4 = _pair(3, 40, 48, 5, False)[0].to(DEV), torch.rand(3, 4, 40, 48, device=DEV)
    got = metrics.image_scores(x, y4[:, :3])
    want = metrics.image_scores(x, y4[:, :3].contiguous())
    assert all(torch.equal(u, v) for u, v in zip(got, want))


def test_float64_and_mixed_devices_raise():
    from dbw_b200 import metrics
    from dbw_b200._lib import DbwError
    a = torch.rand(1, 3, 16, 16, device=DEV)
    with pytest.raises(DbwError, match='float32'):
        metrics.image_scores(a.double(), a.double())
    with pytest.raises(DbwError, match='CUDA'):
        metrics.image_scores(a, a.cpu())


@pytest.mark.parametrize('name', list(CASES))
def test_kernel_reproduces_the_references_own_scores(name):
    """within 1e-5 of the reference's float32 per-image SSIM; on near-constant pairs the reference's own float32 rounding
    is 1e-4 from the exact value (tests/test_image_scores_host.py), and that is the bound there"""
    from dbw_b200 import metrics
    x, y = pairs(name)
    se, ss = metrics.image_scores(x.to(DEV), y.to(DEV))
    ref = 1 - GOLDEN[f'{name}/ssim_loss'].astype(np.float64)
    err = np.abs(ss.cpu().double().numpy() - ref).max()
    print(f'{name}: |ssim - reference| {err:.2e}')
    assert err <= (2e-4 if name in NEAR_CONSTANT else 1e-5), err
    if name.startswith('same'):
        assert (ss == 1).all() and (se == 0).all()
    ref_psnr = float(GOLDEN[f'{name}/psnr'][0])
    got = metrics.psnr_of(se, x[0].numel()).item()
    assert got == ref_psnr if math.isinf(ref_psnr) else abs(got - ref_psnr) <= 1e-5


# ------------------------------------------------------------------------------------------------ quantitative_eval
def _reference_loop(model, loader, device, perceptual):
    """dbw.py:464-493 over the same loader: the pooled 4x render, AverageMeters weighted by N, mse2psnr of each batch's
    MSE, 1 - mean(SSIMLoss) per batch; the scores from the float64 oracle"""
    model.eval()
    scene = model.build_scene(filter_transparent=True)
    sums, count = dict(L_tot=0.0, L_rec=0.0, PSNR=0.0, SSIM=0.0, LPIPS=0.0), 0
    with torch.no_grad():
        for inp, _ in loader:
            inp = {k: v.to(device) for k, v in inp.items()}
            imgs, n = inp['imgs'], len(inp['imgs'])
            rec = model.renderer(scene.extend(n), inp['R'], inp['T'], viz_purpose=True, K=model._view_K(inp))[:, :3]
            losses = model.compute_losses(imgs, rec)
            sums['L_tot'] += losses['total'].item() * n
            sums['L_rec'] += sum(losses[k] for k in ('rgb', 'perceptual') if k in losses).item() * n
            sums['PSNR'] += O.psnr(imgs.cpu(), rec.cpu()).item() * n
            sums['SSIM'] += (1 - (1 - O.ssim(imgs.cpu(), rec.cpu())).mean()).item() * n
            sums['LPIPS'] += (perceptual(imgs, rec).item() if perceptual is not None else float('nan')) * n
            count += n
    return {k: v / count for k, v in sums.items()}


def _loader(B=6, split=(4, 2)):
    from tests.test_model_gpu import _inputs
    inp, *_ = _inputs(DEV, B=B)
    out, i = [], 0
    for n in split:
        out.append(({k: v[i:i + n].cpu() for k, v in inp.items()}, {}))
        i += n
    return out


@pytest.mark.parametrize('term', ['none', 'lpips', 'vgg'])
def test_quantitative_eval_equals_the_references_loop(term):
    from tests.test_model_gpu import _model_and_oracle
    model, *_ = _model_and_oracle(fine=True)
    perceptual = None
    if term == 'lpips':
        from dbw_b200.dbw import PerceptualTerm
        from dbw_b200.perceptual import LPIPS
        from oracle import lpips as OL
        model.set_perceptual_loss(PerceptualTerm(LPIPS.from_state_dict(OL.random_state_dict(2))).to(DEV))
        model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
        perceptual = model.perceptual_loss
    elif term == 'vgg':
        from tests.test_vgg_perceptual_gpu import _model
        model, *_ = _model(True)
    loader = _loader()
    got = model.quantitative_eval(loader, DEV, hard_inference=True)
    want = _reference_loop(model, loader, DEV, perceptual)
    assert list(got)[:6] == ['n_blocks', 'L_tot', 'L_rec', 'PSNR', 'SSIM', 'LPIPS'] and list(got)[6:] == [f'alpha{k}' for k in range(5)]
    opac = model.get_opacities()
    assert got['n_blocks'] == int((opac > 0.5).sum()) and [got[f'alpha{k}'] for k in range(5)] == opac.tolist()
    print(term, {k: (got[k], want[k]) for k in want})
    for k in ('L_tot', 'L_rec'):
        assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]), k
    assert abs(got['PSNR'] - want['PSNR']) <= 1e-5 and abs(got['SSIM'] - want['SSIM']) <= 1e-5
    if term == 'lpips':
        assert abs(got['LPIPS'] - want['LPIPS']) <= 1e-6 * abs(want['LPIPS'])
    else:
        assert math.isnan(got['LPIPS']) and math.isnan(want['LPIPS'])
