"""GPU: the built-in LPIPS term inside the model's objective.  `model(inp)` in training mode with
`PerceptualTerm(LPIPS)` installed against the oracle's restatement of src/model/dbw.py: the composite render
(oracle/dbw_path.py) plus the float64 LPIPS of oracle/lpips.py with the same dropout mask, weighted 0.1 x (1 while
coarse, 0.1 while fine) as at dbw.py:369-371.  Losses and leaf gradients."""
import pytest
import torch

from oracle import dbw_path as D
from oracle import lpips as OL
from tests.test_model_gpu import _inputs, _model_and_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('fine', [False, True])
def test_model_step_with_the_builtin_term(fine):
    from dbw_b200.dbw import PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    inp, imgs, R, T, K = _inputs(dev)
    sd = OL.random_state_dict(2)
    net = LPIPS.from_state_dict(sd)
    model.set_perceptual_loss(PerceptualTerm(net).to(dev))
    model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
    assert not model._fused_loss_ok(inp['imgs'])
    model.train()
    assert net.training                                       # the reference's LPIPSLoss follows model.train(): dropout on
    decim = 0 if fine else 8                                  # as in tests/test_model_gpu.py::test_predict_and_rgb_gradients
    keep = torch.sigmoid(p['alpha_logit'].detach()) > (0.5 if fine else 0.01)
    rec_ref = D.predict(tpl, p, R, T, K, (48, 64), sigma=5e-6 if fine else 1e-4, faces_per_pixel=10, z_clip=0.001, fine=fine,
                        keep=keep, decimate=decim)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)          # pixels whose top-K decisions differ
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    imgs_ref = torch.where(bad, rec_ref.detach(), imgs)

    net.seed.fill_(99)
    losses = model(inp, None)
    assert int(net.seed.item()) == 100
    factor = 0.1 * (0.1 if fine else 1.0)
    ref_p = factor * OL.lpips(sd, imgs_ref, rec_ref[:, :3], normalize=True, mode='tf32', seed=99).mean()
    ref_total = D.mse_loss(imgs_ref, rec_ref) + ref_p
    err_p = abs(losses['perceptual'].item() - ref_p.item()) / abs(ref_p.item())
    print(f'fine={fine}: perceptual {losses["perceptual"].item():.6e} vs {ref_p.item():.6e} (rel {err_p:.2e})')
    assert err_p < 1e-4                                      # the whole-term value bound of tests/test_lpips_gpu.py
    losses['total'].backward()
    ref_total.backward()
    n = 0
    for name, prm in model.named_parameters():
        if not prm.requires_grad:                            # the frozen LPIPS weights
            assert prm.grad is None and name.startswith('perceptual_loss.'), name
            continue
        g_ref = p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            continue
        rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        print(f'fine={fine} {name}: rel grad err {rel:.3e}')
        # the MSE part alone is within 2e-2 (tests/test_model_gpu.py); LPIPS's image gradient is within 3e-2 .. 4e-2 of
        # the emulated oracle at the whole-term shapes (TF32 conditioning, as large for cuDNN's own TF32 gradient).  Measured
        # here on an H100 80GB HBM3: up to 6.0e-2 (pose T, coarse) and 4.1e-2 (textures, fine); bound 1e-1.  A missing
        # LPIPS gradient or a wrong weight is checked by the value above and the texture-gradient difference below.
        assert rel < 1e-1, f'{name}: rel grad err {rel:.3e}'
        n += 1
    assert n >= 3
    # the term really reaches the leaves: without it the texture gradient differs
    g_with = model.textures.grad.clone()
    model.zero_grad(set_to_none=True)
    model.loss_weights = {'rgb': 1.0}
    model(inp, None)['total'].backward()
    assert (model.textures.grad - g_with).norm() > 1e-3 * g_with.norm()
