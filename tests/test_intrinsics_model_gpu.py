"""GPU: the scene model's training paths with a distinct K per view, against the float64 oracle, and with equal K against the
single-camera path.

The reference (oracle.dbw_path.predict / predict_joint) takes one K per call, so the per-view reference renders one view at a
time with its own K[b] and concatenates: the rendered image, the MSE over the whole batch, and by autograd the gradients of the
leaf parameters, of R, T and of the four entries of K that the projection reads.  Every render path of the model's forward():

  fused_loss      decoupled scene, both passes and the MSE in the loss epilogue (dbw_render_forward_loss_grad +
                  dbw_render_backward_deferred for the blocks pass, from per-view NDC vertices)
  composite       the same scene kernels, the two passes rendered separately and composited (fused_loss off)
  eager_static    the eager PyTorch scene construction with static topology (fused_scene off)
  eager_meshes    the reference-shaped Meshes, filtered blocks sliced away (static_topology off)
  joint           environment and blocks as one scene (decouple_rendering off)

Tolerances are those of tests/test_model_gpu.py: pixels where fp32 takes another discrete decision than fp64 (colour off by
more than 1e-4, under 0.1 %) get each side's own reconstruction as target; the loss agrees to 1e-5, every gradient to 1e-3
relative L2."""
import pytest
import torch

from oracle import dbw_path as D
from tests.test_intrinsics_gpu import _per_view_K
from tests.test_model_gpu import _inputs as _model_inputs, _model_and_oracle
from tests.test_raster_matrix_gpu import _rel

pytestmark = pytest.mark.gpu

PATHS = {'fused_loss': {}, 'composite': {'fused_loss': False}, 'eager_static': {'fused_scene': False},
         'eager_meshes': {'fused_scene': False, 'static_topology': False}, 'joint': {'decouple_rendering': False}}
SAME_RESULTS = 1e-6          # gradients of two summation orders: of each array's largest magnitude
FOUR = ((0, 0), (1, 1), (0, 2), (1, 2))


def _model(path):
    model, tpl, p, dev = _model_and_oracle()
    for k, v in PATHS[path].items():
        setattr(model, k, v)
    model.loss_weights = {'rgb': 1.0}
    return model, tpl, p, dev


def _oracle_rec(tpl, p, R, T, Ks, joint, keep):
    """float64 reconstruction of each view with its own K[b] (coarse phase: 8x decimated textures, opacities)"""
    f = D.predict_joint if joint else D.predict
    return torch.cat([f(tpl, p, R[b:b + 1], T[b:b + 1], Ks[b], (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, keep=keep,
                        decimate=8) for b in range(R.shape[0])])


@pytest.mark.parametrize('path', list(PATHS))
def test_model_path_with_per_view_K_matches_oracle(path):
    model, tpl, p, dev = _model(path)
    inp, imgs, R, T, K = _model_inputs(dev)
    Ks = _per_view_K(K, 3, seed=3)
    keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.01                  # kill_blocks
    Rl, Tl, Kl = (t.clone().requires_grad_(True) for t in (R, T, Ks))
    rec_ref = _oracle_rec(tpl, p, Rl, Tl, Kl, path == 'joint', keep)
    model.set_per_view_intrinsics(True)
    with torch.no_grad():
        rec = model.predict(dict(inp, K=Ks.float().to(dev))).detach().cpu().double()
    err = (rec - rec_ref.detach()).abs()
    bad = (err > 1e-4).any(1, keepdim=True)
    print(f'\n{path}: decision-masked pixels {bad.double().mean().item() * 100:.4f}%, max err elsewhere '
          f'{(err * ~bad).max().item():.3e}')
    assert bad.double().mean().item() < 1e-3
    # the switch off: a K that requires grad renders per view by itself
    model.set_per_view_intrinsics(False)
    Rd, Td, Kd = (t.detach().float().to(dev).requires_grad_(True) for t in (R, T, Ks))
    losses = model(dict(inp, imgs=torch.where(bad, rec, imgs).float().to(dev), R=Rd, T=Td, K=Kd), None)
    loss_ref = D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref)
    assert abs(losses['rgb'].item() - loss_ref.item()) < 1e-5 * max(1.0, abs(loss_ref.item())), (losses['rgb'].item(), loss_ref.item())
    losses['total'].backward()
    loss_ref.backward()
    for name, prm in model.named_parameters():
        g_ref = p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            assert prm.grad is None or prm.grad.abs().max().item() < 1e-12, name
            continue
        rel = _rel(prm.grad.cpu().double(), g_ref)
        assert rel < 1e-3, f'{path} {name}: rel grad err {rel:.3e}'
    pick = lambda g: torch.stack([g[:, i, j] for i, j in FOUR], -1)
    for name, g, g_ref in (('R', Rd.grad, Rl.grad), ('T', Td.grad, Tl.grad), ('K', pick(Kd.grad), pick(Kl.grad))):
        rel = _rel(g.cpu().double(), g_ref)
        print(f'{path}: d loss / d{name} rel err {rel:.3e}')
        assert g_ref.abs().max() > 0 and rel < 1e-3, f'{path} {name}: rel grad err {rel:.3e}'
    assert pick(Kd.grad).abs().min() > 0, f'{path}: an intrinsic got no gradient'
    # the product reads only those four entries of each K
    rest = Kd.grad.clone()
    for i, j in FOUR:
        rest[:, i, j] = 0
    assert rest.abs().max() == 0


@pytest.mark.parametrize('path', list(PATHS))
def test_equal_K_model_step_equals_the_single_camera_step(path):
    """every view's K = K[0] with per-view intrinsics on: the same loss (bit for bit on the fused-loss path, whose sum has a
    fixed order), the same leaf and pose gradients up to the atomics' summation order"""
    model, tpl, p, dev = _model(path)
    inp, *_ = _model_inputs(dev)
    params = [q for q in model.parameters() if q.requires_grad]
    runs = []
    for per_view in (False, True):
        model.set_per_view_intrinsics(per_view)
        Rd, Td = (inp[k].detach().clone().requires_grad_(True) for k in ('R', 'T'))
        total = model(dict(inp, R=Rd, T=Td), None)['total']
        grads = torch.autograd.grad(total, params + [Rd, Td], allow_unused=True)
        runs.append((total.detach(), [g if g is not None else torch.zeros_like(q) for g, q in zip(grads, params + [Rd, Td])]))
    (l0, g0), (l1, g1) = runs
    if path == 'fused_loss':
        assert torch.equal(l0, l1)
    else:
        assert (l0 - l1).abs().item() <= 1e-6 * l0.abs().item()
    worst = 0.0
    for name, a, b in zip([n for n, q in model.named_parameters() if q.requires_grad] + ['R', 'T'], g1, g0):
        if b.abs().max() == 0:
            assert a.abs().max() == 0, name
            continue
        err = (a - b).abs().max().item() / b.abs().max().item()
        worst = max(worst, err)
        assert err <= SAME_RESULTS, (path, name, err)
    print(f'\n{path}: equal K, largest gradient difference {worst:.2e} of the array maxima')
