"""GPU: camera-pose gradients through the step objects -- parallel.ViewParallel(max_pose_views=N), graph.GraphedStep and
graph.PipelinedGraphedStep -- on one GPU.  Each must hand the caller's pose leaves the gradient the eager model(inp) step
gives them (1e-5 relative L2: the vertex gradients use atomics, so bits may differ), leave the parameter gradients as they
are without pose gradients, add only the two camera_grad_kernel launches, and refuse what it cannot do."""
import pytest
import torch

from oracle import dbw_path as D
from tests.test_camera_grad_gpu import (POSE_LR, POSE_STEPS, _axis_angle, _pose_inputs, _rotation_error_deg)
from tests.test_model_gpu import _inputs as _model_inputs, _model_and_oracle
from tests.test_raster_matrix_gpu import _rel

pytestmark = pytest.mark.gpu


def _close(a, b, what, rel=1e-5):
    assert b.abs().max() > 0, what
    err = ((a - b).norm() / b.norm()).item()
    assert err <= rel, f'{what}: rel L2 {err:.3e}'


def _eager(model, inp, dR, dT, R0, T0):
    """the reference: model(inp) with the poses computed from leaves; (g_dR, g_dT, parameter gradients in bucket order)"""
    params = [p for p in model.parameters() if p.requires_grad]
    a, b = dR.detach().clone().requires_grad_(True), dT.detach().clone().requires_grad_(True)
    total = model(dict(inp, R=R0 + a, T=T0 + b), None)['total']
    *gp, gR, gT = torch.autograd.grad(total, params + [a, b], allow_unused=True)
    flat = torch.cat([(g if g is not None else torch.zeros_like(p)).reshape(-1) for g, p in zip(gp, params)])
    return gR, gT, flat


def _case():
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K, dR, dT = _pose_inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    with torch.no_grad():
        dR.copy_(0.01 * torch.randn(dR.shape, generator=torch.Generator().manual_seed(3)).to(dev))
        dT.copy_(0.01 * torch.randn(dT.shape, generator=torch.Generator().manual_seed(4)).to(dev))
    return model, tpl, p, dev, inp, imgs, R, T, K, dR, dT


def test_view_parallel_pose_step_equals_the_eager_step_and_the_oracle():
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev, inp, imgs, R, T, K, dR, dT = _case()
    with torch.no_grad():
        dR.zero_(), dT.zero_()
    # the oracle's gradient, with the pixels whose kept faces differ between fp32 and fp64 taken out (test_camera_grad_gpu)
    keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.01
    Rl, Tl = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    rec_ref = D.predict(tpl, p, Rl, Tl, K, (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, keep=keep, decimate=8)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    ref = torch.autograd.grad(D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref), [Rl, Tl])
    R0, T0 = inp['R'], inp['T']
    gR, gT, gp = _eager(model, inp, dR, dT, R0, T0)
    for gather in (None, True):                       # autograd's own .grad tensors / the gathered bucket with its pose region
        vp = ViewParallel(model, seed=5, max_pose_views=len(imgs), gather_grads=gather)
        dR.grad = dT.grad = None
        vp.forward_backward(dict(inp, R=R0 + dR, T=T0 + dT))
        _close(dR.grad, gR, f'gather={gather} g_R')
        _close(dT.grad, gT, f'gather={gather} g_T')
        _close(vp.bucket.grads_flat(), gp, f'gather={gather} parameters')
        for g, r, what in zip((dR.grad, dT.grad), ref, ('R', 'T')):
            assert _rel(g.cpu().double(), r) < 1e-3, f'd/d{what} against the oracle: {_rel(g.cpu().double(), r):.3e}'


def test_graphed_pose_step_matches_eager_steps_and_recaptures_at_milestones():
    """three replays with different images and poses, the last after the coarse -> fine milestone (re-capture), each match
    their eager step; the caller's leaves accumulate; the parameter gradients equal a constant-pose graphed step's"""
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev, inp, imgs, R, T, K, dR, dT = _case()
    R0, T0 = inp['R'], inp['T']
    B = len(imgs)
    vp = ViewParallel(model, seed=5, max_pose_views=B)
    step = GraphedStep(vp, dict(inp, R=R0 + dR, T=T0 + dT), B)
    const = GraphedStep(vp, inp, B)
    assert step.pose is not None and const.pose is None
    g = torch.Generator().manual_seed(11)
    acc_R, acc_T = torch.zeros_like(dR), torch.zeros_like(dT)
    for it in range(3):
        if it == 2:
            model.set_cur_epoch(2000)                   # fine phase, textures no longer decimated: both steps re-capture
            with torch.no_grad():
                model.alpha_logit.copy_(torch.tensor([2., -2., 1., 3., -1.], device=dev))
        x = dict(inp, imgs=torch.rand(imgs.shape, generator=g).float().to(dev))
        with torch.no_grad():
            dR.add_(0.01 * torch.randn(dR.shape, generator=g).to(dev))
            dT.add_(0.01 * torch.randn(dT.shape, generator=g).to(dev))
        gR, gT, gp = _eager(model, x, dR, dT, R0, T0)
        step.run(dict(x, R=R0 + dR, T=T0 + dT))
        torch.cuda.synchronize()
        acc_R, acc_T = acc_R + gR, acc_T + gT
        _close(dR.grad, acc_R, f'replay {it} g_R (accumulated)')
        _close(dT.grad, acc_T, f'replay {it} g_T (accumulated)')
        _close(vp.bucket.grads_flat(), gp, f'replay {it} parameters')
        posed_params = vp.bucket.grads_flat().clone()
        const.run(dict(x, R=(R0 + dR).detach(), T=(T0 + dT).detach()))
        _close(posed_params, vp.bucket.grads_flat(), f'replay {it}: parameters against the constant-pose step')
    assert step.phase == const.phase == step._phase() and step.phase[1] is False


def test_pipelined_pose_step_reads_the_poses_when_it_consumes_them():
    """the poses of the prefetched step change (an optimiser step) between the prefetch and the replay that consumes it:
    the step renders from their value at consume time, and the images are still the prefetched ones"""
    from dbw_b200.graph import PipelinedGraphedStep
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev, inp, imgs, R, T, K, dR, dT = _case()
    B = len(imgs)
    Rp = inp['R'].clone().requires_grad_(True)                # the caller's pose parameter IS inp['R']
    vp = ViewParallel(model, seed=5, max_pose_views=B)
    pipe = PipelinedGraphedStep(vp, dict(inp, R=Rp), B)
    g = torch.Generator().manual_seed(12)
    first = dict(inp, R=Rp)
    second = dict(inp, imgs=torch.rand(imgs.shape, generator=g).float().to(dev), R=Rp)
    pipe.run(first, next_host_inp=second)
    torch.cuda.synchronize()
    g1 = Rp.grad.clone()
    with torch.no_grad():
        Rp.add_(0.02 * torch.randn(Rp.shape, generator=g).to(dev))
    gR, _, gp = _eager(model, second, torch.zeros_like(dR), torch.zeros_like(dT), Rp.detach(), inp['T'])
    pipe.run(second)
    torch.cuda.synchronize()
    _close(Rp.grad - g1, gR, 'g_R at consume time')
    _close(vp.bucket.grads_flat(), gp, 'parameters at consume time')


def test_pose_gradients_add_the_two_camera_kernels_to_a_captured_step():
    """a step captured with pose gradients launches camera_grad_kernel once per pass more than one without, and nothing else
    (counted while the steps are captured: warm-up + capture = 2 bodies each); one GPU: no collective at all"""
    from dbw_b200 import _lib
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev, inp, imgs, R, T, K, dR, dT = _case()
    B = len(imgs)
    vp = ViewParallel(model, seed=5, max_pose_views=B)
    posed = dict(inp, R=inp['R'] + dR, T=inp['T'] + dT)

    def count(x):
        torch.cuda.synchronize()
        n = _lib.launch_count()
        GraphedStep(vp, x, B, warmup=1)
        torch.cuda.synchronize()
        return _lib.launch_count() - n
    count(inp), count(posed)                                   # lazy state
    plain, with_pose, plain2 = count(inp), count(posed), count(inp)
    assert plain == plain2 and with_pose - plain == 2 * 2, (plain, with_pose, plain2)
    assert vp.bucket.peer is None and vp.sum_point is None


def test_pose_steps_refuse_too_many_views_and_a_changed_requires_grad():
    from dbw_b200 import _lib
    from dbw_b200.graph import GraphedStep, PipelinedGraphedStep
    from dbw_b200.parallel import ViewParallel
    model, tpl, p, dev, inp, imgs, R, T, K, dR, dT = _case()
    B = len(imgs)
    posed = dict(inp, R=inp['R'] + dR, T=inp['T'] + dT)
    small = ViewParallel(model, seed=5, max_pose_views=B - 1)
    n = _lib.launch_count()
    for make in (lambda: small.forward_backward(posed), lambda: GraphedStep(small, posed, B),
                 lambda: PipelinedGraphedStep(small, posed, B)):
        with pytest.raises(ValueError, match=f'max_pose_views={B - 1}'):
            make()
    assert _lib.launch_count() == n                            # refused before any work
    vp = ViewParallel(model, seed=5, max_pose_views=B)
    step = GraphedStep(vp, posed, B)
    with pytest.raises(RuntimeError, match='do not'):
        step.run(inp)                                           # captured with pose gradients, run without
    const = GraphedStep(vp, inp, B)
    with pytest.raises(RuntimeError, match='require grad'):
        const.run(dict(inp, R=inp['R'] + dR, T=inp['T'] + dT))  # captured without, run with
    assert dR.grad is None and dT.grad is None


def test_pose_recovery_through_a_graphed_step():
    """test_camera_grad_gpu.test_pose_recovery_from_perturbed_cameras with every step a GraphedStep replay: the same scene,
    targets, perturbation, optimiser and bounds (a quarter of the initial rotation and translation errors)"""
    from copy import deepcopy
    from dbw_b200 import geometry as G
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from tests.test_model_gpu import CFG
    dev = torch.device('cuda:0')
    torch.manual_seed(5)
    model = DifferentiableBlocksWorld((96, 128), **deepcopy(CFG)).to(dev).eval()      # eval: no texture decimation
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for t in (model.textures, model.texture_bkg, model.texture_ground):
            low = 3 * torch.randn(t.shape[0], 3, 4, 4, generator=g)
            t.copy_(torch.nn.functional.interpolate(low, size=t.shape[1:3], mode='bilinear', align_corners=True).permute(0, 2, 3, 1))
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

    R, T = pose()
    step = GraphedStep(ViewParallel(model, seed=5, max_pose_views=4), dict(inp, R=R, T=T), 4)
    e0 = errors()
    for it in range(POSE_STEPS):
        opt.zero_grad(set_to_none=True)
        R, T = pose()
        losses = step.run({'R': R, 'T': T})
        opt.step()
        sched.step()
        if it % 50 == 0 or it == POSE_STEPS - 1:
            e = errors()
            print(f'step {it}: loss {losses["total"].item():.4e}, rotation {e[0]:.3f} deg, translation {e[1]:.4f}')
    e1 = errors()
    print(f'initial errors {e0[0]:.3f} deg / {e0[1]:.4f}, final {e1[0]:.3f} deg / {e1[1]:.4f}')
    assert e1[0] < e0[0] / 4 and e1[1] < e0[1] / 4
