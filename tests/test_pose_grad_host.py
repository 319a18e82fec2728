"""CPU: camera-pose gradients through the data-parallel step (parallel.ViewParallel(max_pose_views=N)).

A toy model with the ViewParallel contract renders each pixel as a torch function of its scene parameters and of the view's
R and T, and routes what it differentiates through the gradient-sum point the way DifferentiableBlocksWorld does.  Two gloo
ranks, whole-view and row-band sharding, the sum at the leaves (the pose region of the bucket, summed by the same all-reduce
as the parameter gradients) and at the scene tensors (the pose leaves ride through the one GradSumPoint exchange): the pose
gradient reaching the caller's leaves is the single-process gradient of the same step, bit-identical on both ranks."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_host_logic import _GlooBucket

B, H, W = 5, 48, 5
MAX_POSE_VIEWS = 8
CONFIGS = [(row_bands, reduce_at) for row_bands in (False, True) for reduce_at in ('leaf', 'scene')]


class _ToyPosed(torch.nn.Module):
    """scene tensors = f(leaves) -> [gradient-sum point] -> per-pixel 'render' of the view's R, T -> MSE, plus a
    view-independent regulariser; honours inp['rows'] the way the kernels do (dbw_render.h view_rows)"""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.linspace(0.1, 0.9, W))
        self.textures = torch.nn.Parameter(torch.linspace(-1, 1, 6))
        self.n_total_views, self.noise_generator, self.grad_sum_point = None, None, None

    def _fused_loss_ok(self, imgs):
        return True

    def can_sum_gradients_at_scene_tensors(self, imgs):
        return True

    def grad_sum_floats(self):
        return W + 3

    def forward(self, inp, labels=None):
        verts, cells = self.w.exp(), torch.sigmoid(self.textures).view(3, 2).mean(1)
        R, T = inp['R'], inp['T']
        if self.grad_sum_point is not None:
            verts, cells = self.grad_sum_point(verts, cells)
            R, T = self.grad_sum_point.cameras(inp)
        imgs = inp['imgs']
        y = torch.arange(H, dtype=imgs.dtype)[None, :, None] / H
        cam = (R * torch.linspace(-1, 1, 9).view(3, 3)).sum((1, 2))[:, None, None] + (T * cells).sum(1)[:, None, None] * y
        err = (imgs * verts[None, None] + torch.sin(cam) * cells.sum() - 0.5) ** 2
        if inp.get('rows') is not None:
            yi = torch.arange(H)[None, :, None]
            err = err * ((yi >= inp['rows'][:, 0, None, None]) & (yi < inp['rows'][:, 1, None, None]))
        rgb = err.sum() / (self.n_total_views * H * W)
        reg = self.textures.pow(2).sum() + self.w.sum()
        return {'rgb': rgb, 'tv': reg, 'total': rgb + reg}


def _data():
    g = torch.Generator().manual_seed(1)
    imgs, R0, T0 = torch.rand(B, H, W, generator=g), torch.rand(B, 3, 3, generator=g), torch.rand(B, 3, generator=g)
    dR = (0.1 * torch.randn(B, 3, 3, generator=g)).requires_grad_(True)
    dT = (0.1 * torch.randn(B, 3, generator=g)).requires_grad_(True)
    return imgs, R0, T0, dR, dT


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from dbw_b200.parallel import ViewParallel
    for row_bands, reduce_at in CONFIGS:
        torch.manual_seed(0)
        model = _ToyPosed()
        vp = ViewParallel(model, seed=123, row_bands=row_bands, reduce_at=reduce_at, max_pose_views=MAX_POSE_VIEWS,
                          peer_factory=_GlooBucket if reduce_at == 'scene' else None)
        imgs, R0, T0, dR, dT = _data()
        inp = {'imgs': imgs, 'R': R0 + dR, 'T': T0 + dT}
        assert vp.reduces_inside_backward(inp) == (reduce_at == 'scene')
        vp.forward_backward(inp)
        first = (dR.grad.clone(), dT.grad.clone(), vp.bucket.grads_flat().clone())
        vp.forward_backward({'imgs': imgs, 'R': R0 + dR, 'T': T0 + dT})      # the caller's leaves accumulate
        sizes = list(vp.bucket.peer.sizes) if vp.bucket.peer is not None else None
        out[(rank, row_bands, reduce_at)] = (*first, dR.grad.clone(), dT.grad.clone(), sizes)
    dist.destroy_process_group()


def _reference():
    """the single-process step: the caller's loss back-propagated straight into dR, dT and the parameters"""
    torch.manual_seed(0)
    model = _ToyPosed()
    model.n_total_views = B
    imgs, R0, T0, dR, dT = _data()
    total = model({'imgs': imgs, 'R': R0 + dR, 'T': T0 + dT})['total']
    params = [p for p in model.parameters()]
    *g, gR, gT = torch.autograd.grad(total, params + [dR, dT])
    return gR, gT, torch.cat([x.reshape(-1) for x in g])


def test_pose_gradients_summed_over_two_gloo_ranks_equal_single_process():
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(2, 35000 + os.getpid() % 2000, out), nprocs=2, join=True)
    gR, gT, gp = _reference()
    assert gR.abs().max() > 0 and gT.abs().max() > 0
    for row_bands, reduce_at in CONFIGS:
        r0, r1 = out[(0, row_bands, reduce_at)], out[(1, row_bands, reduce_at)]
        for i in range(5):
            assert torch.equal(r0[i], r1[i]), (row_bands, reduce_at, i)           # identical on every rank
        got_R, got_T, got_p, acc_R, acc_T, sizes = r0
        what = f'row_bands={row_bands} reduce_at={reduce_at}'
        assert torch.allclose(got_R, gR, rtol=1e-5, atol=1e-7), what
        assert torch.allclose(got_T, gT, rtol=1e-5, atol=1e-7), what
        assert torch.allclose(got_p, gp, rtol=1e-5, atol=1e-7), what
        assert torch.allclose(acc_R, 2 * gR, rtol=1e-5, atol=1e-7) and torch.allclose(acc_T, 2 * gT, rtol=1e-5, atol=1e-7), what
        if reduce_at == 'scene':                  # one exchange per step: the scene tensors' W + 3 floats and 12 per view
            assert sizes == [W + 3 + 12 * B] * 2, (what, sizes)


def test_one_process_pose_step_equals_the_eager_step():
    """world size 1, leaf bucket gathered: the pose gradient lands in the bucket's pose region (B x 9 of g_R, then B x 3
    of g_T, after the padded parameter gradients) and reaches the caller's leaves"""
    from dbw_b200.parallel import ViewParallel
    torch.manual_seed(0)
    model = _ToyPosed()
    vp = ViewParallel(model, seed=123, max_pose_views=MAX_POSE_VIEWS, gather_grads=True)
    imgs, R0, T0, dR, dT = _data()
    vp.forward_backward({'imgs': imgs, 'R': R0 + dR, 'T': T0 + dT})
    gR, gT, gp = _reference()
    assert torch.allclose(dR.grad, gR, rtol=1e-6, atol=1e-8) and torch.allclose(dT.grad, gT, rtol=1e-6, atol=1e-8)
    assert torch.allclose(vp.bucket.grads_flat(), gp, rtol=1e-6, atol=1e-8)
    n_pad = vp.bucket.flat.numel()
    region = vp.bucket._all[n_pad:n_pad + 12 * B]
    assert torch.equal(region, torch.cat([dR.grad.reshape(-1), dT.grad.reshape(-1)]))
    assert vp.bucket._all.numel() == n_pad + 12 * MAX_POSE_VIEWS


def test_pose_steps_refuse_what_they_cannot_do():
    from dbw_b200.parallel import ViewParallel
    imgs, R0, T0, dR, dT = _data()
    posed = {'imgs': imgs, 'R': R0 + dR, 'T': T0}
    with pytest.raises(RuntimeError, match='requires grad'):
        ViewParallel(_ToyPosed(), seed=1).forward_backward(posed)                        # max_pose_views = 0: as before
    with pytest.raises(ValueError, match='max_pose_views=4'):
        ViewParallel(_ToyPosed(), seed=1, max_pose_views=4).forward_backward(posed)     # 5 views > 4
    vp = ViewParallel(_ToyPosed(), seed=1, max_pose_views=8)
    with pytest.raises(ValueError, match='full batch'):
        vp.forward_backward(posed, already_sharded=True, n_total_views=B)
    with pytest.raises(ValueError, match='full batch'):
        vp.forward_backward(dict(posed, R=(R0 + dR)[:3]))
    assert dR.grad is None
