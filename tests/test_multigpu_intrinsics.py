"""Two ranks: intrinsics gradients through the data-parallel step of the scene model (ViewParallel(max_pose_views=N,
intrinsics=True)), whole views and row bands, summed at the leaves (the intrinsics block after the poses in the bucket) or at the
scene tensors (the intrinsics leaves ride through the GradSumPoint exchange, and the model renders from the point's K).  A
focal-scale leaf gets the single-process gradient, bit-identical on both ranks, and so does every parameter.

With two GPUs each rank has its own device and sums with the peer-memory kernel (p2p) or NCCL; eager and captured steps.  With
one GPU the two ranks share it and sum over gloo (the scene-level exchange through a device bucket standing in for the
peer-memory arena); a captured step needs the peer-memory kernel, so its cases need two GPUs."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

B = 5
# (reduce_at, row_bands, graphed)
CASES = [('leaf', False, False), ('leaf', True, False), ('scene', False, False), ('scene', True, False), ('auto', True, True),
         ('leaf', False, True)]


class _DeviceGlooBucket:
    """stands in for parallel.PeerAllReduce on one shared GPU: a device bucket summed in place over gloo"""

    def __init__(self, n_floats, device):
        self.flat = torch.zeros(n_floats, device=device)
        self.sizes = []

    def all_reduce(self, buf):
        assert buf.data_ptr() == self.flat.data_ptr()
        self.sizes.append(buf.numel())
        dist.all_reduce(buf)


def _setup(dev):
    from copy import deepcopy
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from oracle import dbw_path as D
    from tests.test_model_gpu import CFG
    cfg = deepcopy(CFG)
    cfg['loss'] = {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1}
    torch.manual_seed(5)
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev).train()
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=7)
    g = torch.Generator().manual_seed(7)
    Ks = K.float()[None].repeat(B, 1, 1)
    Ks[:, 0, 2] += 0.05 * torch.randn(B, generator=g)
    inp = {'imgs': torch.rand(B, 3, 48, 64, generator=g).to(dev), 'R': R.float().to(dev), 'T': T.float().to(dev),
           'K': Ks.to(dev)}
    scale = (1 + 0.02 * torch.randn(B, generator=g)).to(dev).requires_grad_(True)
    return model, inp, scale


def _focal(K, scale):
    """K with fx, fy scaled per view (the principal point untouched)"""
    f = torch.stack([scale, scale, torch.ones_like(scale), torch.ones_like(scale)], -1)
    return K * torch.diag_embed(f) + K * (1 - torch.eye(4, device=K.device))


def _w_step(rank, world, port, out, reduce_at, row_bands, graphed):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    two = torch.cuda.device_count() >= 2
    dev = torch.device('cuda', rank if two else 0)
    torch.cuda.set_device(dev)
    if two:
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)
    import dbw_b200  # noqa: F401
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, inp, scale = _setup(dev)
    kw = dict(collective='p2p') if two else dict(collective='nccl', peer_factory=_DeviceGlooBucket if reduce_at != 'leaf' else None)
    vp = ViewParallel(model, seed=5, row_bands=row_bands, reduce_at=reduce_at, max_pose_views=B, intrinsics=True, **kw)
    if graphed:
        step = GraphedStep(vp, dict(inp, K=_focal(inp['K'], scale)), B, warmup=1)
        step.run(dict(inp, K=_focal(inp['K'], scale)))
        inside = step.inside
    else:
        vp.forward_backward(dict(inp, K=_focal(inp['K'], scale)))
        inside = vp.reduces_inside_backward(vp.shard(inp)[0])
    torch.cuda.synchronize()
    out[rank] = (scale.grad.cpu(), vp.bucket.grads_flat().cpu(), inside)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('reduce_at,row_bands,graphed', CASES)
def test_two_rank_focal_scale_gradient_equals_single_process(reduce_at, row_bands, graphed):
    if graphed and torch.cuda.device_count() < 2:
        pytest.skip('a captured two-rank step sums with the peer-memory kernel: needs 2 GPUs')
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_w_step, args=(2, 31700 + os.getpid() % 1000, out, reduce_at, row_bands, graphed), nprocs=2, join=True)
    assert out[0][2] == out[1][2] == (reduce_at != 'leaf')
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    import dbw_b200  # noqa: F401
    model, inp, scale = _setup(torch.device('cuda:0'))
    params = [p for p in model.parameters() if p.requires_grad]
    model.n_total_views = B
    total = model(dict(inp, K=_focal(inp['K'], scale)), None)['total']
    *gp, gs = torch.autograd.grad(total, params + [scale], allow_unused=True)
    flat = torch.cat([(g if g is not None else torch.zeros_like(p)).reshape(-1) for g, p in zip(gp, params)]).cpu()
    assert gs.abs().min() > 0
    for got, ref, what in ((out[0][0], gs.cpu(), 'focal scale'), (out[0][1], flat, 'parameters')):
        err = ((got - ref).norm() / ref.norm()).item()
        print(f'\n{reduce_at} row_bands={row_bands} graphed={graphed}: {what} rel err {err:.3e}')
        assert err <= 1e-4, (what, err)
