"""Two GPUs: camera-pose gradients through the data-parallel step (ViewParallel(max_pose_views=N)), eager and graphed, whole
views and row bands, summed at the leaves (the pose region of the bucket: peer-memory kernel or NCCL) or at the scene tensors
(the pose leaves ride through the GradSumPoint exchange).  The pose and parameter gradients equal the single-GPU step's, the
pose gradients are bit-identical on both ranks, and a step issues one collective."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

needs2 = pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
pytestmark = pytest.mark.gpu

B = 5
# (collective, reduce_at, row_bands, graphed)
CASES = [('p2p', 'auto', True, True), ('p2p', 'leaf', False, True), ('nccl', 'auto', True, False), ('nccl', 'leaf', False, True),
         ('p2p', 'auto', False, False)]


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
    inp = {'imgs': torch.rand(B, 3, 48, 64, generator=g).to(dev), 'R': R.float().to(dev), 'T': T.float().to(dev),
           'K': K.float()[None].expand(B, -1, -1).contiguous().to(dev)}
    dR = (0.01 * torch.randn(B, 3, 3, generator=g)).to(dev).requires_grad_(True)
    dT = (0.01 * torch.randn(B, 3, generator=g)).to(dev).requires_grad_(True)
    return model, inp, dR, dT


def _w_step(rank, world, port, out, collective, reduce_at, row_bands, graphed):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    import dbw_b200  # noqa: F401
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    model, inp, dR, dT = _setup(dev)
    vp = ViewParallel(model, seed=5, row_bands=row_bands, collective=collective, reduce_at=reduce_at, max_pose_views=B)
    calls = [0]
    if vp.bucket.peer is not None:
        peer_all_reduce = vp.bucket.peer.all_reduce

        def counted(buf):
            calls[0] += 1
            peer_all_reduce(buf)
        vp.bucket.peer.all_reduce = counted
    nccl_all_reduce = dist.all_reduce

    def counted_nccl(*a, **k):
        calls[0] += 1
        return nccl_all_reduce(*a, **k)
    dist.all_reduce = counted_nccl
    try:
        posed = dict(inp, R=inp['R'] + dR, T=inp['T'] + dT)
        if graphed:
            step = GraphedStep(vp, posed, B, warmup=1)
            built = calls[0]
            step.run(posed)
            per_step = (calls[0] - built) if not step.capture_all_reduce else built / 2   # captured: once per body
            inside = step.inside
        else:
            vp.forward_backward(posed)
            per_step = calls[0]
            inside = vp.reduces_inside_backward(vp.shard(inp)[0])
    finally:
        dist.all_reduce = nccl_all_reduce
    torch.cuda.synchronize()
    out[rank] = (dR.grad.cpu(), dT.grad.cpu(), vp.bucket.grads_flat().cpu(), per_step, inside,
                 vp.bucket.peer.error() if vp.bucket.peer is not None else 0)
    dist.barrier()
    dist.destroy_process_group()


@needs2
@pytest.mark.parametrize('collective,reduce_at,row_bands,graphed', CASES)
def test_two_rank_pose_step_equals_single_gpu_step(collective, reduce_at, row_bands, graphed):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_w_step, args=(2, 29700 + os.getpid() % 1000, out, collective, reduce_at, row_bands, graphed), nprocs=2, join=True)
    assert out[0][5] == out[1][5] == 0
    assert out[0][4] == out[1][4] == (collective == 'p2p' and reduce_at == 'auto')
    assert out[0][3] == out[1][3] == 1, (out[0][3], out[1][3])             # one collective per step
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    import dbw_b200  # noqa: F401
    dev = torch.device('cuda:0')
    model, inp, dR, dT = _setup(dev)
    params = [p for p in model.parameters() if p.requires_grad]
    model.n_total_views = B
    total = model(dict(inp, R=inp['R'] + dR, T=inp['T'] + dT), None)['total']
    *gp, gR, gT = torch.autograd.grad(total, params + [dR, dT], allow_unused=True)
    flat = torch.cat([(g if g is not None else torch.zeros_like(p)).reshape(-1) for g, p in zip(gp, params)]).cpu()
    for got, ref, what in ((out[0][0], gR.cpu(), 'g_R'), (out[0][1], gT.cpu(), 'g_T'), (out[0][2], flat, 'parameters')):
        assert ref.abs().max() > 0, what
        assert (got - ref).norm() <= 1e-4 * ref.norm(), (what, ((got - ref).norm() / ref.norm()).item())
