"""Multi-GPU (skipped with fewer than 2 GPUs): the hand-written NVLink peer-memory all-reduce
(csrc/dbw_comm.cu) against ncclAllReduce, eagerly and captured inside a CUDA graph, and a row-band-sharded 2-rank step
against the single-GPU step."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
needs2 = pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')


def _w_allreduce(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    import dbw_b200  # noqa: F401
    from dbw_b200.parallel import PeerAllReduce
    res = {}
    for n in (64, 36864, 2_400_004):                         # one-shot (tiny), one-shot (the scene-tensor gradients), two-shot (9.6 MB)
        n4 = (n + 3) // 4 * 4
        comm = PeerAllReduce(n4, dev)
        g = torch.Generator(device=dev).manual_seed(100 + rank)
        ok = True
        for it in range(5):                                  # several epochs: flag stamps, inbox / bucket reuse
            x = torch.randn(n4, device=dev, generator=g)
            ref = x.clone()
            dist.all_reduce(ref)
            y = comm.flat                                    # the arena's bucket: the all-reduce works in place on it
            y.copy_(x)
            comm.all_reduce(y)
            torch.cuda.synchronize()
            ok = ok and bool((y - ref).abs().max() <= 1e-5 * ref.abs().max())
            gathered = [torch.empty_like(y) for _ in range(world)]
            dist.all_gather(gathered, y)
            ok = ok and all(torch.equal(gathered[0], t) for t in gathered)       # bit-identical on every rank
            if n4 > 131072:
                # a small exchange on a PREFIX of the same bucket (the one-shot path and its deferred barrier) between two
                # large ones, twice in a row: the paths share the inbox and the flags
                for _ in range(2):
                    small = comm.flat[:36864]
                    xs = torch.randn(36864, device=dev, generator=g)
                    refs = xs.clone()
                    dist.all_reduce(refs)
                    small.copy_(xs)
                    comm.all_reduce(small)
                    torch.cuda.synchronize()
                    ok = ok and bool((small - refs).abs().max() <= 1e-5 * refs.abs().max())
                    gs = [torch.empty_like(small) for _ in range(world)]
                    dist.all_gather(gs, small)
                    ok = ok and all(torch.equal(gs[0], t) for t in gs)
        # captured in a CUDA graph and replayed
        static = comm.flat
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            comm.all_reduce(static)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            comm.all_reduce(static)
        for it in range(3):
            x = torch.randn(n4, device=dev, generator=g)
            ref = x.clone()
            dist.all_reduce(ref)
            static.copy_(x)
            graph.replay()
            torch.cuda.synchronize()
            ok = ok and bool((static - ref).abs().max() <= 1e-5 * ref.abs().max())
        res[n] = (ok, comm.error())
        dist.barrier()
        comm.close()
    out[rank] = res
    dist.destroy_process_group()


@needs2
def test_peer_memory_all_reduce_matches_nccl():
    world = min(torch.cuda.device_count(), 8)
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_w_allreduce, args=(world, 29500 + os.getpid() % 1000, out), nprocs=world, join=True)
    for rank in range(world):
        for n, (ok, err) in out[rank].items():
            assert ok and err == 0, (rank, n, ok, err)


LOSS_RGB = {'rgb_weight': 1}
LOSS_REG = {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1}      # + replicated terms (identical on every rank)


def _w_step(rank, world, port, out, collective, reduce_at, loss):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    import dbw_b200  # noqa: F401
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.graph import GraphedStep
    from tests.test_model_gpu import CFG
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from oracle import dbw_path as D
    from copy import deepcopy
    cfg = deepcopy(CFG)
    cfg['loss'] = dict(loss)
    torch.manual_seed(5)
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev)
    model.train()
    R, T, K = D.ring_cameras(5, jitter=0.3, seed=7)
    g = torch.Generator().manual_seed(7)
    inp = {'imgs': torch.rand(5, 3, 48, 64, generator=g), 'R': R, 'T': T, 'K': K[None].expand(5, -1, -1).contiguous()}
    vp = ViewParallel(model, seed=5, row_bands=True, collective=collective, reduce_at=reduce_at)
    local, n_total = vp.shard(inp)
    local = {k: v.to(dev) for k, v in local.items()}
    graphed = GraphedStep(vp, local, n_total)
    graphed.run()
    graphed.run()                                   # a replay after the first: the bucket / gradient views are reused
    torch.cuda.synchronize()
    out[rank] = (vp.bucket.grads_flat().cpu(), graphed.capture_all_reduce, local['rows'].cpu().tolist(), graphed.noise_buf.cpu(),
                 graphed.inside, vp.bucket.peer.error() if vp.bucket.peer is not None else 0)
    dist.barrier()
    dist.destroy_process_group()


@needs2
@pytest.mark.parametrize('collective,reduce_at,loss', [('p2p', 'auto', LOSS_RGB), ('p2p', 'auto', LOSS_REG), ('p2p', 'leaf', LOSS_REG),
                                                       ('nccl', 'auto', LOSS_RGB)])
def test_two_rank_row_band_step_equals_single_gpu_step(collective, reduce_at, loss):
    """5 views of 48 rows over 2 ranks = 7.5 bands each: the ranks split view 2 in the middle; the gradients -- summed over the
    ranks inside the backward at the scene tensors (GradSumPoint; textures are decimated at iteration 0), or all-reduced at the
    leaves by the peer-memory kernel inside the step's CUDA graph, or by NCCL after the replay -- == the single-GPU step's,
    replicated regularisers included"""
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_w_step, args=(2, 29600 + os.getpid() % 1000, out, collective, reduce_at, loss), nprocs=2, join=True)
    assert out[0][1] == (collective == 'p2p')
    assert out[0][4] == out[1][4] == (collective == 'p2p' and reduce_at == 'auto')
    assert out[0][5] == out[1][5] == 0
    assert out[0][2][-1][1] < 48 and out[1][2][0][0] > 0             # view 2 is shared
    assert torch.equal(out[0][0], out[1][0]) if collective == 'p2p' else torch.allclose(out[0][0], out[1][0], rtol=1e-6, atol=1e-9)
    import dbw_b200  # noqa: F401
    from dbw_b200.parallel import ViewParallel
    from tests.test_model_gpu import CFG
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from oracle import dbw_path as D
    from copy import deepcopy
    cfg = deepcopy(CFG)
    cfg['loss'] = dict(loss)
    torch.manual_seed(5)
    dev = torch.device('cuda:0')
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev)
    model.train()
    R, T, K = D.ring_cameras(5, jitter=0.3, seed=7)
    g = torch.Generator().manual_seed(7)
    inp = {'imgs': torch.rand(5, 3, 48, 64, generator=g).to(dev), 'R': R.to(dev), 'T': T.to(dev), 'K': K[None].expand(5, -1, -1).to(dev)}
    vp = ViewParallel(model, seed=5)
    model.opacity_noise_buffer = out[0][3].to(dev)
    vp.forward_backward(inp)
    ref = vp.bucket.grads_flat().cpu()
    assert (out[0][0] - ref).norm() <= 1e-4 * ref.norm(), ((out[0][0] - ref).norm().item(), ref.norm().item())
