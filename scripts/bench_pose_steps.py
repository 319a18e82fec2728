"""What pose gradients cost a graph-captured training step: graph.GraphedStep replays of the scene model (coarse phase, 10
blocks, fused loss epilogue) with constant poses, and with full-batch poses that require grad (a per-view correction on top of
the dataset poses, as a pose-refining trainer feeds them; ViewParallel(max_pose_views=B)), the two alternating.  Two shapes:

  dtu    49 views x 400x400 (the bench.py workload)
  train  4 views x 300x400 (the DTU training batch)

Per shape and mode: the step time (CUDA events around run(), which for pose steps includes copying the poses into the graph's
leaves and the eager backward into the caller's correction; median and min of --repeat) and the library's launches per step
(counted while the step is captured: replays launch from the graph).  With --gpus N > 1 the views are sharded over N ranks
(row bands, peer-memory collective when it initialises) and rank 0 reports.  Prints one JSON line with the card's name and
power limit.

    python scripts/bench_pose_steps.py [--repeat 20] [--gpus 1]
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_camera_grad import CFG, SHAPES, card  # noqa: E402


def measure(shape, repeat, dev, world):
    from copy import deepcopy
    from dbw_b200 import _lib
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.synthetic import ring_cameras
    B, H, W = SHAPES[shape]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).train()
    R, T, K = ring_cameras(B)
    inp = {'imgs': torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev), 'R': R.to(dev), 'T': T.to(dev),
           'K': K[None].expand(B, -1, -1).contiguous().to(dev)}
    dR = torch.zeros(B, 3, 3, device=dev, requires_grad=True)
    dT = torch.zeros(B, 3, device=dev, requires_grad=True)
    vp = ViewParallel(model, seed=1, row_bands=world > 1, collective='auto', max_pose_views=B)
    local, _ = vp.shard(inp)
    launches = {}
    steps = {}
    for mode in ('constant_poses', 'pose_gradients'):
        n = _lib.launch_count()
        if mode == 'constant_poses':
            steps[mode] = GraphedStep(vp, local, B, warmup=1)
        else:
            steps[mode] = GraphedStep(vp, dict(inp, R=inp['R'] + dR, T=inp['T'] + dT), B, warmup=1)
        torch.cuda.synchronize()
        launches[mode] = (_lib.launch_count() - n) / 2          # warm-up + capture

    def run(mode):
        if mode == 'constant_poses':
            steps[mode].run()
        else:
            dR.grad = dT.grad = None
            steps[mode].run({'R': inp['R'] + dR, 'T': inp['T'] + dT})

    for mode in steps:
        for _ in range(3):
            run(mode)
    torch.cuda.synchronize()
    times = {m: [] for m in steps}
    for _ in range(repeat):
        for mode in steps:
            if world > 1:
                dist.barrier()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run(mode)
            b.record()
            torch.cuda.synchronize()
            times[mode].append(a.elapsed_time(b))
    out = {}
    for mode in steps:
        ms = sorted(times[mode])
        out[mode] = {'step_ms_median': ms[len(ms) // 2], 'step_ms_min': ms[0], 'launches_per_step': launches[mode]}
    out['step_overhead_ms'] = out['pose_gradients']['step_ms_median'] - out['constant_poses']['step_ms_median']
    out['collective'] = vp.collective_name
    out['reduced_inside_backward'] = steps['pose_gradients'].inside
    return out


def _worker(rank, world, port, repeat, res):
    if world > 1:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        torch.cuda.set_device(rank)
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    dev = torch.device('cuda', rank)
    for shape in SHAPES:
        B, H, W = SHAPES[shape]
        row = measure(shape, repeat, dev, world)
        if rank == 0:
            res[f'{shape} ({B} x {H}x{W})'] = row
        torch.cuda.empty_cache()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=20)
    ap.add_argument('--gpus', type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < args.gpus:
        sys.exit(f'needs {args.gpus} CUDA device(s)')
    name, limit = card()
    res = {'card': name, 'power_limit_w': limit, 'repeat': args.repeat, 'gpus': args.gpus}
    if args.gpus == 1:
        _worker(0, 1, 0, args.repeat, res)
    else:
        shared = mp.Manager().dict()
        mp.spawn(_worker, args=(args.gpus, 29800 + os.getpid() % 1000, args.repeat, shared), nprocs=args.gpus, join=True)
        res.update(shared)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
