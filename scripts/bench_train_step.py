"""What the parameter update costs a graph-captured training iteration, and what capturing it saves: full iterations of the
scene model (coarse phase, 10 blocks, 256^2 textures, fused loss epilogue, no perceptual term), each a graph.GraphedStep
replay followed by the update and a scheduler step, three ways, alternating in one process:

  eager_foreach   GraphedStep + torch.optim.Adam (the default multi-tensor path) stepped after the replay
  eager_fused     GraphedStep + torch.optim.Adam(fused=True) stepped after the replay
  captured        GraphedStep(optimizer=optim.BucketAdam): the update is the last kernel of the replay

All three use the reference's two groups (the `texture*` parameters at ten times the rate) and a torch MultiStepLR stepped every
iteration (the host work of the reference's scheduler, src/scheduler.py).  Two shapes:

  train  4 views x 300x400 (the DTU training batch)
  dtu    49 views x 400x400 (the bench.py workload)

Per shape and mode: host wall time per iteration over --iters iterations ending in a device synchronise, after --warmup
iterations (median, min and max of --repeat alternating repeats), and the library's kernel launches per iteration (counted
while the step is captured; torch's own optimiser kernels are not the library's and are not in it).  One GPU; prints one JSON
line with the card's name and power limit.

    python scripts/bench_train_step.py [--iters 200] [--warmup 20] [--repeat 3]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_camera_grad import CFG, SHAPES, card  # noqa: E402

MODES = ('eager_foreach', 'eager_fused', 'captured')
OPT = {'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}


def build(mode, shape, dev):
    """(run one iteration, library launches per iteration)"""
    from copy import deepcopy
    from dbw_b200 import _lib
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.synthetic import ring_cameras
    B, H, W = SHAPES[shape]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).train()
    R, T, K = ring_cameras(B)
    inp = {'imgs': torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev), 'R': R.to(dev), 'T': T.to(dev),
           'K': K[None].expand(B, -1, -1).contiguous().to(dev)}
    vp = ViewParallel(model, seed=1)
    n = _lib.launch_count()
    if mode == 'captured':
        opt = create_optimizer(OPT, model)
        step = GraphedStep(vp, inp, B, warmup=1, optimizer=opt)
        launches = (_lib.launch_count() - n - 1) / 2 + 1          # warm-up + capture; the update is launched in the capture only
    else:
        named = list(model.named_parameters())
        o = OPT['training']['optimizer']
        opt = torch.optim.Adam([{'params': [p for k, p in named if not k.startswith('texture')]},
                                {'params': [p for k, p in named if k.startswith('texture')], **o['texture']}], lr=o['lr'],
                               fused=(mode == 'eager_fused'))
        step = GraphedStep(vp, inp, B, warmup=1)
        launches = (_lib.launch_count() - n) / 2
    sched = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[10 ** 9], gamma=0.1)

    def iteration():
        step.run()
        if mode != 'captured':
            opt.step()
        sched.step()

    return iteration, launches


def measure(shape, iters, warmup, repeat, dev):
    runs, launches = {}, {}
    for mode in MODES:
        runs[mode], launches[mode] = build(mode, shape, dev)
    for mode in MODES:
        for _ in range(warmup):
            runs[mode]()
    torch.cuda.synchronize()
    times = {m: [] for m in MODES}
    for _ in range(repeat):
        for mode in MODES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                runs[mode]()
            torch.cuda.synchronize()
            times[mode].append((time.perf_counter() - t0) * 1e3 / iters)
    out = {}
    for mode in MODES:
        ms = sorted(times[mode])
        out[mode] = {'iteration_ms_median': ms[len(ms) // 2], 'iteration_ms_min': ms[0], 'iteration_ms_max': ms[-1],
                     'library_launches_per_iteration': launches[mode]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--repeat', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    name, limit = card()
    res = {'card': name, 'power_limit_w': limit, 'iters': args.iters, 'warmup': args.warmup, 'repeat': args.repeat}
    dev = torch.device('cuda:0')
    for shape in ('train', 'dtu'):
        B, H, W = SHAPES[shape]
        res[f'{shape} ({B} x {H}x{W})'] = measure(shape, args.iters, args.warmup, args.repeat, dev)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
