"""What the depth outputs cost on the GPU: the scene model's two render passes (environment K = 1, blocks K = 10, coarse phase,
the bench.py scene: 10 blocks, 256^2 textures) with and without depth, two ways, alternating in one process:

  passes  DifferentiableBlocksWorld._render_layers(inp) against _render_layers(inp, depth=True): forward, then backward of a
          weighted sum of the outputs (the depth arm also weighs each pass's depth) -- each timed with CUDA events
  step    one eager step: predict(inp) + MSE against the images, against predict(inp, with_depth=True) + MSE + an L1 depth
          term against a target depth; forward and backward, CUDA-synchronised wall clock

Shapes: dtu (49 views, 400x400) and bmvs (64 views, 576x768).  Per shape, arm and measure: the median of --repeat alternating
runs (after --warmup runs of every arm).  Prints one JSON line with the card's name and power limit.

    python scripts/bench_depth.py [--repeat 9] [--warmup 2] [--shapes dtu,bmvs]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from copy import deepcopy

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'dtu': (49, 400, 400), 'bmvs': (64, 576, 768)}
CFG = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
       'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
       'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                      'decouple_rendering': True, 'opacity_noise': False},
       'loss': {'rgb_weight': 1}}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def setup(n_views, H, W, dev):
    from oracle import dbw_path as D
    from dbw_b200.dbw import DifferentiableBlocksWorld
    torch.manual_seed(0)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev)
    model.train()
    R, T, K = D.ring_cameras(n_views, dtype=torch.float32, jitter=0.1, seed=1)
    imgs = torch.rand(n_views, 3, H, W, generator=torch.Generator().manual_seed(2))
    inp = {'imgs': imgs.to(dev), 'R': R.to(dev), 'T': T.to(dev), 'K': K[None].expand(n_views, -1, -1).to(dev)}
    with torch.no_grad():
        target_depth = model.predict(inp, with_depth=True)[1] * 1.05
    return model, inp, target_depth


def passes_arm(model, inp, depth, weights):
    """(forward ms, backward ms) of the two passes"""
    a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    model.zero_grad(set_to_none=True)
    a.record()
    env, fg = model._render_layers(inp, depth=depth)
    b.record()
    outs = [env[0], env[1], fg[0], fg[1]] if depth else [env, fg]
    torch.autograd.backward(outs, [weights[o.shape[1]] for o in outs])
    c.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), b.elapsed_time(c)


def step_arm(model, inp, depth, target_depth):
    """ms of one eager step: forward, loss, backward"""
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if depth:
        rec, dep = model.predict(inp, with_depth=True)
        loss = F.mse_loss(rec, inp['imgs']) + 0.1 * (dep - target_depth).abs().mean()
    else:
        loss = F.mse_loss(model.predict(inp), inp['imgs'])
    loss.backward()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=9)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--shapes', default='dtu,bmvs')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_depth.py measures the GPU: no CUDA device')
    dev = torch.device('cuda:0')
    name, power = card()
    result = {'gpu': name, 'power_limit_w': power, 'repeat': args.repeat, 'shapes': {}}
    for shape in args.shapes.split(','):
        n_views, H, W = SHAPES[shape]
        model, inp, target_depth = setup(n_views, H, W, dev)
        g = torch.Generator(device=dev).manual_seed(3)
        weights = {4: torch.rand(n_views, 4, H, W, device=dev, generator=g), 1: torch.rand(n_views, 1, H, W, device=dev, generator=g)}
        runs = {k: [] for k in ('fwd_rgba', 'bwd_rgba', 'fwd_depth', 'bwd_depth', 'step_rgba', 'step_depth')}
        for i in range(args.warmup + args.repeat):
            for depth in (False, True):                      # alternating arms
                f, b = passes_arm(model, inp, depth, weights)
                s = step_arm(model, inp, depth, target_depth)
                if i >= args.warmup:
                    arm = 'depth' if depth else 'rgba'
                    runs['fwd_' + arm].append(f); runs['bwd_' + arm].append(b); runs['step_' + arm].append(s)
        med = {k: statistics.median(v) for k, v in runs.items()}
        for m in ('fwd', 'bwd', 'step'):
            med[m + '_cost_pct'] = 100.0 * (med[m + '_depth'] / med[m + '_rgba'] - 1.0)
        result['shapes'][shape] = {'views': n_views, 'size': [H, W], 'median_ms': med}
        del model, inp, target_depth, weights
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
