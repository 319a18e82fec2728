"""What rendering each view with its own intrinsics costs: one training step of the scene model (model(inp) + backward, coarse
phase, 10 blocks, fused loss epilogue) three ways, alternating in one process:

  default         the reference's cameras: K[0] of the first batch for every view (what bench.py runs)
  per_view_K      model.set_per_view_intrinsics(True), every view's own K read on the device, K a constant
  per_view_K_grad K computed from a focal-scale leaf that requires grad (joint pose / focal refinement)

Two shapes:

  dtu    49 views x 400x400 (the bench.py workload)
  train  4 views x 300x400 (the DTU training batch)

Per shape and mode: the step's time (CUDA events, the modes alternating, median of --repeat), the device time of the
projection kernels from torch.profiler, and the library's launch count per step.  Prints one JSON line with the card's name
and power limit.

    python scripts/bench_intrinsics.py [--repeat 20]
"""
import argparse
import json
import os
import subprocess
import sys
from copy import deepcopy

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'dtu': (49, 400, 400), 'train': (4, 300, 400)}
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


def measure(shape, repeat):
    from dbw_b200 import _lib
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.synthetic import ring_cameras
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device('cuda')
    B, H, W = SHAPES[shape]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).train()
    R, T, K = ring_cameras(B)
    Ks = K[None].repeat(B, 1, 1)
    Ks[:, 0, 0] *= 1 + 0.02 * torch.linspace(-1, 1, B)           # every view its own focal length and principal point
    Ks[:, 1, 2] += 0.01 * torch.linspace(-1, 1, B)
    inp = {'imgs': torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev), 'R': R.to(dev), 'T': T.to(dev),
           'K': Ks.contiguous().to(dev)}
    scale = torch.ones(B, device=dev, requires_grad=True)

    def step(mode):
        model.zero_grad(set_to_none=True)
        scale.grad = None
        model.set_per_view_intrinsics(mode == 'per_view_K')
        x = inp
        if mode == 'per_view_K_grad':
            x = dict(inp, K=inp['K'] * torch.stack([scale, scale, torch.ones_like(scale), torch.ones_like(scale)], -1)[:, :, None])
        model(x, None)['total'].backward()

    modes = ('default', 'per_view_K', 'per_view_K_grad')
    times = {m: [] for m in modes}
    for m in modes:                        # warm-up: lazy state, allocator
        step(m); step(m)
    torch.cuda.synchronize()
    for _ in range(repeat):
        for m in modes:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(m)
            b.record()
            torch.cuda.synchronize()
            times[m].append(a.elapsed_time(b))
    out = {}
    for m in modes:
        ms = sorted(times[m])
        row = {'step_ms_median': ms[len(ms) // 2], 'step_ms_min': ms[0]}
        n0 = _lib.launch_count()
        for _ in range(5):
            step(m)
        torch.cuda.synchronize()
        row['launches_per_step'] = (_lib.launch_count() - n0) / 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(m)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            for key in ('project_verts_kernel', 'camera_project_kernel', 'camera_project_verts_backward_kernel',
                        'camera_project_camera_backward_kernel', 'project_verts_backward_kernel', 'camera_grad_kernel'):
                if key in e.key and (key.startswith('camera_') or 'camera_' not in e.key) and (key != 'project_verts_kernel' or 'backward' not in e.key):
                    kern[key] = kern.get(key, 0.0) + e.device_time_total / 1000.0
        row['profiled_ms'] = kern
        out[m] = row
    for m in modes[1:]:
        out[f'{m}_overhead_ms'] = out[m]['step_ms_median'] - out['default']['step_ms_median']
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=20)
    args = ap.parse_args()
    name, limit = card()
    res = {'card': name, 'power_limit_w': limit, 'repeat': args.repeat}
    for shape in SHAPES:
        B, H, W = SHAPES[shape]
        res[f'{shape} ({B} x {H}x{W})'] = measure(shape, args.repeat)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
