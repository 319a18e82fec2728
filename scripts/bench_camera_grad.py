"""What differentiating the camera poses costs: one training step of the scene model (model(inp) + backward, coarse phase,
10 blocks, fused loss epilogue) with the dataset poses as constants, and with R and T computed from leaves that require
grad (a pose correction, as a pose-refining trainer would feed them).  Two shapes:

  dtu    49 views x 400x400 (the bench.py workload)
  train  4 views x 300x400 (the DTU training batch)

Per shape and mode: the step's time (CUDA events, the two modes alternating, median of --repeat), the raster-backward
kernel times of the environment pass (K = 1, both launches of its split backward) and of the blocks pass (K = 10) from
dbw_timing_*, the device time of camera_grad_kernel from torch.profiler, and the library's launch count per step.  Prints
one JSON line with the card's name and power limit.

    python scripts/bench_camera_grad.py [--repeat 20]
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
    inp = {'imgs': torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev), 'R': R.to(dev), 'T': T.to(dev),
           'K': K[None].expand(B, -1, -1).contiguous().to(dev)}
    dR = torch.zeros(B, 3, 3, device=dev, requires_grad=True)
    dT = torch.zeros(B, 3, device=dev, requires_grad=True)

    def step(pose):
        model.zero_grad(set_to_none=True)
        dR.grad = dT.grad = None
        x = dict(inp, R=inp['R'] + dR, T=inp['T'] + dT) if pose else inp
        model(x, None)['total'].backward()

    modes = {'constant_poses': False, 'pose_gradients': True}
    times = {m: [] for m in modes}
    for m, pose in modes.items():          # warm-up: lazy state, allocator
        step(pose); step(pose)
    torch.cuda.synchronize()
    for _ in range(repeat):
        for m, pose in modes.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(pose)
            b.record()
            torch.cuda.synchronize()
            times[m].append(a.elapsed_time(b))
    out = {}
    L = _lib.lib()
    for m, pose in modes.items():
        ms = sorted(times[m])
        row = {'step_ms_median': ms[len(ms) // 2], 'step_ms_min': ms[0]}
        L.dbw_timing_reset()
        L.dbw_timing_enable(1)
        n0 = _lib.launch_count()
        for _ in range(5):
            step(pose)
        torch.cuda.synchronize()
        row['launches_per_step'] = (_lib.launch_count() - n0) / 5
        env_ms, n_env = _lib.kernel_time_ms(1, 1)
        blk_ms, n_blk = _lib.kernel_time_ms(1, 10)
        L.dbw_timing_enable(0)
        L.dbw_timing_reset()
        row['env_backward_ms'] = env_ms / max(n_env, 1)
        row['blocks_backward_ms'] = blk_ms / max(n_blk, 1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(pose)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            for key in ('camera_grad_kernel', 'raster_bary_backward_kernel', 'face_setup_backward_kernel'):
                if key in e.key:
                    kern[key] = kern.get(key, 0.0) + e.device_time_total / 1000.0
        row['profiled_ms'] = kern
        out[m] = row
    out['step_overhead_ms'] = out['pose_gradients']['step_ms_median'] - out['constant_poses']['step_ms_median']
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
