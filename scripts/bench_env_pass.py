"""Device time of the environment pass's three kernels in a training step of the bench's model: the hard forward, the
texture backward (raster_backward_kernel<true, false, true>) and the barycentric-path backward of the ground
(raster_bary_backward_kernel), per step, from torch.profiler over eager steps (a run of its own: tracing slows the host,
not the kernels).  Prints one JSON line with the card's name and power limit.  DBW_RENDER_LIB selects another build of
the library to compare against.

  python scripts/bench_env_pass.py [--workload dtu|bmvs] [--steps N] [--repeat R]"""
import argparse
import json
import os
import subprocess
import sys
from copy import deepcopy

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import bench  # noqa: E402
import dbw_b200  # noqa: F401,E402
from dbw_b200 import _lib  # noqa: E402
from dbw_b200.dbw import DifferentiableBlocksWorld  # noqa: E402
from dbw_b200.parallel import ViewParallel  # noqa: E402

KERNELS = {'env forward': 'raster_hard_forward_kernel', 'env texture backward': 'raster_backward_kernel<true, false, true>',
           'env bary backward': 'raster_bary_backward_kernel'}


def card():
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='dtu', choices=['dtu', 'bmvs'])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--repeat', type=int, default=3)
    args = ap.parse_args()
    w = bench.WORKLOADS[args.workload]
    dev = torch.device('cuda:0')
    torch.manual_seed(bench.SEED)
    model = DifferentiableBlocksWorld((w['height'], w['width']), **deepcopy(bench.model_cfg(w))).to(dev)
    model.train()
    vp = ViewParallel(model, seed=bench.SEED)
    inp = {k: v.to(dev) for k, v in bench.synthetic_inputs(w).items()}
    for _ in range(3):
        vp.forward_backward(inp)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    runs = []
    for _ in range(args.repeat):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                vp.forward_backward(inp)
            torch.cuda.synchronize()
        tot = {k: 0.0 for k in KERNELS}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for k, pat in KERNELS.items():
                if pat in e.name:
                    tot[k] += e.time_range.elapsed_us() / 1e3
        runs.append({k: round(v / args.steps, 4) for k, v in tot.items()})
    print(json.dumps({'workload': args.workload, 'card': card(), 'library': os.path.relpath(_lib.LIB_PATH),
                      'steps_per_run': args.steps, 'ms_per_step': runs}))


if __name__ == '__main__':
    main()
