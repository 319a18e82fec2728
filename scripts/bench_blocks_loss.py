"""The coarse phase's blocks loss pass with its dedicated kernel (blocks_loss_kernel) against the generic
raster_forward_kernel<128, true> (dbw_debug_generic_blocks_loss(1)), in one process, on bench.py's model and inputs.  The two
kernels alternate, `--repeat` runs of `--steps` eager training steps each; per step:
  - blocks pass: the raster forward of the blocks pass (coarse bins + the loss kernel, dbw_timing kind 0 at K), CUDA events;
  - step: the whole eager training step, CUDA events, L2 flushed between steps as bench.py does.  (bench.py measures the
    graph-replayed step of each build.)
Prints one JSON line per workload with the card's name and power limit, the medians and the min..max spread.

  python scripts/bench_blocks_loss.py [--workload dtu bmvs] [--repeat N] [--steps S]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from copy import deepcopy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..')
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip()
    if q:
        return q
    import torch
    return torch.cuda.get_device_name(0)


def spread(xs):
    return {'median': round(statistics.median(xs), 4), 'min': round(min(xs), 4), 'max': round(max(xs), 4)}


def measure(workload, repeat, steps):
    import torch
    import bench
    import dbw_b200  # noqa: F401
    from dbw_b200 import _lib
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.parallel import ViewParallel
    w = bench.WORKLOADS[workload]
    B, K = w['n_views'], w['faces_per_pixel']
    dev = torch.device('cuda:0')
    torch.manual_seed(bench.SEED)
    model = DifferentiableBlocksWorld((w['height'], w['width']), **deepcopy(bench.model_cfg(w))).to(dev)
    model.train()
    vp = ViewParallel(model, seed=bench.SEED, row_bands=True)
    local, _ = vp.shard(bench.synthetic_inputs(w))
    rows = local.pop('rows', None)
    passes = bench.make_passes(local, rows, w)
    assert len(passes) == 1, 'one pass per step at the benched shapes'
    inp = {k: v.to(dev) for k, v in passes[0].items()}
    L = _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def eager():
        vp.forward_backward(inp, None, already_sharded=True, n_total_views=B, all_reduce=False)

    res = {g: {'blocks_pass_ms': [], 'step_ms': [], 'dedicated_launches': 0} for g in (False, True)}
    for r in range(repeat):
        for generic in ((False, True) if r % 2 == 0 else (True, False)):
            L.dbw_debug_generic_blocks_loss(int(generic))
            for _ in range(2):
                eager()
            torch.cuda.synchronize()
            L.dbw_timing_reset()
            L.dbw_timing_enable(1)
            evs = []
            for _ in range(steps):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                eager()
                b.record()
                evs.append((a, b))
            torch.cuda.synchronize()
            L.dbw_timing_enable(0)
            res[generic]['step_ms'].append(sum(a.elapsed_time(b) for a, b in evs) / steps)
            res[generic]['blocks_pass_ms'].append(_lib.kernel_time_ms(0, K)[0] / steps)
            res[generic]['dedicated_launches'] += _lib.kernel_time_ms(2, K)[1]
            L.dbw_timing_reset()
    L.dbw_debug_generic_blocks_loss(0)
    assert res[True]['dedicated_launches'] == 0 and res[False]['dedicated_launches'] > 0, res
    out = {}
    for generic, name in ((False, 'dedicated'), (True, 'generic')):
        out[name] = {k: spread(v) for k, v in res[generic].items() if k != 'dedicated_launches'}
    for k in ('blocks_pass_ms', 'step_ms'):
        out[f'{k}_saved'] = round(out['generic'][k]['median'] - out['dedicated'][k]['median'], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', nargs='+', default=['dtu', 'bmvs'], choices=['dtu', 'bmvs'])
    ap.add_argument('--repeat', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    c = card()
    for wl in args.workload:
        line = {'workload': wl, 'card': c, 'repeat': args.repeat, 'steps_per_run': args.steps}
        line.update(measure(wl, args.repeat, args.steps))
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
