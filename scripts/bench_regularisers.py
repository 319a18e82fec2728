"""What the three regularisers (parsimony, total variation, overlap) cost, as the library's kernels (losses.regularisers) against
the PyTorch statement of the same terms (losses.parsimony / total_variation / overlap, the path CPU parameters take) called on
the device, alternating in one process:

  terms   the three terms alone, forward + backward to every leaf, with the shipped weights (parsimony 0.01, tv 0.1,
          overlap 1), at dtu (10 blocks, 256^2 maps, 256^2 background) and gundam_50 (50 blocks, 128^2 maps, 256^2 background):
          device time per call (CUDA events over --iters calls), kernel launches per call (torch.profiler, every CUDA kernel,
          the library's and torch's) and the peak device memory a call adds
  step    one graph.GraphedStep(optimizer=optim.BucketAdam) training iteration of the scene model with the shipped loss
          weights and no perceptual network, coarse phase, at 4 views x 300x400 and 49 views x 400x400: host wall time per
          iteration ending in a device synchronise, and the peak device memory of building and running the step; `rgb_only`
          is the same step with the RGB term alone, for scale

Medians, minima and maxima of --repeat alternating repeats.  One GPU; prints one JSON line with the card's name and power limit.

    python scripts/bench_regularisers.py [--iters 100] [--warmup 10] [--repeat 5]
"""
import argparse
import json
import os
import sys
import time
from copy import deepcopy

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_camera_grad import CFG, SHAPES, card  # noqa: E402

WEIGHTS = {'parsimony': 0.01, 'tv': 0.1, 'overlap': 1.0}
SCENES = {'dtu': (10, 256, 1), 'gundam_50': (50, 128, 2)}
STEP_LOSS = {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1}


def torch_regularisers(texture_bkg, texture_ground, textures, S, R_6d, T, sq_eps, alpha_full, weights, tv_type, coarse, ratio,
                       scale_min, generator=None, unit_samples=None):
    """losses.regularisers' signature over the PyTorch terms: what compute_losses computes from the leaves on the CPU path"""
    from dbw_b200 import geometry as G
    from dbw_b200 import losses as L
    out = {}
    if 'parsimony' in weights:
        out['parsimony'] = weights['parsimony'] * L.parsimony(alpha_full, coarse)
    if 'tv' in weights:
        out['tv'] = weights['tv'] * L.total_variation(torch.sigmoid(texture_bkg), torch.sigmoid(texture_ground), torch.sigmoid(textures),
                                                      L.TV_NORMS[tv_type], coarse)
    if 'overlap' in weights:
        eps = sq_eps.sigmoid() * 1.8 + 0.1
        out['overlap'] = weights['overlap'] * L.overlap(S.exp() + scale_min, G.rotation_6d_to_matrix(R_6d), T, eps[:, :1], eps[:, 1:],
                                                        alpha_full, ratio, coarse, generator=generator, unit_samples=unit_samples)
    return out


def terms_call(impl, scene, dev):
    from dbw_b200 import losses as L
    N, TS, up = SCENES[scene]
    g = torch.Generator().manual_seed(1)
    q = {'texture_bkg': torch.randn(1, TS * up, TS * up, 3, generator=g) / 10, 'texture_ground': torch.randn(1, TS * up, TS * up, 3, generator=g) / 10,
         'textures': torch.randn(N, TS, TS, 3, generator=g) / 10, 'S': (torch.rand(N, 3, generator=g) + 0.3).log(),
         'R_6d': torch.randn(N, 6, generator=g), 'T': torch.randn(N, 3, generator=g) * 0.1, 'sq_eps': torch.zeros(N, 2),
         'alpha_logit': torch.rand(N, generator=g) * 4 - 1}
    q = {k: v.to(dev).requires_grad_(True) for k, v in q.items()}
    u01 = torch.rand(N, 1000, 3, generator=g).to(dev)
    fn = L.regularisers if impl == 'kernels' else torch_regularisers
    leaves = list(q.values())

    def call():
        alpha_full = torch.sigmoid(q['alpha_logit'])
        out = fn(q['texture_bkg'], q['texture_ground'], q['textures'], q['S'], q['R_6d'], q['T'], q['sq_eps'], alpha_full, WEIGHTS,
                 'l2sq', True, 0.25, 0.2, unit_samples=u01)
        return torch.autograd.grad(sum(out.values()), leaves)
    return call


def kernels_per_call(call):
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    n = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'memcpy' not in e.name.lower()
            and 'memset' not in e.name.lower())
    return n / 5


def peak_added(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def stats(xs):
    xs = sorted(xs)
    return {'median': xs[len(xs) // 2], 'min': xs[0], 'max': xs[-1]}


def measure_terms(scene, iters, warmup, repeat, dev):
    calls, res = {}, {}
    for impl in ('torch', 'kernels'):
        calls[impl] = terms_call(impl, scene, dev)
        _, mib = peak_added(calls[impl])
        res[impl] = {'kernels_per_call': kernels_per_call(calls[impl]), 'peak_added_mib': mib}
        for _ in range(warmup):
            calls[impl]()
    times = {impl: [] for impl in calls}
    for _ in range(repeat):
        for impl, call in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(iters):
                call()
            b.record()
            torch.cuda.synchronize()
            times[impl].append(a.elapsed_time(b) / iters)
    for impl in calls:
        res[impl]['call_ms'] = stats(times[impl])
    return res


def build_step(mode, shape, dev):
    from dbw_b200 import losses as L
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.synthetic import ring_cameras
    B, H, W = SHAPES[shape]
    cfg = deepcopy(CFG)
    cfg['loss'] = {'rgb_weight': 1} if mode == 'rgb_only' else dict(STEP_LOSS)
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **cfg).to(dev).train()
    R, T, K = ring_cameras(B)
    inp = {'imgs': torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev), 'R': R.to(dev), 'T': T.to(dev),
           'K': K[None].expand(B, -1, -1).contiguous().to(dev)}
    opt = create_optimizer({'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}, model)
    kept = L.regularisers
    if mode == 'torch':
        L.regularisers = torch_regularisers          # captured into this step's graph; restored right after
    try:
        step = GraphedStep(ViewParallel(model, seed=1), inp, B, warmup=1, optimizer=opt)
    finally:
        L.regularisers = kept
    return step.run


def measure_steps(shape, iters, warmup, repeat, dev):
    runs, res = {}, {}
    for mode in ('rgb_only', 'torch', 'kernels'):
        runs[mode], mib = peak_added(lambda: build_step(mode, shape, dev))
        res[mode] = {'peak_added_mib': mib}
        for _ in range(warmup):
            runs[mode]()
    times = {m: [] for m in runs}
    for _ in range(repeat):
        for mode, run in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                run()
            torch.cuda.synchronize()
            times[mode].append((time.perf_counter() - t0) * 1e3 / iters)
    for mode in runs:
        res[mode]['iteration_ms'] = stats(times[mode])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--repeat', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    name, limit = card()
    res = {'card': name, 'power_limit_w': limit, 'iters': args.iters, 'warmup': args.warmup, 'repeat': args.repeat,
           'not_measured': ['two GPUs', 'the step with the LPIPS term']}
    dev = torch.device('cuda:0')
    for scene in SCENES:
        res[f'terms {scene}'] = measure_terms(scene, args.iters, args.warmup, args.repeat, dev)
        torch.cuda.empty_cache()
    for shape in ('train', 'dtu'):
        B, H, W = SHAPES[shape]
        res[f'step {B} x {H}x{W}'] = measure_steps(shape, args.iters, args.warmup, args.repeat, dev)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
