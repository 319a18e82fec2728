"""What the scoring stage of `quantitative_eval` costs on the GPU: the final_scores.tsv columns of the scene model (10 blocks,
the bench.py scene) over a loader, two ways, alternating in one process:

  pool    the previous path: Renderer.forward(viz_purpose=True) renders at 4H x 4W and F.avg_pool2d resolves it, SSIM is
          losses.ssim (eager separable convolutions), and every batch reads its five scores back to the host
  kernel  quantitative_eval: Renderer.render_viz resolves the 4x4 samples in the raster kernel, PSNR and SSIM come from the
          image-score kernel (dbw_b200.metrics), and the scores stay on the device until one read at the end

Two loaders, batch 4: 49 views at 400x400 (DTU) and 64 views at 576x768 (BlendedMVS), random targets.  Per loader and arm:
the time of one pass over the loader (CUDA-synchronised wall clock, median of --repeat) and the peak device memory above
what the model and the loader hold.  --check asserts that both arms give the same scores: L_tot and L_rec within 1e-6
relative, PSNR within 1e-5 dB and SSIM within 1e-5.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_image_scores.py [--repeat 5] [--check]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time
from collections import OrderedDict
from copy import deepcopy

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LOADERS = {'dtu': (49, 400, 400), 'bmvs': (64, 576, 768)}
BATCH = 4
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


@torch.no_grad()
def pool_eval(model, loader, device):
    """the scoring loop quantitative_eval ran before the image-score kernel (no perceptual term installed: LPIPS is NaN)"""
    from dbw_b200 import losses as L
    model.eval()
    opacities = model.get_opacities()
    scene = model.build_scene(filter_transparent=True)
    sums, count = dict(L_tot=0.0, L_rec=0.0, PSNR=0.0, SSIM=0.0, LPIPS=0.0), 0
    for inp, labels in loader:
        model._install_cameras(inp)
        imgs, n = inp['imgs'], len(inp['imgs'])
        rec = model.renderer(scene.extend(n), inp['R'], inp['T'], viz_purpose=True, K=model._view_K(inp))[:, :3]
        losses = model.compute_losses(imgs, rec)
        sums['L_tot'] += float(losses['total']) * n
        sums['L_rec'] += float(sum(losses[k] for k in ('rgb', 'perceptual') if k in losses)) * n
        sums['PSNR'] += float(-10.0 * torch.log10(F.mse_loss(imgs, rec))) * n
        sums['SSIM'] += float(L.ssim(imgs, rec).mean()) * n
        sums['LPIPS'] += float('nan') * n
        count += n
    return OrderedDict([('n_blocks', int((opacities > 0.5).sum()))] + [(k, v / max(count, 1)) for k, v in sums.items()]
                       + [(f'alpha{k}', a.item()) for k, a in enumerate(opacities)])


def kernel_eval(model, loader, device):
    return model.quantitative_eval(loader, device, hard_inference=True)


def timed(fn, *args):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out = fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base, out


def measure(name, repeat, check):
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.synthetic import ring_cameras
    dev = torch.device('cuda')
    N, H, W = LOADERS[name]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).eval()
    R, T, K = ring_cameras(N)
    g = torch.Generator().manual_seed(2)
    imgs = torch.rand(N, 3, H, W, generator=g).to(dev)
    K = K[None].expand(N, -1, -1).to(dev)
    loader = [({'imgs': imgs[i:i + BATCH], 'R': R[i:i + BATCH].to(dev), 'T': T[i:i + BATCH].to(dev), 'K': K[i:i + BATCH]}, {})
              for i in range(0, N, BATCH)]
    arms = {'pool': pool_eval, 'kernel': kernel_eval}
    res = {a: {'s': [], 'peak': 0} for a in arms}
    scores = {a: fn(model, loader, dev) for a, fn in arms.items()}        # warm-up of every shape either arm launches
    for _ in range(repeat):
        for a, fn in arms.items():
            s, peak, _ = timed(fn, model, loader, dev)
            res[a]['s'].append(s)
            res[a]['peak'] = max(res[a]['peak'], peak)
    out = {a: {'ms': round(1e3 * statistics.median(r['s']), 2), 'ms_min_max': [round(1e3 * min(r['s']), 2), round(1e3 * max(r['s']), 2)],
               'peak_device_mib': round(r['peak'] / 2 ** 20, 1)} for a, r in res.items()}
    out['views'], out['size'], out['batch'] = N, [H, W], BATCH
    if check:
        p, k = scores['pool'], scores['kernel']
        err = {c: abs(p[c] - k[c]) / (abs(p[c]) if c in ('L_tot', 'L_rec') else 1.0) for c in ('L_tot', 'L_rec', 'PSNR', 'SSIM')}
        out['check'] = {c: float(f'{e:.3e}') for c, e in err.items()}
        out['scores'] = {c: k[c] for c in ('L_tot', 'L_rec', 'PSNR', 'SSIM')}
        assert err['L_tot'] <= 1e-6 and err['L_rec'] <= 1e-6 and err['PSNR'] <= 1e-5 and err['SSIM'] <= 1e-5, err
        assert p['n_blocks'] == k['n_blocks'] and math.isnan(p['LPIPS']) and math.isnan(k['LPIPS'])
        assert [p[f'alpha{i}'] for i in range(10)] == [k[f'alpha{i}'] for i in range(10)]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--repeat', type=int, default=5)
    ap.add_argument('--check', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_image_scores.py needs a GPU')
    gpu, power = card()
    res = {'card': gpu, 'power_limit_w': power}
    for name in LOADERS:
        res[name] = measure(name, args.repeat, args.check)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
