"""Times the LPIPS target cache (LPIPS.cache_targets) and prints one JSON line with the card's name and power limit:

  term   LPIPS forward + backward (d/d rec) at 4 x 300x400 (the DTU training batch) and 49 x 400x400 (the bench.py shape):
         no cache, a cache that holds every in0 image (all hits) and one that holds none of them (all misses), alternating
         in one process; CUDA events around whole calls
  step   one training step of the scene model at 4 x 300x400 (coarse phase, 10 blocks, LPIPS at weight 0.1): eager
         model(inp) + backward and a GraphedStep replay, each without and with the training images cached
  arena  the cache's device bytes per image and for 49 views, at 300x400, 400x400 and 576x768

Random LPIPS weights (oracle.lpips.random_state_dict): the kernels' time does not depend on the weights' values.

    python scripts/bench_lpips_cache.py [--repeat 20]
"""
import argparse
import json
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_lpips import card, timed  # noqa: E402


def term(B, H, W, repeat, sd):
    from dbw_b200.perceptual import LPIPS
    net = LPIPS.from_state_dict(sd).cuda().eval()
    g = torch.Generator().manual_seed(B)
    a = torch.rand(B, 3, H, W, generator=g).cuda()
    b = (a + 0.2 * torch.randn(B, 3, H, W, generator=g).cuda()).clamp(0, 1)
    others = torch.rand(B, 3, H, W, generator=g).cuda()

    def one():
        x = b.detach().requires_grad_(True)
        net(a, x, normalize=True).sum().backward()
    t = dict(no_cache=[], all_hits=[], all_misses=[])
    for _ in range(3):                                       # alternate
        for mode in t:
            net.clear_target_cache()
            torch.cuda.empty_cache()
            if mode != 'no_cache':
                net.cache_targets(a if mode == 'all_hits' else others)
            t[mode].append(timed(one, repeat))
    hits = int(net.target_hits.item())
    net.clear_target_cache()
    torch.cuda.empty_cache()
    return dict(shape=f'{B}x{H}x{W}', **{f'{k}_ms': round(min(v), 3) for k, v in t.items()}, last_hits=hits,
                cache_bytes=net.target_cache_bytes(H, W, B))


def step(repeat, sd):
    from oracle import dbw_path as D
    from dbw_b200.dbw import DifferentiableBlocksWorld, PerceptualTerm
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.perceptual import LPIPS
    cfg = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
           'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
           'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                          'decouple_rendering': True, 'opacity_noise': False},
           'loss': {'rgb_weight': 1, 'perceptual_weight': 0.1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1}}
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')                      # the lpips package is absent: the term starts dropped
        model = DifferentiableBlocksWorld((300, 400), **cfg).to(torch.device('cuda')).train()
    # two copies of the term: a graph captured with a cache reads its arena, so the cache stays registered throughout
    plain, cached = (PerceptualTerm(LPIPS.from_state_dict(sd)).cuda() for _ in range(2))
    model.set_perceptual_loss(plain)
    B = 4
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=1)
    g = torch.Generator().manual_seed(1)
    inp = {'imgs': torch.rand(B, 3, 300, 400, generator=g).cuda(), 'R': R.float().cuda(), 'T': T.float().cuda(),
           'K': K.float()[None].expand(B, -1, -1).cuda()}

    def eager():
        model.zero_grad(set_to_none=True)
        model(inp)['total'].backward()
    vp = ViewParallel(model, seed=5)
    graphed_plain = GraphedStep(vp, inp, B)
    model.set_perceptual_loss(cached)
    model.cache_perceptual_targets(inp['imgs'])
    graphed_cached = GraphedStep(vp, inp, B)
    t = dict(eager_no_cache=[], eager_cached=[], graphed_no_cache=[], graphed_cached=[])
    for _ in range(3):                                       # alternate
        model.set_perceptual_loss(plain)
        t['eager_no_cache'].append(timed(eager, repeat))
        model.set_perceptual_loss(cached)
        t['eager_cached'].append(timed(eager, repeat))
        t['graphed_no_cache'].append(timed(graphed_plain.run, repeat))
        t['graphed_cached'].append(timed(graphed_cached.run, repeat))
    return dict(shape=f'{B}x300x400', **{f'{k}_ms': round(min(v), 3) for k, v in t.items()},
                last_hits=int(cached.loss.target_hits.item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lpips_cache.py needs a GPU')
    from oracle import lpips as OL
    from dbw_b200.perceptual import LPIPS
    sd = OL.random_state_dict(0)
    name, watts = card()
    m = LPIPS()
    out = dict(card=name, power_limit_w=watts,
               arena={f'{H}x{W}': dict(bytes_per_image=m.target_cache_bytes(H, W), bytes_49_views=m.target_cache_bytes(H, W, 49))
                      for H, W in ((300, 400), (400, 400), (576, 768))})
    out['term'] = [term(4, 300, 400, args.repeat, sd), term(49, 400, 400, 3, sd)]
    out['step'] = step(max(3, args.repeat // 2), sd)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
