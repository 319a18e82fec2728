"""Times the VGG16 feature-reconstruction loss (perceptual.PerceptualLoss on dbw_vgg_loss_* of csrc/dbw_lpips.cu) and prints
one JSON line with the card's name and power limit:

  term     forward + backward (d/d rec) at 4 x 300x400 and 49 x 400x400, for the default relu3_3 and for all five levels;
           beside it the same term restated in torch (cuDNN, TF32, tests/_vgg_oracle.py in float32 with its weights
           resident on the GPU), NCHW and channels_last, alternating with the kernels in one process; and LPIPS at the
           same shape (its share is the measured counterpart of the 61 % of MACs per pixel that relu3_3 needs)
  step     a GraphedStep replay of the scene model at 4 x 300x400 (coarse phase, 10 blocks) with this term at weight 0.1,
           with LPIPS at weight 0.1, and with neither (the fused RGB loss epilogue)

--check compares the kernels' and cuDNN's value and gradient with the float64 oracle at 4 x 300x400.

    python scripts/bench_vgg_perceptual.py [--check] [--repeat 20]
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

LEVELS = {'relu3_3': [3], 'relu1_2..relu5_3': [1, 2, 3, 4, 5]}


def term(B, H, W, repeat, sd, lp_sd, check):
    from dbw_b200.perceptual import LPIPS, PerceptualLoss
    from tests import _vgg_oracle as OV
    sd_nchw = {k: v.cuda() for k, v in sd.items()}
    sd_cl = {k: v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v for k, v in sd_nchw.items()}
    g = torch.Generator().manual_seed(B)
    a = torch.rand(B, 3, H, W, generator=g)
    b = (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)
    a, b = a.cuda(), b.cuda()
    lpips = LPIPS.from_state_dict(lp_sd).cuda().eval()
    rows = []
    for name, levels in LEVELS.items():
        mod = PerceptualLoss.from_state_dict(sd, feature_levels=levels).cuda()

        def ours():
            x = b.detach().requires_grad_(True)
            v = mod.per_image(a, x)
            v.sum().backward()
            return v.detach(), x.grad

        def cudnn(channels_last=False):
            x = b.detach().requires_grad_(True)
            v = OV.vgg_perceptual(sd_cl if channels_last else sd_nchw, a, x, levels, mode='exact', dtype=torch.float32,
                                  channels_last=channels_last)
            v.sum().backward()
            return v.detach(), x.grad

        def lp():
            x = b.detach().requires_grad_(True)
            lpips(a, x, normalize=True).sum().backward()
        t = dict(ours=[], nchw=[], cl=[], lpips=[])
        for _ in range(3):                                   # alternate
            t['ours'].append(timed(ours, repeat))
            t['nchw'].append(timed(cudnn, repeat))
            t['cl'].append(timed(lambda: cudnn(True), repeat))
            t['lpips'].append(timed(lp, repeat))
        ms = {k: min(v) for k, v in t.items()}
        res = dict(shape=f'{B}x{H}x{W}', levels=name, ms=round(ms['ours'], 3), cudnn_nchw_ms=round(ms['nchw'], 3),
                   cudnn_channels_last_ms=round(ms['cl'], 3), lpips_ms=round(ms['lpips'], 3),
                   share_of_lpips=round(ms['ours'] / ms['lpips'], 3))
        if check:
            vo, go = ours()
            vc, gc = cudnn(True)
            vx, gx = OV.value_and_grad(sd_nchw, a, b, levels, mode='exact')
            rel = lambda u, w: float((u.double() - w).norm() / w.norm())
            res.update(value_rel_err=rel(vo, vx), grad_rel_err=rel(go, gx), cudnn_value_rel_err=rel(vc, vx),
                       cudnn_grad_rel_err=rel(gc, gx))
        print(json.dumps(res), file=sys.stderr)
        rows.append(res)
        del mod
        torch.cuda.empty_cache()
    return rows


def step(repeat, sd, lp_sd):
    """ms of a GraphedStep replay at 4 x 300x400 with this term, with LPIPS, and with no perceptual term"""
    from oracle import dbw_path as D
    from dbw_b200.dbw import DifferentiableBlocksWorld, PerceptualTerm
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.perceptual import LPIPS, PerceptualLoss
    cfg = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
           'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
           'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                          'decouple_rendering': True, 'opacity_noise': False},
           'loss': {'rgb_weight': 1, 'perceptual_weight': 0.1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1,
                    'perceptual_name': 'perceptual'}}
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')                      # no VGG16 weights in the hub cache: the term starts dropped
        model = DifferentiableBlocksWorld((300, 400), **cfg).to(torch.device('cuda')).train()
    B = 4
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=1)
    g = torch.Generator().manual_seed(1)
    inp = {'imgs': torch.rand(B, 3, 300, 400, generator=g).cuda(), 'R': R.float().cuda(), 'T': T.float().cuda(),
           'K': K.float()[None].expand(B, -1, -1).cuda()}
    vp = ViewParallel(model, seed=5)
    steps = {}
    for name, term in (('vgg_relu3_3', PerceptualLoss.from_state_dict(sd).cuda()),
                       ('lpips', PerceptualTerm(LPIPS.from_state_dict(lp_sd)).cuda()), ('none', None)):
        model.set_perceptual_loss(term)
        steps[name] = GraphedStep(vp, inp, B)
    t = {k: [] for k in steps}
    for _ in range(3):                                       # alternate
        for k, s in steps.items():
            t[k].append(timed(s.run, repeat))
    return dict(shape=f'{B}x300x400', **{f'graphed_{k}_ms': round(min(v), 3) for k, v in t.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true')
    ap.add_argument('--repeat', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_vgg_perceptual.py needs a GPU')
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    from oracle import lpips as OL
    from tests import _vgg_oracle as OV
    sd, lp_sd = OV.random_state_dict(0), OL.random_state_dict(0)
    name, watts = card()
    out = dict(card=name, power_limit_w=watts)
    out['term'] = term(4, 300, 400, max(3, args.repeat // 4), sd, lp_sd, args.check) + term(49, 400, 400, 3, sd, lp_sd, False)
    out['step'] = step(max(3, args.repeat // 2), sd, lp_sd)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
