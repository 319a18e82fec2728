"""Generates tests/golden/image_scores.npz: the reference's OWN `gaussian`, `SSIMLoss` and `mse2psnr` (src/model/loss.py) of
a checkout of monniert/differentiable-blocksworld named by DBW_REFERENCE, extracted with `ast` by tests/_refextract.py and
run in float32 on the CPU, as its evaluation calls them: `SSIMLoss(padding=False)(imgs, rec)` (per image) and
`mse2psnr(nn.MSELoss()(imgs, rec))` (per batch).  The image pairs are regenerated from their seeds by `pairs()`; only the
results and a checksum of each pair are stored.  They cover 11x11, odd sizes, 40x48 and 300x400, identical pairs (SSIM = 1),
near-constant images (where C1 and C2 dominate) and random and correlated pairs.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_image_scores_golden.py
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from _refextract import extract, have_reference  # noqa: E402

OUT = os.path.join(HERE, 'image_scores.npz')

# name: (B, H, W, kind, seed)
CASES = {
    'rand_11x11': (3, 11, 11, 'random', 1),
    'rand_13x17': (2, 13, 17, 'random', 2),
    'corr_37x29': (2, 37, 29, 'correlated', 3),
    'rand_40x48': (2, 40, 48, 'random', 4),
    'corr_40x48': (4, 40, 48, 'correlated', 5),
    'same_40x48': (2, 40, 48, 'identical', 6),
    'flat_40x48': (2, 40, 48, 'flat', 7),
    'flat_apart_23x31': (2, 23, 31, 'flat_apart', 8),
    'corr_300x400': (2, 300, 400, 'correlated', 9),
}


def pairs(name):
    """the float32 (imgs, rec) of a case, (B,3,H,W) in [0, 1]"""
    B, H, W, kind, seed = CASES[name]
    g = np.random.default_rng(seed)
    u = lambda: g.random((B, 3, H, W))
    if kind == 'random':
        x, y = u(), u()
    elif kind == 'correlated':                    # a blurred-looking target and a noisy reconstruction of it
        x = u()
        x = (x + np.roll(x, 1, 2) + np.roll(x, 1, 3) + np.roll(x, (1, 1), (2, 3))) / 4
        y = np.clip(x + 0.08 * (u() - 0.5) + 0.03, 0, 1)
    elif kind == 'identical':
        x = u()
        y = x
    elif kind == 'flat':                          # sigma ~ 1e-3: the C2 term dominates
        x, y = 0.5 + 2e-3 * (u() - 0.5), 0.5 + 2e-3 * (u() - 0.5)
    elif kind == 'flat_apart':                    # two nearly constant levels: C1 and C2 both matter
        x, y = 0.2 + 1e-3 * u(), 0.75 + 1e-3 * u()
    else:
        raise KeyError(kind)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)), torch.from_numpy(np.ascontiguousarray(y, np.float32))


def checksum(x, y):
    return np.float64([x.double().sum().item(), y.double().sum().item()])


def main():
    if not have_reference():
        print('DBW_REFERENCE is not a reference checkout: tests/golden/image_scores.npz left untouched')
        return
    ns = extract('src/model/loss.py', {'gaussian', 'SSIMLoss', 'mse2psnr'}, extra_ns={'exp': math.exp, 'nn': torch.nn})
    ssim_loss, mse = ns['SSIMLoss'](padding=False), torch.nn.MSELoss()
    out = {'window': ns['gaussian'](11, 1.5).numpy()}
    for name in CASES:
        x, y = pairs(name)
        out[f'{name}/ssim_loss'] = ssim_loss(x, y).numpy()
        out[f'{name}/psnr'] = ns['mse2psnr'](mse(x, y)).numpy()
        out[f'{name}/checksum'] = checksum(x, y)
    np.savez_compressed(OUT, **out)
    print(f'wrote {OUT}: {len(CASES)} cases')


if __name__ == '__main__':
    main()
