"""Generates tests/golden/lpips_bits.npz on a GPU: LPIPS values and d value / d in1 of perceptual.LPIPS on fixed inputs, as
the checkout this script sits in computes them.  Frozen from the build before the VGG feature loss joined
csrc/dbw_lpips.cu (this file copied into a built checkout of that commit), so tests/test_vgg_perceptual_gpu.py can check
that the LPIPS kernels it shares still give the same bits.  Only data is stored.

    python tests/golden/make_lpips_bits_golden.py [out.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

# (B, H, W, normalize, train)
CASES = ((2, 37, 50, True, False), (2, 37, 50, True, True), (1, 64, 96, False, False))


def inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g)
    return a, (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)


def run(net, B, H, W, normalize, train, i):
    dev = net.prepared.device if net.prepared.numel() else torch.device('cuda:0')
    a, b = inputs(B, H, W, 500 + i)
    net.train(train)
    net.seed.fill_(4321)
    x = b.to(dev).requires_grad_(True)
    v = net(a.to(dev), x, normalize=normalize).flatten()
    (v * torch.linspace(0.5, 1.5, B, device=dev)).sum().backward()
    return v.detach().cpu().numpy(), x.grad.cpu().numpy()


def lpips_bits():
    from oracle import lpips as OL
    from dbw_b200.perceptual import LPIPS
    net = LPIPS.from_state_dict(OL.random_state_dict(0)).to(torch.device('cuda:0'))
    data = {}
    for i, c in enumerate(CASES):
        data[f'c{i}__value'], data[f'c{i}__grad'] = run(net, *c, i)
    return data


if __name__ == '__main__':
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'lpips_bits.npz')
    data = lpips_bits()
    np.savez_compressed(out, **data)
    print('wrote', out, len(data), 'arrays,', os.path.getsize(out), 'bytes')
