"""Generates tests/golden/vgg_bits.npz on a GPU: the values and d value / d rec of perceptual.PerceptualLoss.per_image for
every option set of tests/_vgg_oracle.OPTION_SETS on fixed inputs, as the checkout this script sits in computes them.
Frozen from the build before the VGG feature loss and LPIPS shared one host pipeline in csrc/dbw_lpips.cu, so
tests/test_vgg_bits_gpu.py can check that the VGG term still gives the same bits.  Only data is stored.

    python tests/golden/make_vgg_bits_golden.py [out.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

# (B, H, W): 37x53 floors at every pool
SHAPE = (2, 37, 53)


def inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g)
    return a, (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)


def vgg_bits():
    from dbw_b200.perceptual import PerceptualLoss
    from tests import _vgg_oracle as OV
    dev = torch.device('cuda:0')
    sd = OV.random_state_dict(0)
    B, H, W = SHAPE
    data = {}
    for i, (name, opts) in enumerate(OV.OPTION_SETS.items()):
        m = PerceptualLoss.from_state_dict(sd, **opts).to(dev)
        a, b = inputs(B, H, W, 700 + i)
        x = b.to(dev).requires_grad_(True)
        v = m.per_image(a.to(dev), x)
        (v * torch.linspace(0.5, 1.5, B, device=dev)).sum().backward()
        data[f'{name}__value'], data[f'{name}__grad'] = v.detach().cpu().numpy(), x.grad.cpu().numpy()
    return data


if __name__ == '__main__':
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'vgg_bits.npz')
    data = vgg_bits()
    np.savez_compressed(out, **data)
    print('wrote', out, len(data), 'arrays,', os.path.getsize(out), 'bytes')
