"""Generates tests/golden/vgg_perceptual.npz: the reference's OWN `PerceptualLoss.forward` (src/model/loss.py) of a checkout of
monniert/differentiable-blocksworld named by DBW_REFERENCE, extracted with `ast` by tests/_refextract.py and run in float64
on the CPU on a stand-in object.  The reference's `__init__` downloads the ImageNet weights, so the stand-in builds what
it would: the ImageNet statistics as buffers and torchvision's `vgg16(weights=None).features` (with the seeded weights of
tests/_vgg_oracle.random_state_dict) cut [:4], [4:9], [9:16], [16:23], [23:30] into slice1 .. slice5.  It freezes the
images, the value and d value / d rec of every option set of tests/_vgg_oracle.OPTION_SETS at two shapes (2x37x53 floors
at every pool), and a checksum of the weights.  Only data is stored.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_vgg_perceptual_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from _refextract import extract_method, have_reference  # noqa: E402

WEIGHT_SEED = 0
SHAPES = ((2, 37, 53), (1, 16, 24))


def images(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g)
    return a, (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)


def weight_checksum(sd):
    """sum of |w| per convolution, in torchvision index order: the weights a test rebuilds are the frozen ones"""
    return np.array([float(v.double().abs().sum()) for k, v in sorted(sd.items(), key=lambda kv: kv[0]) if k.startswith('slice')])


class StandIn(torch.nn.Module):
    """what the reference's PerceptualLoss.__init__ builds, without its download"""

    def __init__(self, sd, normalize_input=True, normalize_features=True, feature_levels=None, sum_channels=False):
        super().__init__()
        from torchvision.models import vgg16
        self.normalize_input = normalize_input
        self.normalize_features = normalize_features
        self.sum_channels = sum_channels
        self.feature_levels = feature_levels if feature_levels is not None else [3]
        self.max_level = max(self.feature_levels)
        self.register_buffer('mean_rgb', torch.Tensor([0.485, 0.456, 0.406]))
        self.register_buffer('std_rgb', torch.Tensor([0.229, 0.224, 0.225]))
        layers = vgg16(weights=None).features
        self.slice1, self.slice2, self.slice3, self.slice4, self.slice5 = \
            layers[:4], layers[4:9], layers[9:16], layers[16:23], layers[23:30]
        self.load_state_dict(sd, strict=True)
        for p in self.parameters():
            p.requires_grad = False


def ref_vgg_perceptual_golden():
    assert have_reference()
    from _vgg_oracle import OPTION_SETS, random_state_dict
    forward = extract_method('src/model/loss.py', 'PerceptualLoss', 'forward')
    sd = random_state_dict(WEIGHT_SEED)
    data = {'weight_checksum': weight_checksum(sd)}
    meta = dict(weight_seed=WEIGHT_SEED, shapes=SHAPES, cases=[])
    for s, (B, H, W) in enumerate(SHAPES):
        imgs, rec = images(B, H, W, 100 + s)
        data[f's{s}__imgs'], data[f's{s}__rec'] = imgs.numpy(), rec.numpy()
        for name, kw in OPTION_SETS.items():
            mod = StandIn(sd, **kw).double()
            x = rec.double().requires_grad_(True)
            v = forward(mod, imgs.double(), x)
            v.backward()
            data[f's{s}__{name}__value'] = np.array(v.item())
            data[f's{s}__{name}__grad'] = x.grad.numpy().astype(np.float32)
            meta['cases'].append(dict(shape=s, name=name, kwargs=kw))
    data['meta'] = np.array(json.dumps(meta))
    return data


if __name__ == '__main__':
    if not have_reference():
        sys.exit('DBW_REFERENCE names no reference checkout')
    out = ref_vgg_perceptual_golden()
    path = os.path.join(HERE, 'vgg_perceptual.npz')
    np.savez_compressed(path, **out)
    print('wrote vgg_perceptual.npz', len(out), 'arrays,', os.path.getsize(path), 'bytes')
