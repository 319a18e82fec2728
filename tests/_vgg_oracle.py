"""Float64 restatement of the reference's VGG16 feature-reconstruction loss (`PerceptualLoss`, src/model/loss.py:66-111) for
the tests of dbw_vgg_loss_* (csrc/dbw_lpips.cu) and perceptual.PerceptualLoss.

The trunk is that of oracle/lpips.py (torchvision's vgg16 features, `conv` in its 'exact' or 'tf32' mode), run only
through the deepest requested level, with the ImageNet transform (x - mean_rgb) / std_rgb in place of lpips's scaling
layer.  Per requested level: optionally f / (||f||_2 + 1e-10) (oracle/lpips.py's normalize_tensor, whose norm has a zero
gradient at 0), the squared difference averaged over C*H*W, or summed over channels and averaged over pixels; the levels
summed.  Plain torch, any dtype and device."""
import torch
import torch.nn.functional as F

from oracle import lpips as OL

SLICE_OF = {0: 1, 2: 1, 5: 2, 7: 2, 10: 3, 12: 3, 14: 3, 17: 4, 19: 4, 21: 4, 24: 5, 26: 5, 28: 5}
MEAN_RGB = (0.485, 0.456, 0.406)
STD_RGB = (0.229, 0.224, 0.225)
# the reference's option sets the tests cover: name -> PerceptualLoss keyword arguments
OPTION_SETS = {
    'default': {},
    'levels_1_5': dict(feature_levels=[1, 2, 3, 4, 5]),
    'levels_2_4': dict(feature_levels=[2, 4]),
    'levels_3_3': dict(feature_levels=[3, 3]),
    'raw_features': dict(normalize_features=False),
    'sum_channels': dict(sum_channels=True),
    'raw_input': dict(normalize_input=False),
}


def options(normalize_input=True, normalize_features=True, feature_levels=None, sum_channels=False):
    """the keyword arguments of an option set, defaults filled in, levels as a sorted tuple without duplicates"""
    levels = tuple(sorted(set(feature_levels if feature_levels is not None else [3])))
    return dict(levels=levels, normalize_input=normalize_input, normalize_features=normalize_features, sum_channels=sum_channels)


def random_state_dict(seed=0):
    """PerceptualLoss-named weights: oracle/lpips.py's seeded torchvision initialisation with small random biases"""
    lp = OL.random_state_dict(seed)
    sd = {'mean_rgb': torch.tensor(MEAN_RGB), 'std_rgb': torch.tensor(STD_RGB)}
    for i, s in SLICE_OF.items():
        for n in ('weight', 'bias'):
            sd[f'slice{s}.{i}.{n}'] = lp[f'net.slice{s}.{i}.{n}']
    return sd


def level_features(sd, x, levels, normalize_input, mode='exact', dtype=torch.float64, channels_last=False):
    """{level k: the tap relu{k}_* of x (B,3,H,W)} for the requested levels, the trunk stopped at the deepest"""
    dev = x.device
    x = x.to(dtype).contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    if normalize_input:
        x = (x - sd['mean_rgb'].to(dev, dtype).view(1, 3, 1, 1)) / sd['std_rgb'].to(dev, dtype).view(1, 3, 1, 1)
    last = OL.TAP_AFTER[max(levels) - 1]
    taps = {}
    for i, m in enumerate(OL._arch()[:last + 1]):
        if m == 'conv':
            k = f'slice{SLICE_OF[i]}.{i}.'
            x = OL.conv(x, sd[k + 'weight'].to(dev, dtype), sd[k + 'bias'].to(dev, dtype), mode, first=(i == 0))
        elif m == 'relu':
            x = F.relu(x)
        else:
            x = F.max_pool2d(x, 2, 2)
        if i in OL.TAP_AFTER and OL.TAP_AFTER.index(i) + 1 in levels:
            taps[OL.TAP_AFTER.index(i) + 1] = x
    return taps


def vgg_perceptual(sd, imgs, rec, levels=(3,), normalize_input=True, normalize_features=True, sum_channels=False, mode='exact',
                   dtype=torch.float64, channels_last=False):
    """per-image value (B,) (the reference returns its batch mean); differentiable in rec"""
    levels = tuple(sorted(set(levels)))
    f0 = level_features(sd, imgs.detach(), levels, normalize_input, mode, dtype, channels_last)
    f1 = level_features(sd, rec, levels, normalize_input, mode, dtype, channels_last)
    val = 0
    for k in levels:
        a, b = f0[k], f1[k]
        if normalize_features:
            a, b = OL.normalize_tensor(a), OL.normalize_tensor(b)
        d = (a - b) ** 2
        val = val + (d.sum(1).mean((1, 2)) if sum_channels else d.mean((1, 2, 3)))
    return val


def value_and_grad(sd, imgs, rec, levels=(3,), normalize_input=True, normalize_features=True, sum_channels=False, mode='exact',
                   grad_value=None, dtype=torch.float64):
    """(value (B,), d sum_b grad_value[b] value[b] / d rec), in float64 by default"""
    x = rec.detach().to(dtype).requires_grad_(True)
    v = vgg_perceptual(sd, imgs.detach().to(dtype), x, levels, normalize_input, normalize_features, sum_channels, mode, dtype)
    g = torch.ones_like(v) if grad_value is None else grad_value.to(v)
    (v * g).sum().backward()
    return v.detach(), x.grad
