"""Restatement of LPIPS (lpips 0.1.4, LPIPS(net='vgg', version='0.1'), as recalled) for the tests of csrc/dbw_lpips.cu.

The trunk is torchvision's `vgg16(weights=None).features[0:30]` (the right architecture; the weights come from an
lpips-named state dict), the heads are restated from lpips: f / (||f||_2 + 1e-10) per pixel, the squared difference, the
dropout mask, the 1x1 lin conv, the spatial mean, the taps summed.  Plain torch, any dtype and device; the tests run it on
the CPU in float64, in two modes:

  exact   every product and sum in the working precision;
  tf32    the convolutions of layers 1..12 (64..512 channels, the tensor-core layers) round both operands as the kernels
          do (round to nearest, ties away from zero, at bit 13 of the float32 value), in the forward and in the input
          gradient (the incoming gradient and the flipped weights), and accumulate in the working precision.  The first
          layer and its input gradient are fp32 FMA in the kernels and are not rounded here.

`mask_np` restates the dropout hash of csrc/dbw_lpips_hash.cuh in numpy."""
import functools

import numpy as np
import torch
import torch.nn.functional as F

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
TAP_AFTER = (3, 8, 15, 22, 29)          # features indices of relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
_M32 = 0xffffffff


# ------------------------------------------------------------------------------------------------ dropout hash
def _fmix(h):
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x85ebca6b)
    h = h ^ (h >> np.uint32(13))
    h = h * np.uint32(0xc2b2ae35)
    return h ^ (h >> np.uint32(16))


def hash_image(seed, tap, image):
    s = np.asarray([(int(seed) + 0x9e3779b9 * (int(tap) + 1)) & _M32], np.uint32)
    return _fmix(_fmix(s) ^ np.uint32(image))[0]


def mask_np(seed, tap, B, C, H, W, images=None):
    """(B,C,H,W) float64 dropout mask of one tap: 2 where the element is kept, 0 where dropped; with `images` (indices
    into the batch), only those images' masks, (len(images),C,H,W)"""
    images = range(B) if images is None else images
    with np.errstate(over='ignore'):
        out = np.empty((len(images), C, H, W))
        c = np.arange(C, dtype=np.uint32)[:, None, None]
        yx = (np.arange(H, dtype=np.uint32)[:, None] << np.uint32(16)) | np.arange(W, dtype=np.uint32)[None, :]
        for i, b in enumerate(images):
            h = _fmix(_fmix(np.uint32(hash_image(seed, tap, b)) ^ c) ^ yx[None])
            out[i] = np.where(h < np.uint32(0x80000000), 2.0, 0.0)
    return out


def masks(seed, shapes):
    """the five taps' masks for the tap shapes [(B,C,H,W)] * 5"""
    return [torch.from_numpy(mask_np(seed, k, *s)) for k, s in enumerate(shapes)]


# ------------------------------------------------------------------------------------------------ TF32
def tf32(t):
    """round as the kernels round an fp32 operand (the value is first taken to float32)"""
    b = t.to(torch.float32).contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32).to(t.dtype)


class _Tf32Conv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        wr = tf32(w)
        ctx.save_for_backward(wr)
        return F.conv2d(tf32(x), wr, b, padding=1)

    @staticmethod
    def backward(ctx, g):
        (wr,) = ctx.saved_tensors
        return F.conv2d(tf32(g), wr.flip(2, 3).transpose(0, 1), None, padding=1), None, None


def conv(x, w, b, mode, first=False):
    if mode == 'tf32' and not first:
        return _Tf32Conv.apply(x, w, b)
    return F.conv2d(x, w, b, padding=1)


def conv_abs_bound(x, w, b):
    """sum_k |a_k b_k| (+ |bias|) per output element: the scale of the fp32 accumulation error of one convolution"""
    return F.conv2d(x.abs(), w.abs(), None if b is None else b.abs(), padding=1)


# ------------------------------------------------------------------------------------------------ heads
class _SafeSqrt(torch.autograd.Function):
    """sqrt whose gradient at 0 is 0 (the kernels drop the norm's gradient term of an all-zero feature vector)"""
    @staticmethod
    def forward(ctx, x):
        r = x.sqrt()
        ctx.save_for_backward(r)
        return r

    @staticmethod
    def backward(ctx, g):
        (r,) = ctx.saved_tensors
        return torch.where(r > 0, g / (2 * r), torch.zeros_like(g))


def normalize_tensor(f, eps=1e-10):
    return f / (_SafeSqrt.apply((f * f).sum(1, keepdim=True)) + eps)


@functools.lru_cache(maxsize=1)
def _arch():
    """('conv' | 'relu' | 'pool') of each module of torchvision's vgg16 features[0:30]"""
    from torchvision.models import vgg16
    kind = {torch.nn.Conv2d: 'conv', torch.nn.ReLU: 'relu', torch.nn.MaxPool2d: 'pool'}
    return tuple(kind[type(m)] for m in vgg16(weights=None).features[:30])


def features(sd, x, normalize, mode='exact', dtype=torch.float64, channels_last=False):
    """the five taps of one image batch (B,3,H,W), in `dtype`, on x's device (sd is best already there: its tensors are
    moved on every call otherwise)"""
    dev = x.device
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    x = x.to(dtype).contiguous(memory_format=fmt)
    if normalize:
        x = 2 * x - 1
    x = (x - sd['scaling_layer.shift'].to(dev, dtype)) / sd['scaling_layer.scale'].to(dev, dtype)
    taps = []
    slice_of = {0: 1, 2: 1, 5: 2, 7: 2, 10: 3, 12: 3, 14: 3, 17: 4, 19: 4, 21: 4, 24: 5, 26: 5, 28: 5}
    for i, m in enumerate(_arch()):
        if m == 'conv':
            k = f'net.slice{slice_of[i]}.{i}.'
            x = conv(x, sd[k + 'weight'].to(dev, dtype).contiguous(memory_format=fmt), sd[k + 'bias'].to(dev, dtype), mode,
                     first=(i == 0))
        elif m == 'relu':
            x = F.relu(x)
        else:
            x = F.max_pool2d(x, 2, 2)
        if i in TAP_AFTER:
            taps.append(x)
    return taps


def lpips(sd, in0, in1, normalize=True, mode='exact', seed=None, dtype=torch.float64, channels_last=False):
    """per-image value (B,) of LPIPS(in0, in1); seed None: eval (no dropout), else the training mask of that seed.
    Differentiable in in1 (pass it with requires_grad)."""
    f0 = features(sd, in0.detach(), normalize, mode, dtype, channels_last)
    f1 = features(sd, in1, normalize, mode, dtype, channels_last)
    ms = masks(seed, [tuple(f.shape) for f in f1]) if seed is not None else None
    val = 0
    for k in range(5):
        d = (normalize_tensor(f0[k]) - normalize_tensor(f1[k])) ** 2
        if ms is not None:
            d = d * ms[k].to(d.device, dtype)
        w = sd[f'lin{k}.model.1.weight'].to(d.device, dtype)
        val = val + F.conv2d(d, w).mean((2, 3))
    return val[:, 0]


def value_and_grad(sd, in0, in1, normalize=True, mode='exact', seed=None, grad_value=None, dtype=torch.float64):
    """(value (B,), d sum_b grad_value[b] value[b] / d in1) on the CPU in float64 by default"""
    x = in1.detach().to(dtype).requires_grad_(True)
    v = lpips(sd, in0.detach().to(dtype), x, normalize, mode, seed, dtype)
    g = torch.ones_like(v) if grad_value is None else grad_value.to(v)
    (v * g).sum().backward()
    return v.detach(), x.grad


def random_state_dict(seed=0):
    """lpips-named weights: torchvision's default conv init (seeded) and |randn| lin weights (lpips's are >= 0)"""
    from torchvision.models import vgg16
    torch.manual_seed(seed)
    feats = vgg16(weights=None).features
    sd = {'scaling_layer.shift': torch.tensor(SHIFT)[None, :, None, None],
          'scaling_layer.scale': torch.tensor(SCALE)[None, :, None, None]}
    slice_of = {0: 1, 2: 1, 5: 2, 7: 2, 10: 3, 12: 3, 14: 3, 17: 4, 19: 4, 21: 4, 24: 5, 26: 5, 28: 5}
    for i, s in slice_of.items():
        sd[f'net.slice{s}.{i}.weight'] = feats[i].weight.detach().clone()
        # torchvision zeroes the biases; small random ones exercise the bias path of the kernels
        sd[f'net.slice{s}.{i}.bias'] = 0.02 * torch.randn(feats[i].bias.shape)
    for k, c in enumerate((64, 128, 256, 512, 512)):
        sd[f'lin{k}.model.1.weight'] = torch.randn(1, c, 1, 1).abs()
        sd[f'lins.{k}.model.1.weight'] = sd[f'lin{k}.model.1.weight']
    return sd
