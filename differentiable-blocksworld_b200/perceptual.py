"""LPIPS (lpips 0.1.4, `LPIPS(net='vgg', version='0.1')`, as recalled; the package is not needed) on the sm_90a kernels of
csrc/dbw_lpips.cu: the perceptual term every shipped config weighs into the objective (`LPIPSLoss`,
src/model/loss.py:32-40 of the reference).

`LPIPS` carries lpips's own parameter and buffer names, so a reference checkpoint's `perceptual_loss.loss.*` entries load
into it unchanged.  Install it with

    model.set_perceptual_loss(PerceptualTerm(LPIPS.from_files('vgg16-397923af.pth', 'weights/v0.1/vgg.pth').cuda()))

Semantics (as recalled): with `normalize`, x -> 2x - 1; then (x - shift) / scale; torchvision's VGG16 features[0:30]
with the taps relu1_2 .. relu5_3; per tap and pixel f / (||f||_2 + 1e-10) for both images, the squared difference,
Dropout(0.5) and a 1x1 conv C -> 1 without bias, the spatial mean; the five taps summed, (B,1,1,1).  The dropout follows
the module's `training` flag, as in the reference (trainer.py calls model.train() every step): in training each
(image, tap, channel, pixel) element is kept with probability 1/2 and doubled, by a counter-based hash of a seed held in
a device buffer that the forward advances (csrc/dbw_lpips_hash.cuh; not torch's dropout stream).  The 64..512-channel
convolutions take TF32 operands and accumulate in fp32, as the reference's cuDNN convolutions do under torch 1.12's
default allow_tf32.  Gradients flow to `in1` only; CUDA float32 tensors only (no CPU fallback).

Target cache (opt in): `cache_targets(imgs)` computes the taps of fixed `in0` images (a scene's training views) once;
every later forward looks each `in0` image up on the device (a fingerprint, confirmed by comparing the whole image bit for
bit) and runs the VGG16 trunk of `in0` over the misses only.  Results are the uncached ones bit for bit, hits or not; the
caller never says which view is which.  A forward uses the cache when its `normalize` and (H, W) are the cache's; any
change of the weights drops it.

`PerceptualLoss` is the reference's other perceptual term, the VGG16 feature-reconstruction loss (`perceptual_name:
perceptual`), on the same trunk kernels (dbw_vgg_loss_* in csrc/dbw_lpips.cu)."""
import ctypes
from collections import OrderedDict

import torch
from torch import nn

from . import _lib
from ._lib import DbwError, check

# (slice, torchvision features index, C_in, C_out) of the 13 convolutions
CONVS = [(1, 0, 3, 64), (1, 2, 64, 64), (2, 5, 64, 128), (2, 7, 128, 128), (3, 10, 128, 256), (3, 12, 256, 256),
         (3, 14, 256, 256), (4, 17, 256, 512), (4, 19, 512, 512), (4, 21, 512, 512), (5, 24, 512, 512), (5, 26, 512, 512),
         (5, 28, 512, 512)]
TAP_CHANNELS = (64, 128, 256, 512, 512)
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def state_dict_shapes():
    """{key: shape} of an lpips vgg LPIPS state dict (the lin layers appear as lin{k} and as lins.{k}, one module each)"""
    shapes = OrderedDict([('scaling_layer.shift', (1, 3, 1, 1)), ('scaling_layer.scale', (1, 3, 1, 1))])
    for s, i, ci, co in CONVS:
        shapes[f'net.slice{s}.{i}.weight'] = (co, ci, 3, 3)
        shapes[f'net.slice{s}.{i}.bias'] = (co,)
    for k, c in enumerate(TAP_CHANNELS):
        shapes[f'lin{k}.model.1.weight'] = (1, c, 1, 1)
    for k, c in enumerate(TAP_CHANNELS):
        shapes[f'lins.{k}.model.1.weight'] = (1, c, 1, 1)
    return shapes


def tf32_round(t):
    """round float32 to TF32 as the kernels do: to nearest, ties away from zero, at bit 13 (low 13 bits cleared)"""
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def kmajor(w):
    """(C_out, C_in, 3, 3) -> the K-major GEMM operand (C_out, 9*C_in) ordered (ky, kx, ci), as dbw_lpips_conv3x3 takes it"""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def dgrad_weight(w):
    """the weight whose forward convolution is the input gradient of w: W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx]"""
    return w.flip(2, 3).transpose(0, 1).contiguous()


class _Lin(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.model = nn.Sequential(OrderedDict([('0', nn.Dropout()), ('1', nn.Conv2d(c, 1, 1, bias=False))]))


class _Scaling(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer('shift', torch.tensor(SHIFT)[None, :, None, None])
        self.register_buffer('scale', torch.tensor(SCALE)[None, :, None, None])


class _Vgg(nn.Module):
    def __init__(self):
        super().__init__()
        for s in range(1, 6):
            self.add_module(f'slice{s}', nn.Sequential(OrderedDict(
                (str(i), nn.Conv2d(ci, co, 3, padding=1)) for sl, i, ci, co in CONVS if sl == s)))

    def convs(self):
        return [getattr(getattr(self, f'slice{s}'), str(i)) for s, i, _, _ in CONVS]


class _LpipsFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in0, in1, mod, normalize, train, save, cache):
        B, _, H, W = in1.shape
        net = mod._net_struct()
        ws_bytes = mod._bytes(B, H, W, save)[0]
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=in1.device)
        value = torch.empty(B, dtype=torch.float32, device=in1.device)
        if cache is None:
            route = torch.empty(0, dtype=torch.int32, device=in1.device)
            check(_lib.lib().dbw_lpips_forward(ctypes.byref(net), _vp(in0), _vp(in1), B, H, W, int(normalize), int(train), int(save),
                                               _vp(mod.seed), _vp(value), _vp(ws), ws_bytes, _stream(in1.device)), 'dbw_lpips_forward')
        else:
            route = torch.empty(B, 2, dtype=torch.int32, device=in1.device)
            check(_lib.lib().dbw_lpips_forward_cached(ctypes.byref(net), ctypes.byref(cache.desc), _vp(in0), _vp(in1), B, H, W,
                                                      int(normalize), int(train), int(save), _vp(mod.seed), _vp(value), _vp(route),
                                                      _vp(cache.hits), _vp(ws), ws_bytes, _stream(in1.device)),
                  'dbw_lpips_forward_cached')
        # the cache object holds the arena the backward reads, even if the module's cache is replaced in between
        ctx.mod, ctx.flags, ctx.cache = mod, (int(normalize), int(train)), cache
        ctx.save_for_backward(ws, route)
        ctx.shape = in1.shape
        return value.view(B, 1, 1, 1)

    @staticmethod
    def backward(ctx, grad_value):
        ws, route = ctx.saved_tensors
        B, _, H, W = ctx.shape
        g = grad_value.reshape(B).to(torch.float32).contiguous()
        grad = torch.empty(ctx.shape, dtype=torch.float32, device=ws.device)
        net = ctx.mod._net_struct()
        if ctx.cache is None:
            check(_lib.lib().dbw_lpips_backward(ctypes.byref(net), _vp(g), B, H, W, ctx.flags[0], ctx.flags[1], _vp(grad), _vp(ws),
                                                ws.numel(), _stream(ws.device)), 'dbw_lpips_backward')
        else:
            check(_lib.lib().dbw_lpips_backward_cached(ctypes.byref(net), ctypes.byref(ctx.cache.desc), _vp(route), _vp(g), B, H, W,
                                                       ctx.flags[0], ctx.flags[1], _vp(grad), _vp(ws), ws.numel(),
                                                       _stream(ws.device)), 'dbw_lpips_backward_cached')
        return None, grad, None, None, None, None, None


class _TargetCache:
    """a registered target cache: the arena (device bytes), its C descriptor, the weights key it was computed with, and
    `hits`, a device int32 (1,) the cached forwards write their hit count to"""

    def __init__(self, arena, N, H, W, normalize, key):
        self.arena, self.N, self.H, self.W, self.normalize, self.key = arena, N, H, W, bool(normalize), key
        self.desc = _lib.DbwLpipsTargetCache(arena.data_ptr(), N, H, W, int(normalize))
        self.hits = torch.zeros(1, dtype=torch.int32, device=arena.device)


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _strip(sd, prefixes):
    """sd with each of `prefixes` that some key carries stripped, in order (the keys without it dropped)"""
    sd = dict(sd)
    for prefix in prefixes:
        if any(k.startswith(prefix) for k in sd):
            sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    return sd


class _Trunk(nn.Module):
    """What LPIPS and PerceptualLoss share: torchvision's VGG16 convolutions on the kernels of csrc/dbw_lpips.cu, their TF32
    copies in `prepared`, loading their weights, and the checks on the two images.  A subclass names its convolutions
    (`_convs`), its input transform (`_transform`) and its lin weights (`_lins`)."""

    def __init__(self):
        super().__init__()
        self.register_buffer('prepared', torch.zeros(0), persistent=False)
        self._prepared_key = None

    def _lins(self):
        return []

    @classmethod
    def _load(cls, sd, shapes, **options):
        """an instance holding sd's entries of `shapes`; raises on a missing or misshapen key"""
        missing = [k for k in shapes if k not in sd]
        if missing:
            raise KeyError(f'{cls.__name__}.from_state_dict: missing keys {missing}')
        bad = [(k, tuple(sd[k].shape), s) for k, s in shapes.items() if tuple(sd[k].shape) != s]
        if bad:
            raise ValueError(f'{cls.__name__}.from_state_dict: misshapen keys (key, got, want) {bad}')
        m = cls(**options)
        m.load_state_dict({k: sd[k] for k in shapes}, strict=True)
        return m

    @classmethod
    def _features(cls, vgg16_pth, prefix):
        """{prefix + 'slice{s}.{i}.weight' / '.bias': torchvision's `features.{i}.*`} of its vgg16 state dict"""
        vgg = torch.load(vgg16_pth, map_location='cpu', weights_only=True)
        sd = {}
        for s, i, _, _ in CONVS:
            for n in ('weight', 'bias'):
                if f'features.{i}.{n}' not in vgg:
                    raise KeyError(f'{cls.__name__}.from_files: {vgg16_pth} lacks features.{i}.{n}')
                sd[f'{prefix}slice{s}.{i}.{n}'] = vgg[f'features.{i}.{n}']
        return sd

    def _net_struct(self):
        net = _lib.DbwLpipsNet()
        for i, c in enumerate(self._convs()):
            net.conv_w[i], net.conv_b[i] = c.weight.data_ptr(), c.bias.data_ptr()
        for k, w in enumerate(self._lins()):
            net.lin_w[k] = w.data_ptr()
        shift, scale = self._transform()
        net.shift, net.scale = shift.data_ptr(), scale.data_ptr()
        net.prepared = self.prepared.data_ptr()
        return net

    def _prepare(self):
        """(re)write the TF32 forward and input-gradient weight copies when a weight tensor was replaced or modified"""
        convs = self._convs()
        params = [c.weight for c in convs] + [c.bias for c in convs] + self._lins() + list(self._transform())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if key == self._prepared_key:
            return
        for p in params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise DbwError(f'{type(self).__name__}: weights must be contiguous CUDA float32 tensors (call .cuda() on the module)')
        ws, prep = ctypes.c_size_t(0), ctypes.c_size_t(0)
        check(_lib.lib().dbw_lpips_workspace_bytes(1, 16, 16, 0, ctypes.byref(ws), ctypes.byref(prep)), 'dbw_lpips_workspace_bytes')
        dev = params[0].device
        if self.prepared.numel() * 4 != prep.value or self.prepared.device != dev:
            self.prepared = torch.empty(prep.value // 4, dtype=torch.float32, device=dev)
        check(_lib.lib().dbw_lpips_prepare_weights(ctypes.byref(self._net_struct()), _stream(dev)), 'dbw_lpips_prepare_weights')
        self._prepared_key = key

    def _check_images(self, target, rendering, names, min_hw, why):
        """target and rendering: (B,3,H,W) CUDA float32 images of one shape, H and W >= min_hw, target without a gradient"""
        who = type(self).__name__
        if target.requires_grad:
            raise DbwError(f'{who}: {names[0]} requires a gradient; only {names[1]} (the rendering) is differentiated')
        if not (torch.is_tensor(target) and torch.is_tensor(rendering) and target.is_cuda and rendering.is_cuda):
            raise DbwError(f'{who}: expected CUDA tensors (there is no CPU fallback)')
        if target.dtype != torch.float32 or rendering.dtype != torch.float32:
            raise DbwError(f'{who}: expected float32 images, got {target.dtype} / {rendering.dtype}')
        if target.shape != rendering.shape or rendering.dim() != 4 or rendering.shape[1] != 3:
            raise DbwError(f'{who}: expected two (B,3,H,W) images of one shape, got {tuple(target.shape)} / {tuple(rendering.shape)}')
        if min(rendering.shape[2:]) < min_hw:
            raise DbwError(f'{who}: H and W must be >= {min_hw} {why}, got {tuple(rendering.shape[2:])}')


class LPIPS(_Trunk):
    """lpips.LPIPS(net='vgg', version='0.1') with the lin-layer dropout lpips builds by default; forward(in0, in1,
    normalize=False) -> (B,1,1,1).  `in0` must not require a gradient.  Build it with `from_state_dict` or `from_files`;
    a bare LPIPS() has torchvision's default random initialisation (tests only)."""

    def __init__(self):
        super().__init__()
        self.scaling_layer = _Scaling()
        self.net = _Vgg()
        for k, c in enumerate(TAP_CHANNELS):
            setattr(self, f'lin{k}', _Lin(c))
        self.lins = nn.ModuleList([getattr(self, f'lin{k}') for k in range(5)])
        for p in self.parameters():
            p.requires_grad_(False)
        # the dropout seed (uint32 bits in an int32), advanced on the device by every forward; not part of lpips's state
        self.register_buffer('seed', torch.zeros(1, dtype=torch.int32), persistent=False)
        self._target_cache = None

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_state_dict(cls, sd):
        """from an lpips-named state dict; a `perceptual_loss.loss.` or `module.` prefix is stripped.  Either of the
        `lin{k}` / `lins.{k}` spellings suffices.  Raises on a missing or misshapen key."""
        sd = _strip(sd, ('module.', 'perceptual_loss.loss.'))
        for k in range(5):
            a, b = f'lin{k}.model.1.weight', f'lins.{k}.model.1.weight'
            if a not in sd and b in sd:
                sd[a] = sd[b]
            if b not in sd and a in sd:
                sd[b] = sd[a]
        return cls._load(sd, state_dict_shapes())

    @classmethod
    def from_files(cls, vgg16_pth, lin_pth):
        """from torchvision's vgg16 state dict (`features.N.weight` / `.bias`) and lpips's `weights/v0.1/vgg.pth`
        (`lin{k}.model.1.weight`)"""
        sd = cls._features(vgg16_pth, 'net.')
        lin = torch.load(lin_pth, map_location='cpu', weights_only=True)
        sd.update({'scaling_layer.shift': torch.tensor(SHIFT)[None, :, None, None],
                   'scaling_layer.scale': torch.tensor(SCALE)[None, :, None, None]})
        for k in range(5):
            key = f'lin{k}.model.1.weight'
            if key not in lin:
                raise KeyError(f'LPIPS.from_files: {lin_pth} lacks {key}')
            sd[key] = lin[key]
        return cls.from_state_dict(sd)

    # ------------------------------------------------------------------ device plumbing
    def _bytes(self, B, H, W, save=True):
        ws, prep = ctypes.c_size_t(0), ctypes.c_size_t(0)
        check(_lib.lib().dbw_lpips_workspace_bytes(B, H, W, int(save), ctypes.byref(ws), ctypes.byref(prep)), 'dbw_lpips_workspace_bytes')
        return ws.value, prep.value

    def _convs(self):
        return self.net.convs()

    def _transform(self):
        return self.scaling_layer.shift, self.scaling_layer.scale

    def _lins(self):
        return [getattr(self, f'lin{k}').model[1].weight for k in range(5)]

    # ------------------------------------------------------------------ target cache
    def target_cache_bytes(self, H, W, N=1):
        """device bytes of a target cache of N images of H x W: their five taps in fp32, a copy of each image and its
        fingerprint (about 59.9 MB per 300x400 image, 221 MB per 576x768 one)"""
        b = ctypes.c_size_t(0)
        check(_lib.lib().dbw_lpips_cache_bytes(H, W, ctypes.byref(b)), 'dbw_lpips_cache_bytes')
        return N * b.value

    def cache_targets(self, imgs, normalize=True, chunk=8):
        """register (N,3,H,W) CUDA float32 target images, replacing any previous cache: later forwards with the same
        `normalize` and (H, W) read the taps of any `in0` image equal to one of them, bit for bit, from the cache instead of
        recomputing them.  `chunk` images are computed at a time.  A CUDA graph captured before this call keeps computing
        its targets, and one captured with a cache must be captured again after the cache is replaced or cleared."""
        if not (torch.is_tensor(imgs) and imgs.is_cuda and imgs.dtype == torch.float32 and imgs.dim() == 4 and imgs.shape[1] == 3):
            raise DbwError(f'LPIPS.cache_targets: expected (N,3,H,W) CUDA float32 images, got '
                           f'{tuple(imgs.shape) if torch.is_tensor(imgs) else type(imgs).__name__}')
        N, _, H, W = imgs.shape
        if N < 1 or min(H, W) < 16:
            raise DbwError(f'LPIPS.cache_targets: need N >= 1 and H, W >= 16, got {tuple(imgs.shape)}')
        self.clear_target_cache()
        self._prepare()
        dev = self.prepared.device
        imgs = imgs.detach().to(dev).contiguous()
        cache = _TargetCache(torch.empty(self.target_cache_bytes(H, W, N), dtype=torch.uint8, device=dev), N, H, W, normalize,
                             self._prepared_key)
        c = max(1, min(N, int(chunk)))
        ws = torch.empty(self._bytes(c, H, W, False)[0], dtype=torch.uint8, device=dev)
        check(_lib.lib().dbw_lpips_cache_targets(ctypes.byref(self._net_struct()), _vp(imgs), ctypes.byref(cache.desc), c, _vp(ws),
                                                 ws.numel(), _stream(dev)), 'dbw_lpips_cache_targets')
        self._target_cache = cache

    def clear_target_cache(self):
        """drop the target cache (its device memory is freed once no pending backward holds it)"""
        self._target_cache = None

    @property
    def target_hits(self):
        """device int32 (1,): the hit count of the last forward that used the cache (None without a cache); not synchronised"""
        return self._target_cache.hits if self._target_cache is not None else None

    def _usable_cache(self, in0, normalize):
        c = self._target_cache
        if c is None:
            return None
        if c.key != self._prepared_key:          # the weights changed since registration: never serve stale taps
            self._target_cache = None
            return None
        if c.normalize != bool(normalize) or (c.H, c.W) != tuple(in0.shape[2:]) or c.arena.device != in0.device:
            return None
        return c

    def forward(self, in0, in1, normalize=False):
        self._check_images(in0, in1, ('in0', 'in1'), 16, '(relu5_3 at least 1x1)')
        self._prepare()
        # rec's activations are kept only when a backward can follow (not under no_grad, as in quantitative_eval)
        save = torch.is_grad_enabled() and in1.requires_grad
        return _LpipsFunction.apply(in0.contiguous(), in1.contiguous(), self, bool(normalize), bool(self.training), save,
                                    self._usable_cache(in0, normalize))


# ------------------------------------------------------------------------------------------------ VGG feature loss
MEAN_RGB = (0.485, 0.456, 0.406)
STD_RGB = (0.229, 0.224, 0.225)


def vgg_loss_state_dict_shapes():
    """{key: shape} of the reference's PerceptualLoss state dict: the ImageNet statistics, then the 13 convolutions under
    their torchvision indices in the slices relu1_2 .. relu5_3 (all of them, whatever feature_levels is)"""
    shapes = OrderedDict([('mean_rgb', (3,)), ('std_rgb', (3,))])
    for s, i, ci, co in CONVS:
        shapes[f'slice{s}.{i}.weight'] = (co, ci, 3, 3)
        shapes[f'slice{s}.{i}.bias'] = (co,)
    return shapes


class _VggLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, imgs, rec, mod, save):
        B, _, H, W = rec.shape
        net, opt = mod._net_struct(), mod._options()
        ws_bytes = mod._bytes(B, H, W, save)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=rec.device)
        value = torch.empty(B, dtype=torch.float32, device=rec.device)
        check(_lib.lib().dbw_vgg_loss_forward(ctypes.byref(net), ctypes.byref(opt), _vp(imgs), _vp(rec), B, H, W, int(save), _vp(value),
                                              _vp(ws), ws_bytes, _stream(rec.device)), 'dbw_vgg_loss_forward')
        ctx.mod, ctx.opt, ctx.shape = mod, opt, rec.shape
        ctx.save_for_backward(ws)
        return value

    @staticmethod
    def backward(ctx, grad_value):
        (ws,) = ctx.saved_tensors
        B, _, H, W = ctx.shape
        g = grad_value.reshape(B).to(torch.float32).contiguous()
        grad = torch.empty(ctx.shape, dtype=torch.float32, device=ws.device)
        net = ctx.mod._net_struct()
        check(_lib.lib().dbw_vgg_loss_backward(ctypes.byref(net), ctypes.byref(ctx.opt), _vp(g), B, H, W, _vp(grad), _vp(ws), ws.numel(),
                                               _stream(ws.device)), 'dbw_vgg_loss_backward')
        return None, grad, None, None


class PerceptualLoss(_Trunk):
    """The reference's VGG16 feature-reconstruction loss (`PerceptualLoss`, src/model/loss.py:66-111; `perceptual_name:
    perceptual`) on the sm_90a kernels of csrc/dbw_lpips.cu.  forward(imgs, rec) -> scalar, differentiable in `rec` only:
    with `normalize_input`, (x - mean_rgb) / std_rgb; torchvision's VGG16 features only through the deepest of
    `feature_levels` (default [3], relu3_3; a level listed twice counts once); per requested level, optionally
    f / (||f||_2 over channels + 1e-10), the squared difference averaged over C*H*W (or, with `sum_channels`, summed over
    channels and averaged over pixels); the levels summed and the batch averaged.  The 64..512-channel convolutions take
    TF32 operands, as for LPIPS.  CUDA float32 tensors only (no CPU fallback).

    Its buffers and parameters carry the reference's names (`mean_rgb`, `std_rgb`, `slice{s}.{i}.weight` / `.bias`, all 13
    convolutions), so a reference checkpoint's `perceptual_loss.*` entries load into it.  Build it with `from_files`
    (torchvision's vgg16-397923af.pth) or `from_state_dict`; a bare PerceptualLoss() has torchvision's default random
    initialisation (tests only).  With several levels and `sum_channels` the reference's own forward fails to broadcast
    its per-row means; here the levels' values are summed as for the other options."""

    def __init__(self, normalize_input=True, normalize_features=True, feature_levels=None, sum_channels=False, requires_grad=False):
        super().__init__()
        if requires_grad:
            raise NotImplementedError('PerceptualLoss(requires_grad=True): the kernels give no gradient to the VGG weights')
        self.normalize_input = normalize_input
        self.normalize_features = normalize_features
        self.sum_channels = sum_channels
        self.feature_levels = feature_levels if feature_levels is not None else [3]
        if not isinstance(self.feature_levels, (list, tuple)) or not self.feature_levels \
                or any(k not in (1, 2, 3, 4, 5) for k in self.feature_levels):
            raise DbwError(f'PerceptualLoss: feature_levels must be a non-empty list of levels 1..5, got {feature_levels!r}')
        self.max_level = max(self.feature_levels)
        self.register_buffer('mean_rgb', torch.tensor(MEAN_RGB))
        self.register_buffer('std_rgb', torch.tensor(STD_RGB))
        vgg = _Vgg()
        for s in range(1, 6):
            self.add_module(f'slice{s}', getattr(vgg, f'slice{s}'))
        for p in self.parameters():
            p.requires_grad_(False)

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_state_dict(cls, sd, **options):
        """from a state dict with the reference's names; a `perceptual_loss.` or `module.` prefix is stripped.  Raises on a
        missing or misshapen key."""
        return cls._load(_strip(sd, ('module.', 'perceptual_loss.')), vgg_loss_state_dict_shapes(), **options)

    @classmethod
    def from_files(cls, vgg16_pth, **options):
        """from torchvision's vgg16 state dict (`features.N.weight` / `.bias`), the file LPIPS.from_files also reads"""
        sd = cls._features(vgg16_pth, '')
        sd.update({'mean_rgb': torch.tensor(MEAN_RGB), 'std_rgb': torch.tensor(STD_RGB)})
        return cls.from_state_dict(sd, **options)

    # ------------------------------------------------------------------ device plumbing
    def _options(self):
        levels = 0
        for k in self.feature_levels:
            levels |= 1 << (k - 1)
        return _lib.DbwVggLossOptions(levels, int(bool(self.normalize_input)), int(bool(self.normalize_features)),
                                      int(bool(self.sum_channels)))

    def _bytes(self, B, H, W, save=True):
        ws = ctypes.c_size_t(0)
        check(_lib.lib().dbw_vgg_loss_workspace_bytes(B, H, W, ctypes.byref(self._options()), int(save), ctypes.byref(ws)),
              'dbw_vgg_loss_workspace_bytes')
        return ws.value

    def _convs(self):
        return [getattr(getattr(self, f'slice{s}'), str(i)) for s, i, _, _ in CONVS]

    def _transform(self):
        return self.mean_rgb, self.std_rgb

    def per_image(self, imgs, rec):
        """(B,) float32: each image's value, whose batch mean forward() returns"""
        self._check_images(imgs, rec, ('imgs', 'rec'), 2 ** (self.max_level - 1), f'for level {self.max_level}')
        self._prepare()
        # rec's activations are kept only when a backward can follow (not under no_grad)
        save = torch.is_grad_enabled() and rec.requires_grad
        return _VggLossFunction.apply(imgs.contiguous(), rec.contiguous(), self, save)

    def forward(self, imgs, rec):
        return self.per_image(imgs, rec).mean()
