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
change of the weights drops it."""
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


class LPIPS(nn.Module):
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
        self.register_buffer('prepared', torch.zeros(0), persistent=False)
        self._prepared_key = None
        self._target_cache = None

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_state_dict(cls, sd):
        """from an lpips-named state dict; a `perceptual_loss.loss.` or `module.` prefix is stripped.  Either of the
        `lin{k}` / `lins.{k}` spellings suffices.  Raises on a missing or misshapen key."""
        sd = dict(sd)
        for prefix in ('module.', 'perceptual_loss.loss.'):
            if any(k.startswith(prefix) for k in sd):
                sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
        for k in range(5):
            a, b = f'lin{k}.model.1.weight', f'lins.{k}.model.1.weight'
            if a not in sd and b in sd:
                sd[a] = sd[b]
            if b not in sd and a in sd:
                sd[b] = sd[a]
        shapes = state_dict_shapes()
        missing = [k for k in shapes if k not in sd]
        if missing:
            raise KeyError(f'LPIPS.from_state_dict: missing keys {missing}')
        bad = [(k, tuple(sd[k].shape), s) for k, s in shapes.items() if tuple(sd[k].shape) != s]
        if bad:
            raise ValueError(f'LPIPS.from_state_dict: misshapen keys (key, got, want) {bad}')
        m = cls()
        m.load_state_dict({k: sd[k] for k in shapes}, strict=True)
        return m

    @classmethod
    def from_files(cls, vgg16_pth, lin_pth):
        """from torchvision's vgg16 state dict (`features.N.weight` / `.bias`) and lpips's `weights/v0.1/vgg.pth`
        (`lin{k}.model.1.weight`)"""
        vgg = torch.load(vgg16_pth, map_location='cpu', weights_only=True)
        lin = torch.load(lin_pth, map_location='cpu', weights_only=True)
        sd = {'scaling_layer.shift': torch.tensor(SHIFT)[None, :, None, None],
              'scaling_layer.scale': torch.tensor(SCALE)[None, :, None, None]}
        for s, i, _, _ in CONVS:
            for n in ('weight', 'bias'):
                if f'features.{i}.{n}' not in vgg:
                    raise KeyError(f'LPIPS.from_files: {vgg16_pth} lacks features.{i}.{n}')
                sd[f'net.slice{s}.{i}.{n}'] = vgg[f'features.{i}.{n}']
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

    def _weights(self):
        convs = self.net.convs()
        return ([c.weight for c in convs], [c.bias for c in convs], [getattr(self, f'lin{k}').model[1].weight for k in range(5)])

    def _net_struct(self):
        ws, bs, ls = self._weights()
        net = _lib.DbwLpipsNet()
        for i in range(13):
            net.conv_w[i], net.conv_b[i] = ws[i].data_ptr(), bs[i].data_ptr()
        for k in range(5):
            net.lin_w[k] = ls[k].data_ptr()
        net.shift, net.scale = self.scaling_layer.shift.data_ptr(), self.scaling_layer.scale.data_ptr()
        net.prepared = self.prepared.data_ptr()
        return net

    def _prepare(self):
        """(re)write the TF32 forward and input-gradient weight copies when a weight tensor was replaced or modified"""
        ws, bs, ls = self._weights()
        params = ws + bs + ls + [self.scaling_layer.shift, self.scaling_layer.scale]
        key = tuple((p.data_ptr(), p._version) for p in params)
        if key == self._prepared_key:
            return
        for p in params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise DbwError('LPIPS: weights must be contiguous CUDA float32 tensors (call .cuda() on the module)')
        nbytes = self._bytes(1, 16, 16)[1]
        if self.prepared.numel() * 4 != nbytes or self.prepared.device != ws[0].device:
            self.prepared = torch.empty(nbytes // 4, dtype=torch.float32, device=ws[0].device)
        check(_lib.lib().dbw_lpips_prepare_weights(ctypes.byref(self._net_struct()), _stream(ws[0].device)),
              'dbw_lpips_prepare_weights')
        self._prepared_key = key

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
        if in0.requires_grad:
            raise DbwError('LPIPS: in0 requires a gradient; only in1 (the rendering) is differentiated')
        if not (in0.is_cuda and in1.is_cuda):
            raise DbwError('LPIPS: expected CUDA tensors (there is no CPU fallback)')
        if in0.dtype != torch.float32 or in1.dtype != torch.float32:
            raise DbwError(f'LPIPS: expected float32 images, got {in0.dtype} / {in1.dtype}')
        if in0.shape != in1.shape or in1.dim() != 4 or in1.shape[1] != 3:
            raise DbwError(f'LPIPS: expected two (B,3,H,W) images of one shape, got {tuple(in0.shape)} / {tuple(in1.shape)}')
        if min(in1.shape[2:]) < 16:
            raise DbwError(f'LPIPS: H and W must be >= 16 (relu5_3 at least 1x1), got {tuple(in1.shape[2:])}')
        self._prepare()
        # rec's activations are kept only when a backward can follow (not under no_grad, as in quantitative_eval)
        save = torch.is_grad_enabled() and in1.requires_grad
        return _LpipsFunction.apply(in0.contiguous(), in1.contiguous(), self, bool(normalize), bool(self.training), save,
                                    self._usable_cache(in0, normalize))
