"""Image scores of the evaluation (`quantitative_eval`, the reference's src/model/dbw.py:464-493): PSNR and SSIM of
rendered views against their targets, computed on the device by the library's kernels (csrc/dbw_metrics.cu, two launches
per batch, deterministic).  SSIM is the reference's SSIMLoss(padding=False) (src/model/loss.py:119-156): an 11x11
Gaussian window of sigma 1.5, C1 = 0.01^2, C2 = 0.03^2, valid borders.  There is no CPU fallback: CPU tensors raise.
`losses.ssim` is the PyTorch statement of the same SSIM."""
import ctypes
import math

import torch

from . import _lib
from ._lib import DbwError, check

WINDOW_SIZE, SIGMA = 11, 1.5


def _window():
    """the reference's gaussian(11, 1.5): math.exp in double, float32 values normalised by their float32 sum"""
    g = torch.tensor([math.exp(-(x - WINDOW_SIZE // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(WINDOW_SIZE)],
                     dtype=torch.float32)
    return (ctypes.c_float * WINDOW_SIZE)(*(g / g.sum()).tolist())


_WINDOW = _window()


def image_scores(imgs, rec):
    """(se_sum (B,), ssim (B,)) of two (B,3,H,W) CUDA float32 images, H and W >= 11, as device tensors: the per-view sum of
    (imgs - rec)^2 over its 3 H W values, and the per-view mean of the SSIM map (1 - SSIMLoss(padding=False)(imgs, rec))"""
    if imgs.dim() != 4 or imgs.shape[1] != 3 or imgs.shape[0] < 1 or rec.shape != imgs.shape:
        raise ValueError(f'image_scores: expected two (B,3,H,W) images of one shape, got {tuple(imgs.shape)} and {tuple(rec.shape)}')
    B, _, H, W = imgs.shape
    if H < WINDOW_SIZE or W < WINDOW_SIZE:
        raise ValueError(f'image_scores: H and W must be at least {WINDOW_SIZE} (the SSIM window), got {H}x{W}')
    if not (imgs.is_cuda and rec.is_cuda) or imgs.device != rec.device:
        raise DbwError('image_scores: expected CUDA tensors on one device (there is no CPU fallback)')
    if imgs.dtype != torch.float32 or rec.dtype != torch.float32:
        raise DbwError(f'image_scores: expected float32 images, got {imgs.dtype} / {rec.dtype}')
    imgs, rec = imgs.contiguous(), rec.contiguous()
    L = _lib.lib()
    se = torch.empty(B, dtype=torch.float32, device=imgs.device)
    ss = torch.empty(B, dtype=torch.float32, device=imgs.device)
    ws = torch.empty(L.dbw_image_scores_workspace_bytes(B, H, W), dtype=torch.uint8, device=imgs.device)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    check(L.dbw_image_scores(B, H, W, vp(imgs), vp(rec), _WINDOW, vp(se), vp(ss), vp(ws), ws.numel(),
                             ctypes.c_void_p(torch.cuda.current_stream(imgs.device).cuda_stream)), 'dbw_image_scores')
    return se, ss


def ssim(img1, img2):
    """(B,) mean SSIM per image: losses.ssim on the device"""
    return image_scores(img1, img2)[1]


def psnr(imgs, rec):
    """mse2psnr(nn.MSELoss()(imgs, rec)) = -10 log10 of the whole batch's mean squared error, a 0-d device tensor"""
    se, _ = image_scores(imgs, rec)
    return psnr_of(se, imgs[0].numel())


def psnr_of(se_sum, numel_per_view):
    """the batch PSNR from image_scores' per-view squared-error sums, in float64"""
    return -10.0 * torch.log10(se_sum.double().sum() / (se_sum.numel() * numel_per_view))
