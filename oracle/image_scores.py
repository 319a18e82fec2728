"""float64 restatement of the evaluation's image scores as the reference writes them (src/model/loss.py:28-29,119-156):
`gaussian`, `SSIMLoss(padding=False)` -- one 2-D 11x11 window conv2d per moment, valid borders -- and
`mse2psnr(nn.MSELoss()(imgs, rec))`.  Test infrastructure only (tests/ and scripts/); the product never imports it.

The window's values are the reference's float32 ones (`gaussian` builds them with math.exp in double, converts them to
float32 and normalises them by their float32 sum); everything after that is float64."""
from math import exp

import torch
import torch.nn.functional as F

C1, C2 = 0.01 ** 2, 0.03 ** 2


def gaussian(window_size=11, sigma=1.5):
    """the reference's 1-D window, float32"""
    gauss = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                         dtype=torch.float32)
    return gauss / gauss.sum()


def window_2d(window_size=11, channel=3):
    """SSIMLoss.create_window: the outer product of the 1-D window, one copy per channel, float64"""
    g = gaussian(window_size, 1.5).double().unsqueeze(1)
    return g.mm(g.t()).expand(channel, 1, window_size, window_size).contiguous()


def ssim_map(img1, img2, window_size=11):
    """SSIMLoss(padding=False).ssim before its `1 -`: the (B, C, H - 10, W - 10) SSIM map, float64"""
    img1, img2 = img1.double(), img2.double()
    C = img1.shape[1]
    w = window_2d(window_size, C).to(img1.device)
    conv = lambda t: F.conv2d(t, w, groups=C)
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(img1 * img1) - mu1_sq
    sigma2_sq = conv(img2 * img2) - mu2_sq
    sigma12 = conv(img1 * img2) - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))


def ssim(img1, img2):
    """(B,) per-image mean SSIM: 1 - SSIMLoss(padding=False)(img1, img2)"""
    return ssim_map(img1, img2).flatten(1).mean(1)


def se_sum(imgs, rec):
    """(B,) per-image sum of squared errors, float64"""
    return (imgs.double() - rec.double()).pow(2).flatten(1).sum(1)


def mse2psnr(x):
    return -10. * torch.log10(x)


def psnr(imgs, rec):
    """mse2psnr(nn.MSELoss()(imgs, rec)): the PSNR of the whole batch's mean squared error"""
    return mse2psnr((imgs.double() - rec.double()).pow(2).mean())
