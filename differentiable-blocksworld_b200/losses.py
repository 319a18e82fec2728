"""Parameter-only regularisers of the DBW objective (what the reference's src/model/dbw.py:373-405 adds to the pixel
terms) as standalone functions: they never touch an image, so they stay plain PyTorch on the leaf parameters -- tiny,
view-independent, and (in a multi-GPU step) identical on every rank (parallel.py divides them by the world size)."""
import torch

from . import geometry as G

OVERLAP_N_POINTS = 1000        # samples per block for the overlap term (dbw.py:33)
OVERLAP_N_BLOCKS = 1.95        # more than ~2 blocks claiming a point is penalised (dbw.py:34)
OVERLAP_TEMPERATURE = 0.005    # softness of the inside/outside decision (dbw.py:35)

TV_NORMS = {
    'l2': lambda d: G.safe_pow(d.pow(2).sum(-1), 0.5),        # clamped at 1e-6 like loss.py:45: finite gradient at 0
    'l1': lambda d: d.abs().sum(-1),
    'l2sq': lambda d: d.pow(2).sum(-1),
}


def effective_opacities(alpha_full, coarse):
    """soft opacities while they are being learned, their 0/1 decision afterwards (dbw.py:375,402)"""
    return alpha_full if coarse else (alpha_full > 0.5).float()


def parsimony(alpha_full, coarse):
    """sqrt-opacity sparsity prior on the number of blocks (dbw.py:373-376); switched off in the fine phase"""
    if not coarse:
        return alpha_full.new_zeros(())
    return G.safe_pow(effective_opacities(alpha_full, coarse), 0.5).mean()


def _tv_map(maps, norm, wrap_u=False):
    """total variation of (M,H,W,3) maps along v and u; block maps are periodic in u (their u axis closes the sphere)"""
    dv = norm(maps[:, 1:] - maps[:, :-1])
    if wrap_u:
        du = norm(torch.roll(maps, shifts=-1, dims=2) - maps)
        return du.sum(0).mean() + dv.sum(0).mean()          # summed over blocks: every map receives the same gradient scale
    du = norm(maps[:, :, 1:] - maps[:, :, :-1])
    return dv.mean() + du.mean()


def total_variation(bkg_maps, ground_maps, block_maps, norm, coarse):
    """dbw.py:378-387: background + blocks at full weight, the ground at the phase factor (1 coarse, 0.1 fine); the whole
    term is scaled by the same factor again by the caller"""
    factor = 1.0 if coarse else 0.1
    tv = _tv_map(bkg_maps, norm)
    if block_maps is not None and len(block_maps) > 0:
        tv = tv + _tv_map(block_maps, norm, wrap_u=True)
    tv = tv + _tv_map(ground_maps, norm) * factor
    return tv * factor


def overlap(S, R, T, eps1, eps2, alpha_full, ratio, coarse, generator=None, unit_samples=None):
    """dbw.py:389-405: sample points inside every block's bounding box, count (softly, opacity-weighted) how many
    superquadrics contain each of them, penalise counts above OVERLAP_N_BLOCKS.  Off in the fine phase.
    unit_samples: pre-drawn U(0,1) samples (N, OVERLAP_N_POINTS, 3) used instead of drawing here (CUDA-graph capture)."""
    if not coarse:
        return alpha_full.new_zeros(())
    N = S.shape[0]
    with torch.no_grad():
        u01 = unit_samples if unit_samples is not None else torch.rand(N, OVERLAP_N_POINTS, 3, device=S.device, generator=generator)
        pts = u01 * 2 - 1
        pts = torch.bmm(pts * ratio * S[:, None], R) + T[:, None]              # into the scene frame
        pts = pts.reshape(1, -1, 3).expand(N, -1, -1)
    local = torch.bmm(pts - T[:, None], R.transpose(1, 2)) / (S[:, None] * ratio)  # every point in every block's frame
    sdf = G.superquadric_implicit(local, eps1, eps2)
    occupancy = torch.sigmoid(-sdf / OVERLAP_TEMPERATURE) * effective_opacities(alpha_full, coarse)[:, None]
    return (occupancy.sum(0) - OVERLAP_N_BLOCKS).clamp(min=0).mean()


def ssim(img1, img2, window_size=11, sigma=1.5):
    """mean structural similarity of two (B,C,H,W) images in [0,1] with the Gaussian window of the reference's evaluation
    (`SSIMLoss(padding=False)`, src/model/loss.py:113-155: 11 taps, sigma 1.5, C1 = 0.01^2, C2 = 0.03^2, 'valid' borders),
    evaluated separably (two 1-D passes per moment instead of one 11x11 pass).  Returns (B,) = mean SSIM per image."""
    C = img1.shape[1]
    x = torch.arange(window_size, dtype=img1.dtype, device=img1.device) - window_size // 2
    g = torch.exp(-x.pow(2) / (2 * sigma ** 2))
    g = g / g.sum()
    kh, kv = g.view(1, 1, 1, -1).expand(C, 1, 1, -1), g.view(1, 1, -1, 1).expand(C, 1, -1, 1)
    blur = lambda t: torch.nn.functional.conv2d(torch.nn.functional.conv2d(t, kh, groups=C), kv, groups=C)
    mu1, mu2 = blur(img1), blur(img2)
    s11, s22, s12 = blur(img1 * img1) - mu1 * mu1, blur(img2 * img2) - mu2 * mu2, blur(img1 * img2) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s11 + s22 + c2))
    return smap.flatten(1).mean(1)
