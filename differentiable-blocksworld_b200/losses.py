"""Parameter-only regularisers of the DBW objective (what the reference's src/model/dbw.py:373-405 adds to the pixel
terms): they never touch an image, so they are view-independent and (in a multi-GPU step) identical on every rank
(parallel.py divides them by the world size).  On CUDA parameters the three run in the library's kernels (regularisers():
two launches forward, at most two backward, deterministic); the per-term functions below are the PyTorch statement of the
same function and the path CPU parameters take."""
import ctypes

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


class _RegularisersFn(torch.autograd.Function):
    """dbw_regularisers_forward / _backward: the weighted terms that are on, one 0-d tensor each, in the order parsimony, tv,
    overlap.  The inputs no term that is on reads are None.  The gradients are written whole by the backward (no zero-fill)."""

    @staticmethod
    def forward(ctx, cfg, tex_bkg, tex_ground, textures, S, R_6d, T, sq_eps, alpha_full, unit_samples):
        from . import _lib
        from .renderer import _c, _stream
        ins = [t.detach().contiguous().float() if t is not None else None
               for t in (tex_bkg, tex_ground, textures, S, R_6d, T, sq_eps, alpha_full, unit_samples)]
        r = _lib.DbwRegularisers(*[t.data_ptr() if t is not None else None for t in ins], **cfg)
        ws_bytes = ctypes.c_size_t(0)
        _lib.check(_lib.lib().dbw_regularisers_workspace_bytes(ctypes.byref(r), ctypes.byref(ws_bytes)), 'dbw_regularisers_workspace_bytes')
        dev = next(t.device for t in ins if t is not None)
        ws = torch.empty(max(ws_bytes.value, 1), dtype=torch.uint8, device=dev)
        on = [bit for bit in (_lib.REG_PARSIMONY, _lib.REG_TV, _lib.REG_OVERLAP) if cfg['terms'] & bit]
        outs = {bit: torch.empty((), dtype=torch.float32, device=dev) for bit in on}
        _lib.check(_lib.lib().dbw_regularisers_forward(ctypes.byref(r), *[_c(outs.get(bit)) for bit in (1, 2, 4)], _c(ws), ws.numel(),
                                                       _stream()), 'dbw_regularisers_forward')
        ctx.save_for_backward(*[t for t in ins if t is not None])
        ctx.present = [t is not None for t in ins]
        ctx.cfg, ctx.on, ctx.device = cfg, on, dev
        return tuple(outs[bit] for bit in on)

    @staticmethod
    def backward(ctx, *g_outs):
        from . import _lib
        from .renderer import _c, _stream
        saved = iter(ctx.saved_tensors)
        ins = [next(saved) if p else None for p in ctx.present]
        r = _lib.DbwRegularisers(*[t.data_ptr() if t is not None else None for t in ins], **ctx.cfg)
        g_up = {bit: g.detach().contiguous().float() for bit, g in zip(ctx.on, g_outs)}
        grads = [torch.empty_like(t) if t is not None and need else None for t, need in zip(ins[:8], ctx.needs_input_grad[1:9])]
        ws_bytes = ctypes.c_size_t(0)
        _lib.check(_lib.lib().dbw_regularisers_workspace_bytes(ctypes.byref(r), ctypes.byref(ws_bytes)), 'dbw_regularisers_workspace_bytes')
        ws = torch.empty(max(ws_bytes.value, 1), dtype=torch.uint8, device=ctx.device)
        _lib.check(_lib.lib().dbw_regularisers_backward(ctypes.byref(r), *[_c(g_up.get(bit)) for bit in (1, 2, 4)],
                                                        *[_c(g) for g in grads], _c(ws), ws.numel(), _stream()),
                   'dbw_regularisers_backward')
        return (None, *grads, None)


def regularisers(texture_bkg, texture_ground, textures, S, R_6d, T, sq_eps, alpha_full, weights, tv_type, coarse, ratio,
                 scale_min, generator=None, unit_samples=None):
    """{name: weight * term} for each of 'parsimony', 'tv', 'overlap' in `weights`, computed by the library's kernels from the
    leaf parameters (S, R_6d and sq_eps as the model holds them: log-scales, 6D rotations, exponent logits; alpha_full the
    opacities of the opacity path) -- the same function as parsimony(), total_variation() and overlap() of the maps and poses
    the model derives from them.  In the fine phase parsimony and overlap are zeros, as there.  The overlap points come from
    `unit_samples` or are drawn here exactly as overlap() draws them."""
    from . import _lib
    coarse = bool(coarse)
    terms = 0
    if 'tv' in weights:
        terms |= _lib.REG_TV
    if coarse and 'parsimony' in weights:
        terms |= _lib.REG_PARSIMONY
    u01 = None
    if coarse and 'overlap' in weights:
        terms |= _lib.REG_OVERLAP
        N = S.shape[0]
        u01 = unit_samples if unit_samples is not None else torch.rand(N, OVERLAP_N_POINTS, 3, device=S.device, generator=generator)
    if textures.shape[1] != textures.shape[2] or texture_bkg.shape[1:] != texture_ground.shape[1:] \
            or texture_bkg.shape[1] != texture_bkg.shape[2]:
        raise ValueError('regularisers: the texture maps must be square, the background and the ground of one size')
    cfg = dict(n_blocks=S.shape[0], n_points=u01.shape[1] if u01 is not None else 0, env_size=texture_bkg.shape[1],
               txt_size=textures.shape[1], terms=terms, tv_norm=_lib.REG_TV_NORMS[tv_type], coarse=int(coarse),
               ratio_block_scene=float(ratio), scale_min=float(scale_min), w_parsimony=float(weights.get('parsimony', 0.)),
               w_tv=float(weights.get('tv', 0.)), w_overlap=float(weights.get('overlap', 0.)))
    # only what a term that is on reads enters the autograd graph: the fine phase's backward reaches S, R_6d, T, sq_eps and
    # the opacities no more than the PyTorch terms' does
    tv, ov, par = terms & _lib.REG_TV, terms & _lib.REG_OVERLAP, terms & _lib.REG_PARSIMONY
    ins = [t if on else None for t, on in zip((texture_bkg, texture_ground, textures, S, R_6d, T, sq_eps, alpha_full),
                                              (tv, tv, tv, ov, ov, ov, ov, ov or par))]
    outs = iter(_RegularisersFn.apply(cfg, *ins, u01) if terms else ())
    got = {}
    for name, bit in (('parsimony', _lib.REG_PARSIMONY), ('tv', _lib.REG_TV), ('overlap', _lib.REG_OVERLAP)):
        if name in weights:
            got[name] = next(outs) if terms & bit else weights[name] * alpha_full.new_zeros(())
    return got


def ssim(img1, img2, window_size=11, sigma=1.5):
    """mean structural similarity of two (B,C,H,W) images in [0,1] with the Gaussian window of the reference's evaluation
    (`SSIMLoss(padding=False)`, src/model/loss.py:113-155: 11 taps, sigma 1.5, C1 = 0.01^2, C2 = 0.03^2, 'valid' borders),
    evaluated separably (two 1-D passes per moment instead of one 11x11 pass).  Returns (B,) = mean SSIM per image.  The
    PyTorch statement of the evaluation's SSIM; quantitative_eval computes it on the device with metrics.ssim."""
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
