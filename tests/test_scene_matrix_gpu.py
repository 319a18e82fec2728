"""GPU: every entry point of csrc/dbw_scene.cu against a float64 autograd oracle, element by element.

The oracle evaluates the same float32 inputs in float64 with oracle/dbw_path.py's pieces (parametric_sq, the 6D rotation,
SceneTemplate.to_world / _decimate / build_env / build_blocks, circular F.pad, sigmoid).  Every output gets random cotangents
and every leaf gradient is compared element by element:
  * geometry -- scene_geometry_passes and the raw C-ABI entries: icosphere levels 1-3 and one vertex per
    block (the backward's 64-thread stride loop), 0 .. 300 blocks with and without a ground, exponents from cube-like to
    pinched (the ln|x| terms at the poles), log-scales -5 .. 3, unnormalised 6D vectors of magnitude 1e-3 .. 1e3, a posed world;
  * opacities -- block_opacities and the raw entries: up to 1000 blocks x 300 faces, saturating logits, each upstream gradient
    NULL on its own, keep decisions and face map exact;
  * texture preparation -- the four stages in 1-4 job launches, sizes that are not multiples of the 32 x 8 CTA tile, padding up
    to the whole map, environment maps larger and smaller than the blocks', logits up to +-90, CELLS4 gradients at any float
    offset of a larger buffer;
  * the model chain -- DifferentiableBlocksWorld._scene_tensors in each training phase against build_env / build_blocks.

Bars are fractions of each array's largest magnitude, BAR_FACTOR times what the oracle's own float32 evaluation shows against
float64 over the same cases (tests/test_scene_matrix_host.py checks that on the CPU).  All outputs are prefilled with NaN: the
kernels write every element ("written, not accumulated", include/dbw_render.h).

This module is importable without a GPU: the host module reuses its case tables and oracle."""
import ctypes
import json
import math
import os
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import dbw_path as D
from oracle import pt3d

pytestmark = pytest.mark.gpu

BAR_FACTOR = 8
# Each bar is about BAR_FACTOR times the worst deviation of the oracle's own float32 evaluation from float64 over this module's
# cases (fraction of each array's largest magnitude; tests/test_scene_matrix_host.py measures it on the CPU and keeps the two
# consistent).  Bars above 2e-6 are explained in BAR_NOTES.
BARS = {
    'geom.verts': 1e-5, 'geom.sq_eps': 2.5e-5, 'geom.sq_eps+6': 2e-4, 'geom.S': 1e-5, 'geom.R_6d': 2.5e-5, 'geom.T': 2e-6,
    'geom.R_6d_ground': 3e-6, 'geom.T_ground': 2e-6,
    'opacity.alpha': 7e-7, 'opacity.g_logit': 3e-6,
    'tex.out': 4e-6, 'tex.grad': 5e-6,
    'chain.env_verts': 1.2e-6, 'chain.env_atlas': 2.5e-6, 'chain.blk_verts': 1.5e-6, 'chain.atlas': 3e-6, 'chain.alpha': 5e-7,
    'chain.sq_eps': 2.5e-6, 'chain.S': 2e-6, 'chain.R_6d': 2e-6, 'chain.T': 8e-7, 'chain.R_6d_ground': 2e-6,
    'chain.T_ground': 5e-6, 'chain.alpha_logit': 2e-6, 'chain.texture_bkg': 2.5e-6, 'chain.texture_ground': 3e-6,
    'chain.textures': 2.5e-6,
}
BAR_NOTES = {
    'geom.verts': 'log-scales up to 3 make a few blocks 400x larger than others; the rounding of the small ones is measured '
                  'against the largest, after five float32 products and sums (superquadric, scale, rotation, world transform)',
    'geom.sq_eps': 'd/d eps sums sign(x)|x|^e ln|x| over the vertices, with terms of both signs that cancel (up to -3x the '
                   'upstream gradient at the poles where cos(eta) = -4.4e-8 and e = 0.1)',
    'geom.sq_eps+6': 'at sq_eps = 6 the exponent is 1.9 and d e / d eps = 1.8 s (1 - s) with s = sigmoid(6) = 0.9975: 1 - s '
                     'keeps only the last 13 bits of s in float32 (the oracle and the kernel compute it the same way)',
    'geom.S': 'as geom.verts: gradients of exp(S) for S in [-5, 3] span 3.5 decades within one array',
    'geom.R_6d': 'the 6D vectors span 1e-3 .. 1e3, so the rotation gradients (~1/|a|) span six decades; random vector pairs '
                 'include nearly parallel ones, whose Gram-Schmidt step loses bits to cancellation',
    'geom.R_6d_ground': 'the ground has 81 vertices whose rotation gradients cancel in a sum over the plane',
    'opacity.g_logit': 'a (1 - a) loses bits to cancellation as logits saturate (the oracle and the kernel alike)',
    'tex.out': 'an 8x8 cell is the float32 mean of 64 sigmoids',
    'tex.grad': 's (1 - s) of the sigmoid loses bits to cancellation as logits saturate (logits up to +-90)',
    'chain.env_atlas': 'as tex.out', 'chain.atlas': 'as tex.out', 'chain.texture_bkg': 'as tex.grad',
    'chain.texture_ground': 'as tex.grad', 'chain.textures': 'as tex.grad', 'chain.sq_eps': 'as geom.sq_eps',
    'chain.T_ground': 'the ground translation gradient sums 81 vertex gradients of '
                                                                 'both signs',
}

WORST = {}          # bar name -> worst error / bar seen in this session (written out when DBW_SCENE_MATRIX_REPORT names a file)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    path = os.environ.get('DBW_SCENE_MATRIX_REPORT')
    if path:
        with open(path, 'w') as f:
            json.dump({k: {'worst_rel_err': v, 'bar': BARS[k]} for k, v in sorted(WORST.items())}, f, indent=1)


def rel_err(got, want):
    """max |got - want| over max |want| (0 when both are all zero, inf when only `got` is not)"""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (got.shape, want.shape)
    if got.numel() == 0:
        return 0.
    err, scale = (got - want).abs().max().item(), want.abs().max().item()
    if not math.isfinite(err):
        return math.inf
    return err / scale if scale > 0 else (0. if err == 0 else math.inf)


def check(bar, got, want, what=''):
    e = rel_err(got, want)
    WORST[bar] = max(WORST.get(bar, 0.), e)
    assert e <= BARS[bar], f'{bar} {what}: max error {e:.3g} of max |oracle| > bar {BARS[bar]:.3g}'


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _uniform(g, shape, lo, hi):
    return torch.rand(shape, generator=g) * (hi - lo) + lo


# ---------------------------------------------------------------------------------------------------------- geometry
# (name, n_blocks, icosphere level (0: one vertex per block, picked at random, poles included), ground, sq_eps kind, world)
GEOM_CASES = [
    ('n0-ground', 0, 1, True, 'plain', 'template'),
    ('n1-l1-boxy', 1, 1, True, 'boxy', 'posed'),
    ('n1-vb1-m6', 1, 0, False, '-6', 'posed'),
    ('n10-l1-plain', 10, 1, True, 'plain', 'template'),
    ('n10-l1-boxy-noground', 10, 1, False, 'boxy', 'template'),
    ('n10-l2-p6', 10, 2, False, '+6', 'posed'),
    ('n10-l3-m6', 10, 3, True, '-6', 'posed'),
    ('n50-l2-boxy', 50, 2, True, 'boxy', 'posed'),
    ('n50-l3-mixed-noground', 50, 3, False, 'mixed', 'template'),
    ('n50-vb1-m6', 50, 0, True, '-6', 'posed'),
    ('n300-l1-boxy', 300, 1, True, 'boxy', 'posed'),
    ('n300-l3-mixed', 300, 3, True, 'mixed', 'posed'),
]
GEOM_LEAVES = ('sq_eps', 'S', 'R_6d', 'T', 'R_6d_ground', 'T_ground')

_TEMPLATE = {}


def _template_ground():
    if 'ground' not in _TEMPLATE:
        _TEMPLATE['ground'] = D.SceneTemplate(n_blocks=1, txt_size=8).ground_verts.contiguous()
    return _TEMPLATE['ground']


def geom_inputs(case, seed=0):
    """float32 CPU inputs of one geometry case: leaves, the (N, Vb) eta / omega the model derives from the icosphere, the
    ground vertices and the world transform"""
    name, N, level, ground, eps_kind, world = case
    g = _gen(1000 + seed + sum(map(ord, name)))
    if level:
        v = D.get_icosphere(level)[0]
        eta = torch.asin(v[:, 1])[None].expand(N, -1).contiguous()
        omega = torch.atan2(v[:, 0], v[:, 2])[None].expand(N, -1).contiguous()
    else:
        v = D.get_icosphere(1)[0]
        pick = torch.randint(0, v.shape[0], (N,), generator=g)
        poles = (v[:, 1].abs() == 1).nonzero().flatten()
        pick[:min(N, 2)] = poles[:min(N, 2)]                                # the first blocks sit on the poles
        eta, omega = torch.asin(v[pick, 1])[:, None].contiguous(), torch.atan2(v[pick, 0], v[pick, 2])[:, None].contiguous()
    kinds = {'plain': lambda n: torch.zeros(n, 2), 'boxy': lambda n: _uniform(g, (n, 2), -3, 3),
             '+6': lambda n: torch.full((n, 2), 6.), '-6': lambda n: torch.full((n, 2), -6.)}
    if eps_kind == 'mixed':
        choice = torch.randint(0, 4, (N,), generator=g)
        sq_eps = torch.stack([kinds[k](N) for k in ('plain', 'boxy', '+6', '-6')])[choice, torch.arange(N)]
    else:
        sq_eps = kinds[eps_kind](N)
    mag = 10 ** _uniform(g, (N, 1), -3, 3)
    x = {
        'eta': eta.float(), 'omega': omega.float(),
        'ground': _template_ground() if ground else torch.zeros(0, 3),
        'sq_eps': sq_eps.float().contiguous(),
        'S': _uniform(g, (N, 3), -5, 3),
        'R_6d': torch.randn(N, 6, generator=g) * mag,
        'T': torch.randn(N, 3, generator=g) / 2,
        'R_6d_ground': torch.tensor([[1., 0., 0., 0., 1., 0.]]) + 0.3 * torch.randn(1, 6, generator=g),
        'T_ground': torch.tensor([[0., -0.9, 0.]]) + 0.1 * torch.randn(1, 3, generator=g),
        'ratio': 0.25, 'scale_min': 0.2,
    }
    if world == 'template':
        x.update(S_world=0.5, R_world=D.world_rotation(115, 0, 0)[0], T_world=torch.zeros(3))
    else:
        x.update(S_world=0.8, R_world=D.world_rotation(115, 40, -25)[0], T_world=torch.tensor([0.3, -0.2, 0.5]))
    return x


def oracle_geometry(x, dtype):
    """(block vertices (N*Vb, 3), ground vertices (Vg, 3), leaves) in `dtype`, differentiable w.r.t. the leaves"""
    leaves = [x[k].to(dtype).requires_grad_(True) for k in GEOM_LEAVES]
    sq_eps, S, R6, T, R6g, Tg = leaves
    e1, e2 = (torch.sigmoid(sq_eps) * 1.8 + 0.1).split([1, 1], dim=-1)
    u = D.parametric_sq(x['eta'].to(dtype), x['omega'].to(dtype), e1, e2) * x['ratio']
    blk = torch.bmm(u * (S.exp() + x['scale_min'])[:, None], pt3d.rotation_6d_to_matrix(R6)) + T[:, None]
    gr = x['ground'].to(dtype) @ pt3d.rotation_6d_to_matrix(R6g)[0] + Tg
    world = types.SimpleNamespace(S_world=x['S_world'], R_world=x['R_world'][None], T_world=x['T_world'][None])
    return D.SceneTemplate.to_world(world, blk.reshape(-1, 3)), D.SceneTemplate.to_world(world, gr), leaves


def geom_cotangents(x, seed=0):
    g = _gen(77 + seed)
    N, Vb = x['eta'].shape
    return torch.randn(N * Vb, 3, generator=g, dtype=torch.float64), torch.randn(x['ground'].shape[0], 3, generator=g, dtype=torch.float64)


def oracle_geometry_grads(x, dtype, wb, wg):
    blk, gr, leaves = oracle_geometry(x, dtype)
    grads = torch.autograd.grad((blk * wb.to(dtype)).sum() + (gr * wg.to(dtype)).sum(), leaves, allow_unused=True)
    return blk.detach(), gr.detach(), [torch.zeros_like(l) if gg is None else gg for l, gg in zip(leaves, grads)]


def _geom_static(x, dev):
    N, Vb = x['eta'].shape
    return dict(n_blocks=N, verts_per_block=Vb, n_ground_verts=x['ground'].shape[0], sq_eta=x['eta'].to(dev).contiguous(),
                sq_omega=x['omega'].to(dev).contiguous(), ground_verts=x['ground'].to(dev).contiguous(), ratio=x['ratio'],
                scale_min=x['scale_min'], S_world=x['S_world'], R_world=[float(v) for v in x['R_world'].flatten()],
                T_world=[float(v) for v in x['T_world'].flatten()])


def geom_bar(name, case):
    """bar name of a geometry array: the exponent gradient of the sq_eps = 6 cases has its own"""
    return 'geom.sq_eps+6' if name == 'sq_eps' and case[4] == '+6' else f'geom.{name}'


def _check_geom(case, tag, blk, gr, grads, want_blk, want_gr, want_grads):
    check('geom.verts', blk, want_blk, f'{tag} blocks')
    check('geom.verts', gr, want_gr, f'{tag} ground')
    for n, a, b in zip(GEOM_LEAVES, grads, want_grads):
        check(geom_bar(n, case), a, b, tag)


@pytest.mark.parametrize('case', GEOM_CASES, ids=[c[0] for c in GEOM_CASES])
def test_geometry_seams_match_the_float64_oracle(case):
    """scene_geometry_passes (no static environment, and 37 static vertices ahead of the ground)"""
    from dbw_b200.scene_ops import scene_geometry_passes
    dev = torch.device('cuda:0')
    x = geom_inputs(case)
    wb, wg = geom_cotangents(x)
    want_blk, want_gr, want_grads = oracle_geometry_grads(x, torch.float64, wb, wg)
    static = _geom_static(x, dev)
    leaves = [x[k].to(dev).requires_grad_(True) for k in GEOM_LEAVES]
    wb_d, wg_d = wb.float().to(dev), wg.float().to(dev)
    for n_static in (0, 37):
        env_static = torch.randn(n_static, 3, generator=_gen(n_static)).to(dev)
        blk, env = scene_geometry_passes(*leaves, static, env_static)
        assert torch.equal(env[:n_static], env_static)
        w_env = torch.cat([torch.randn(n_static, 3, generator=_gen(5)).to(dev), wg_d])
        grads = torch.autograd.grad((blk * wb_d).sum() + (env * w_env).sum(), leaves)
        _check_geom(case, f'passes n_static={n_static}', blk, env[n_static:], grads, want_blk, want_gr, want_grads)


def _nan(n, dev):
    return torch.full((n,), float('nan'), device=dev)


@pytest.mark.parametrize('case', GEOM_CASES, ids=[c[0] for c in GEOM_CASES])
def test_geometry_cabi_writes_every_output_and_leaves_the_absent_ground_alone(case):
    """the raw entries on NaN-prefilled outputs: the forward without and with static environment vertices (nothing written
    past the end), the backward from two separate gradient blocks and from the two halves of one (ground | blocks) buffer.
    Without a ground its two gradients keep whatever the caller left there; with neither blocks nor a ground nothing is
    written at all"""
    from dbw_b200 import _lib
    from dbw_b200.scene_ops import _geom_struct
    from dbw_b200.renderer import _stream
    L = _lib.lib()
    dev = torch.device('cuda:0')
    x = geom_inputs(case, seed=1)
    wb, wg = geom_cotangents(x, seed=1)
    want_blk, want_gr, want_grads = oracle_geometry_grads(x, torch.float64, wb, wg)
    leaves = [x[k].to(dev).contiguous() for k in GEOM_LEAVES]
    static = _geom_static(x, dev)                       # the struct holds its device pointers: keep the tensors alive
    g = _geom_struct(static, *leaves)
    N, Vb = x['eta'].shape
    Vg, nb = x['ground'].shape[0], N * x['eta'].shape[1]
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    for n_static in (0, 5):
        env_static = torch.randn(n_static, 3, generator=_gen(9)).to(dev)
        out = _nan((n_static + Vg + nb) * 3 + 1, dev)
        _lib.check(L.dbw_scene_geometry_forward(ctypes.byref(g), p(env_static) if n_static else None, n_static, p(out), _stream()),
                   'dbw_scene_geometry_forward')
        assert torch.isnan(out[-1])
        o = out[:-1].view(-1, 3)
        assert torch.equal(o[:n_static], env_static)
        check('geom.verts', o[n_static:n_static + Vg], want_gr, f'forward n_static={n_static} ground')
        check('geom.verts', o[n_static + Vg:], want_blk, f'forward n_static={n_static} blocks')
    g_env_blocks = torch.cat([wg, wb]).float().to(dev).contiguous()         # the forward's (ground | blocks) layout
    sentinel = 12345.
    for separate in (False, True):
        grads = [_nan(t.numel(), dev).view_as(t) for t in leaves[:4]] + [torch.full_like(t, sentinel) for t in leaves[4:]]
        if Vg:
            for t in grads[4:]:
                t.fill_(float('nan'))
        if separate:
            gb, gg = wb.float().to(dev), wg.float().to(dev)                   # two separate allocations
            rc = L.dbw_scene_geometry_backward(ctypes.byref(g), p(gb) if nb else None, p(gg) if Vg else None,
                                               *[p(t) for t in grads], _stream())
        else:
            rc = L.dbw_scene_geometry_backward(ctypes.byref(g), p(g_env_blocks[Vg:]), p(g_env_blocks[:Vg]), *[p(t) for t in grads],
                                               _stream())
        _lib.check(rc, 'dbw_scene_geometry_backward')
        tag = 'backward separate' if separate else 'backward one buffer'
        for n, a, b in zip(GEOM_LEAVES[:4], grads[:4], want_grads[:4]):
            check(geom_bar(n, case), a, b, tag)
        for n, a, b in zip(GEOM_LEAVES[4:], grads[4:], want_grads[4:]):
            if Vg:
                check(geom_bar(n, case), a, b, tag)
            else:
                assert (a == sentinel).all(), (tag, n)


def test_geometry_cabi_with_nothing_to_build_writes_nothing():
    from dbw_b200 import _lib
    from dbw_b200.scene_ops import _geom_struct
    from dbw_b200.renderer import _stream
    L = _lib.lib()
    dev = torch.device('cuda:0')
    x = geom_inputs(('empty', 0, 1, False, 'plain', 'posed'))
    leaves = [x[k].to(dev).contiguous() for k in GEOM_LEAVES]
    static = _geom_static(x, dev)
    g = _geom_struct(static, *leaves)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    out = torch.full((12,), 7., device=dev)
    _lib.check(L.dbw_scene_geometry_forward(ctypes.byref(g), None, 0, p(out), _stream()), 'forward without static vertices')
    torch.cuda.synchronize()
    assert (out == 7.).all()
    env_static = torch.randn(3, 3, generator=_gen(1)).to(dev)
    _lib.check(L.dbw_scene_geometry_forward(ctypes.byref(g), p(env_static), 3, p(out), _stream()), 'forward with static vertices')
    assert torch.equal(out[:9], env_static.reshape(-1)) and (out[9:] == 7.).all()
    grads = [torch.full((6,), 7., device=dev) for _ in range(6)]
    _lib.check(L.dbw_scene_geometry_backward(ctypes.byref(g), p(out), p(out), *[p(t) for t in grads], _stream()), 'backward')
    _lib.check(L.dbw_scene_geometry_backward(ctypes.byref(g), None, None, *[p(t) for t in grads], _stream()), 'backward, no pointers')
    torch.cuda.synchronize()
    assert all((t == 7.).all() for t in grads)


# ---------------------------------------------------------------------------------------------------------- opacities
# (n_blocks, faces_per_block, keep_threshold, noisy)
OPACITY_CASES = [(1, 1, -1., False), (7, 80, 0.01, True), (1000, 1, 0.5, True), (1000, 80, 0.01, False), (333, 300, 0.5, False),
                 (1000, 300, -1., True), (50, 300, 0.01, True)]
NOISE_SCALE = 0.7


def opacity_inputs(case):
    """logits: half saturating (up to +-100), half moderate, none within 0.05 of logit(threshold) so that the keep decision is
    the same in any precision"""
    N, fpb, thr, noisy = case
    g = _gen(31 + N + fpb)
    lg = torch.where(torch.rand(N, generator=g) < 0.5, _uniform(g, (N,), -100, 100), 4 * torch.randn(N, generator=g))
    if N > 2:
        lg[:3] = torch.tensor([100., -100., -6.])
    if thr > 0:
        t = math.log(thr / (1 - thr))
        close = (lg - t).abs() < 0.05
        lg = torch.where(close, t + 0.1 * torch.where(lg >= t, 1., -1.), lg)
    noise = 3 * torch.randn(N, generator=g) if noisy else None
    fmap = torch.randint(-1, 1 << 20, (N * fpb,), generator=g, dtype=torch.int32)
    return lg.float(), (noise.float() if noisy else None), fmap


def oracle_opacity(lg, noise, thr, dtype):
    l = lg.to(dtype).requires_grad_(True)
    a = torch.sigmoid(l + NOISE_SCALE * noise.to(dtype) if noise is not None else l)
    keep = torch.sigmoid(lg.double()) > thr if thr >= 0 else torch.ones(lg.shape, dtype=torch.bool)
    return l, a, a * keep, keep


@pytest.mark.parametrize('case', OPACITY_CASES, ids=[f'n{c[0]}-f{c[1]}-thr{c[2]}-{"noisy" if c[3] else "clean"}' for c in OPACITY_CASES])
def test_opacities_match_the_float64_oracle(case):
    """block_opacities and the raw entries: alpha, alpha_kept, the face map (exact), d/d logit with either upstream gradient
    NULL on its own and both present"""
    from dbw_b200 import _lib
    from dbw_b200.scene_ops import block_opacities
    from dbw_b200.renderer import _stream
    L = _lib.lib()
    dev = torch.device('cuda:0')
    N, fpb, thr, noisy = case
    lg, noise, fmap0 = opacity_inputs(case)
    l64, a64, k64, keep = oracle_opacity(lg, noise, thr, torch.float64)
    want_fmap = torch.where(keep[:, None], fmap0.view(N, fpb), torch.full((), -1, dtype=torch.int32)).reshape(-1)
    ga, gk = torch.randn(N, generator=_gen(2), dtype=torch.float64), torch.randn(N, generator=_gen(3), dtype=torch.float64)
    lg_d = lg.to(dev).requires_grad_(True)
    nz_d = noise.to(dev) if noisy else None
    fm_d = fmap0.to(dev)
    alpha, kept, fmap = block_opacities(lg_d, nz_d, NOISE_SCALE if noisy else 0., thr, fm_d, fpb)
    check('opacity.alpha', alpha, a64, 'alpha')
    check('opacity.alpha', kept, k64, 'alpha_kept')
    assert torch.equal(fmap.cpu(), want_fmap)
    assert thr >= 0 or fmap.data_ptr() == fm_d.data_ptr()
    for wa, wk, tag in ((ga, gk, 'both'), (ga, None, 'alpha only'), (None, gk, 'kept only')):
        want, = torch.autograd.grad(sum((t * w).sum() for t, w in ((a64, wa), (k64, wk)) if w is not None), l64, retain_graph=True)
        got, = torch.autograd.grad(sum((t * w.float().to(dev)).sum() for t, w in ((alpha, wa), (kept, wk)) if w is not None), lg_d,
                                   retain_graph=True)
        check('opacity.g_logit', got, want, f'seam, {tag}')
        # the C-ABI itself, NULL for each absent gradient, on a NaN-prefilled output
        g_out = _nan(N, dev)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        wa_d, wk_d = (w.float().to(dev) if w is not None else None for w in (wa, wk))
        _lib.check(L.dbw_opacity_backward(p(lg_d), p(nz_d), NOISE_SCALE if noisy else 0., thr, p(wa_d), p(wk_d), N, p(g_out),
                                          _stream()), 'dbw_opacity_backward')
        check('opacity.g_logit', g_out, want, f'C-ABI, {tag}')
    # forward without the optional outputs, on NaN-prefilled ones
    a_out, k_out, f_out = _nan(N, dev), _nan(N, dev), torch.full((N * fpb,), -7, dtype=torch.int32, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(L.dbw_opacity_forward(p(lg_d), p(nz_d) if noisy else None, NOISE_SCALE if noisy else 0., thr, p(fm_d), N, fpb,
                                     p(a_out), None, None, _stream()), 'dbw_opacity_forward')
    check('opacity.alpha', a_out, a64, 'C-ABI alpha')
    _lib.check(L.dbw_opacity_forward(p(lg_d), p(nz_d) if noisy else None, NOISE_SCALE if noisy else 0., thr, p(fm_d), N, fpb,
                                     p(a_out), p(k_out), p(f_out), _stream()), 'dbw_opacity_forward')
    check('opacity.alpha', k_out, k64, 'C-ABI alpha_kept')
    assert torch.equal(f_out.cpu(), want_fmap if thr >= 0 else fmap0)


# ---------------------------------------------------------------------------------------------------------- texture preparation
FUSED, CELLS, EXPAND, CELLS4 = 0, 1, 2, 3
STAGE_NAMES = {FUSED: 'fused', CELLS: 'cells', EXPAND: 'expand', CELLS4: 'cells4'}
# one launch per case: jobs (stage, n_maps, txt_size, decimate, p_left, p_right, logit range)
TEX_CASES = [
    [(FUSED, 3, 16, 1, 0, 3, 5.)],
    [(FUSED, 2, 8, 8, 8, 8, 5.)],
    [(FUSED, 4, 33, 1, 33, 33, 90.)],
    [(CELLS4, 3, 40, 8, 0, 0, 5.)],
    [(EXPAND, 2, 72, 8, 0, 3, 1.)],
    [(FUSED, 1, 256, 8, 0, 0, 0.5), (FUSED, 1, 256, 8, 0, 0, 0.5), (FUSED, 50, 72, 8, 0, 3, 90.)],
    [(CELLS4, 1, 256, 8, 0, 0, 5.), (CELLS4, 1, 256, 8, 0, 0, 5.), (CELLS4, 50, 40, 8, 0, 0, 90.)],
    [(CELLS, 2, 16, 8, 0, 0, 5.), (CELLS4, 3, 72, 8, 0, 0, 5.), (EXPAND, 4, 72, 8, 72, 72, 1.), (FUSED, 5, 40, 8, 40, 0, 90.)],
    [(EXPAND, 2, 16, 1, 0, 0, 1.), (FUSED, 3, 40, 1, 0, 3, 90.), (CELLS, 20, 33, 1, 0, 0, 5.), (CELLS4, 2, 8, 1, 0, 0, 5.)],
    [(FUSED, 2, 8, 1, 8, 8, 90.), (EXPAND, 1, 256, 8, 0, 3, 1.), (CELLS, 7, 256, 1, 0, 0, 0.5), (CELLS4, 6, 16, 1, 0, 0, 5.)],
]


def _tex_id(case):
    return '+'.join(f'{STAGE_NAMES[j[0]]}{j[1]}x{j[2]}f{j[3]}p{j[4]}_{j[5]}' for j in case)


def tex_inputs(case, k):
    """float32 inputs of job k: logits in +-range, or cell colours in [0, 1] for EXPAND (its input is the cells' RGB)"""
    stage, M, TS, f, pl, pr, rng = case[k]
    g = _gen(500 + 17 * k + TS + M)
    side = TS // f if stage == EXPAND else TS
    x = _uniform(g, (M, side, side, 3), -rng, rng)
    if stage != EXPAND and rng >= 90:                                        # the range's ends themselves, too
        x.view(-1)[::7], x.view(-1)[3::7] = rng, -rng
    return torch.sigmoid(x) if stage == EXPAND else x


def tex_out_shape(job):
    stage, M, TS, f, pl, pr, _ = job
    if stage in (CELLS, CELLS4):
        return (M, TS // f, TS // f, 3 if stage == CELLS else 4)
    return (M, TS, pl + TS + pr, 4)


def oracle_texture(job, x, dtype):
    """(input leaf, RGB output) in `dtype`: the atlas (M, TS, pl + TS + pr, 3) or the cells (M, TS/f, TS/f, 3)"""
    stage, M, TS, f, pl, pr, _ = job
    t = x.to(dtype).requires_grad_(True)
    if stage == EXPAND:
        maps = F.interpolate(t.permute(0, 3, 1, 2), scale_factor=f, mode='nearest').permute(0, 2, 3, 1) if f > 1 else t
    else:
        s = torch.sigmoid(t)
        if stage in (CELLS, CELLS4):
            return t, F.avg_pool2d(s.permute(0, 3, 1, 2), kernel_size=f, stride=f).permute(0, 2, 3, 1)
        maps = D.SceneTemplate._decimate(s, f) if f > 1 else s
    return t, F.pad(maps.permute(0, 3, 1, 2), pad=(pl, pr, 0, 0), mode='circular').permute(0, 2, 3, 1)


def tex_cotangent(job, k):
    return torch.randn(tex_out_shape(job), generator=_gen(900 + k), dtype=torch.float64)


def oracle_texture_grads(job, x, w, dtype):
    t, out = oracle_texture(job, x, dtype)
    grad, = torch.autograd.grad((out * w[..., :3].to(dtype)).sum(), t)
    return out.detach(), grad


def _tex_job(tex, atlas, g_tex, job):
    from dbw_b200._lib import DbwTexJob
    stage, M, TS, f, pl, pr, _ = job
    return DbwTexJob(tex.data_ptr(), atlas.data_ptr(), g_tex.data_ptr() if g_tex is not None else None, M, TS, pl, pr, f, stage)


@pytest.mark.parametrize('case', TEX_CASES, ids=[_tex_id(c) for c in TEX_CASES])
def test_texture_preparation_matches_the_float64_oracle(case):
    """dbw_texture_prep_{forward,backward}_multi, every job of the launch against its oracle; the float4 outputs' fourth
    channel is exactly 0"""
    from dbw_b200.scene_ops import _tex_launch
    dev = torch.device('cuda:0')
    xs = [tex_inputs(case, k) for k in range(len(case))]
    ws = [tex_cotangent(job, k) for k, job in enumerate(case)]
    want = [oracle_texture_grads(job, x, w, torch.float64) for job, x, w in zip(case, xs, ws)]
    xd = [x.to(dev).contiguous() for x in xs]
    outs = [torch.full(tex_out_shape(job), float('nan'), device=dev) for job in case]
    _tex_launch([_tex_job(x, o, None, job) for x, o, job in zip(xd, outs, case)], False)
    wd = [w.float().to(dev).contiguous() for w in ws]
    gs = [torch.full_like(x, float('nan')) for x in xd]
    _tex_launch([_tex_job(w if job[0] == EXPAND else x, w, gx, job) for x, w, gx, job in zip(xd, wd, gs, case)], True)
    for k, (job, o, gx, (wo, wg)) in enumerate(zip(case, outs, gs, want)):
        tag = f'job {k} {STAGE_NAMES[job[0]]}'
        check('tex.out', o[..., :3], wo, tag)
        if o.shape[-1] == 4:
            assert (o[..., 3] == 0).all(), tag
        check('tex.grad', gx, wg, tag)


@pytest.mark.parametrize('offset', [0, 1, 2, 3])
def test_cells4_backward_reads_a_gradient_view_at_any_float_offset(offset):
    """the CELLS4 backward takes its float4 cell gradient as a view of a gradient bucket at any 4-byte offset
    (parallel.GradSumPoint): the environment (64^2, f = 8) and blocks (5 x 40^2, f = 8) stacks in one launch"""
    from dbw_b200.scene_ops import _tex_launch
    dev = torch.device('cuda:0')
    jobs = [(CELLS4, 2, 64, 8, 0, 0, 5.), (CELLS4, 5, 40, 8, 0, 0, 5.)]
    xs = [tex_inputs(jobs, k) for k in range(2)]
    ws = [tex_cotangent(job, k) for k, job in enumerate(jobs)]
    want = [oracle_texture_grads(job, x, w, torch.float64)[1] for job, x, w in zip(jobs, xs, ws)]
    n = [w.numel() for w in ws]
    bucket = torch.full((offset + 1 + sum(n) + 3,), float('nan'), device=dev)
    views = [bucket[offset + 1:offset + 1 + n[0]].view(ws[0].shape), bucket[offset + 1 + n[0]:offset + 1 + sum(n)].view(ws[1].shape)]
    for v, w in zip(views, ws):
        v.copy_(w.float())
    xd = [x.to(dev).contiguous() for x in xs]
    gs = [torch.full_like(x, float('nan')) for x in xd]
    _tex_launch([_tex_job(x, v, gx, job) for x, v, gx, job in zip(xd, views, gs, jobs)], True)
    for gx, wg in zip(gs, want):
        check('tex.grad', gx, wg, f'offset {offset}')


# ---------------------------------------------------------------------------------------------------------- the model chain
CHAIN_N, CHAIN_TS, CHAIN_UP = 6, 32, 2
CHAIN_WORLD = dict(S_world=0.6, R_world=(115, 30, -20), T_world=(0.1, -0.2, 0.3))
# phase -> (epoch, cells, kill one block, opacity noise, one-rank gradient-sum point)
CHAIN_PHASES = {
    'coarse-decimated-cells': (0, True, False, False, False),
    'coarse-decimated-atlas': (0, False, False, False, False),
    'coarse-undecimated': (1000, True, False, False, False),
    'fine': (2000, True, False, False, False),
    'kill-blocks': (0, True, True, False, False),
    'opacity-noise': (0, True, False, True, False),
    'grad-sum-cells': (0, True, False, False, True),
    'grad-sum-atlas': (0, False, False, True, True),
}
CHAIN_LEAVES = ('sq_eps', 'S', 'R_6d', 'T', 'R_6d_ground', 'T_ground', 'alpha_logit', 'texture_bkg', 'texture_ground', 'textures')
CHAIN_OUTPUTS = ('env_verts', 'env_atlas', 'blk_verts', 'atlas', 'alpha')


def chain_params(phase):
    """float32 leaf values of the model chain: boxy exponents, a perturbed ground pose, opacities on both sides of 0.5 (and one
    block at sigmoid 0.0025, killed at 0.01, in the kill-blocks phase)"""
    epoch, cells, kill, noisy, _ = CHAIN_PHASES[phase]
    p = D.init_params(n_blocks=CHAIN_N, txt_size=CHAIN_TS, txt_bkg_upscale=CHAIN_UP, seed=41, boxy=True)
    g = _gen(42)
    p['R_6d_ground'] = p['R_6d_ground'] + 0.2 * torch.randn(1, 6, generator=g)
    p['T_ground'] = p['T_ground'] + 0.1 * torch.randn(1, 3, generator=g)
    p['alpha_logit'] = torch.tensor([2., -2., 1., 3., -1., 0.5])
    if kill:
        p['alpha_logit'][3] = -6.
    for k in ('texture_bkg', 'texture_ground', 'textures'):
        p[k] = p[k] * 20                      # logits over +-2 or so: sigmoid slopes well away from 1/4
    p['noise'] = torch.randn(CHAIN_N, generator=g) if noisy else None
    return p


def chain_phase_settings(phase):
    """(decim_env, decim_blocks, hard_filter, keep threshold, cells) the model uses in this phase (coarse_learning 1500,
    decimate_txt 750, decimate_factor 8, kill_blocks on)"""
    epoch, cells, *_ = CHAIN_PHASES[phase]
    decim = 8 if epoch < 750 else 1
    fine = epoch >= 1500
    return decim, (decim if not fine else 1), fine, (0.5 if fine else 0.01), cells and decim == 8


def chain_oracle(phase, dtype, cotangents=None):
    """oracle outputs (dict, the layout of _scene_tensors with RGB only) and, with cotangents, the leaf gradients"""
    p32 = chain_params(phase)
    noise = p32.pop('noise')
    decim_env, decim_blocks, fine, thr, cells = chain_phase_settings(phase)
    tpl = D.SceneTemplate(n_blocks=CHAIN_N, txt_size=CHAIN_TS, txt_bkg_upscale=CHAIN_UP, **CHAIN_WORLD)
    p = {k: v.to(dtype).requires_grad_(True) for k, v in p32.items()}
    env = tpl.build_env(p, decimate=decim_env if decim_env > 1 else 0)
    blocks, alpha = tpl.build_blocks(p, keep=None, decimate=decim_blocks if decim_blocks > 1 else 0,
                                     alpha_noise=None if noise is None else float(chain_noise_scale()) * noise.to(dtype))
    env_maps, blk_maps = torch.stack(env['maps']), torch.stack(blocks['maps'])
    if cells:                                         # a decimated map is constant over its cells: one texel per cell
        pl = tpl.txt_padding[0]
        env_maps, blk_maps = env_maps[:, ::8, ::8], blk_maps[:, ::8, pl:pl + CHAIN_TS:8]
    out = {'env_verts': env['verts'], 'env_atlas': env_maps, 'blk_verts': blocks['verts'], 'atlas': blk_maps,
           'alpha': None if fine else alpha}
    keep = torch.sigmoid(p32['alpha_logit'].double()) > thr
    if cotangents is None:
        return out, keep, None
    loss = sum((out[k] * _rgb(k, cotangents[k]).to(dtype)).sum() for k in CHAIN_OUTPUTS if out[k] is not None)
    grads = torch.autograd.grad(loss, [p[k] for k in CHAIN_LEAVES], allow_unused=True)
    return {k: v.detach() if v is not None else None for k, v in out.items()}, keep, dict(zip(CHAIN_LEAVES, grads))


def _rgb(k, t):
    return t[..., :3] if k in ('env_atlas', 'atlas') else t


def chain_noise_scale():
    return 0.7


def chain_cotangents(phase, shapes):
    g = _gen(4242)
    return {k: torch.randn(shapes[k], generator=g, dtype=torch.float64) for k in CHAIN_OUTPUTS if shapes.get(k) is not None}


def chain_shapes(phase):
    """the RGB(A) shapes of the oracle outputs, with the float4 layouts' fourth channel"""
    out, _, _ = chain_oracle(phase, torch.float32)
    shapes = {}
    for k, v in out.items():
        if v is not None:
            shapes[k] = tuple(v.shape[:-1]) + ((4,) if k in ('env_atlas', 'atlas') else (v.shape[-1],))
    return shapes


@pytest.mark.parametrize('phase', list(CHAIN_PHASES))
def test_model_scene_tensors_match_the_float64_oracle(phase):
    """DifferentiableBlocksWorld._scene_tensors -> build_env / build_blocks (no rasterizer): every output and every leaf
    gradient; the face map exactly (killed / filtered blocks at -1)"""
    from copy import deepcopy
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.parallel import GradSumPoint
    epoch, cells_arg, kill, noisy, grad_sum = CHAIN_PHASES[phase]
    dev = torch.device('cuda:0')
    cfg = {
        'mesh': {'n_blocks': CHAIN_N, 'txt_size': CHAIN_TS, 'txt_bkg_upscale': CHAIN_UP, **{k: list(v) if isinstance(v, tuple) else v
                                                                                          for k, v in CHAIN_WORLD.items()}},
        'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
        'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                       'decouple_rendering': True, 'opacity_noise': chain_noise_scale() if noisy else False},
        'loss': {'rgb_weight': 1},
    }
    torch.manual_seed(0)
    model = DifferentiableBlocksWorld((48, 64), **deepcopy(cfg)).to(dev)
    model.train()
    model.set_cur_epoch(epoch)
    p32 = chain_params(phase)
    with torch.no_grad():
        for k in CHAIN_LEAVES:
            getattr(model, k).copy_(p32[k])
    assert torch.equal(model.R_world.cpu(), D.world_rotation(*CHAIN_WORLD['R_world']))
    shapes = chain_shapes(phase)
    ws = chain_cotangents(phase, shapes)
    want, keep, want_grads = chain_oracle(phase, torch.float64, ws)
    if noisy:
        model.opacity_noise_buffer = p32['noise'].to(dev)

    class OneRankBucket:
        def __init__(self):
            self.flat = torch.full((model.grad_sum_floats() + 3,), float('nan'), device=dev)
            self.calls = 0

        def all_reduce(self, buf):
            self.calls += 1

    bucket = OneRankBucket()
    if grad_sum:
        model.grad_sum_point = GradSumPoint(bucket)
    _, hard_filter, _ = model._phase()
    (env_verts, env_atlas, env_table), (blk_verts, atlas, table, fmap, alpha) = model._scene_tensors(hard_filter, cells=cells_arg)
    got = {'env_verts': env_verts, 'env_atlas': env_atlas.view(shapes['env_atlas']), 'blk_verts': blk_verts,
           'atlas': atlas.view(shapes['atlas']), 'alpha': alpha}
    assert (alpha is None) == (want['alpha'] is None)
    for k in CHAIN_OUTPUTS:
        if want[k] is not None:
            check(f'chain.{k}', _rgb(k, got[k]), want[k], k)
    for k in ('env_atlas', 'atlas'):
        assert (got[k][..., 3] == 0).all(), k
    want_fmap = torch.where(keep[:, None], torch.arange(CHAIN_N, dtype=torch.int32)[:, None].expand(-1, model.BNF),
                            torch.full((), -1, dtype=torch.int32)).reshape(-1)
    assert torch.equal(fmap.cpu(), want_fmap)
    loss = sum((got[k] * ws[k].float().to(dev)).sum() for k in CHAIN_OUTPUTS if got[k] is not None)
    leaves = [getattr(model, k) for k in CHAIN_LEAVES]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True)
    assert bucket.calls == (1 if grad_sum else 0)
    for k, a in zip(CHAIN_LEAVES, grads):
        b = want_grads[k]
        assert (a is None) == (b is None), k
        if b is not None:
            check(f'chain.{k}', a, b, k)

