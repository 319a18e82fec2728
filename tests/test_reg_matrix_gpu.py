"""GPU: the regulariser kernels (csrc/dbw_reg.cu) -- parsimony, total variation, overlap and every leaf gradient -- against a
float64 oracle, element by element, through the raw C-ABI (dbw_regularisers_*) and through losses.regularisers.

The oracle evaluates the same float32 inputs in float64: the statement of oracle.dbw_path.regularisers with the opacities
alpha_full as a leaf, its overlap term computed over chunks of blocks (the per-point occupancy without grad first, then one
backward per chunk), so that 257 blocks or 50 x 1000 points stay within memory (tests/test_reg_matrix_host.py checks it
against D.regularisers to 1e-12).  Every term gets its own upstream gradient, drawn from +- values and 0.  The cases cover:
  * the overlap CTAs' block chunks: 1, 2, 127, 128, 129, 256 and 257 blocks (REG_OV_CHUNK = 128), killed blocks, all killed;
  * point counts 1, 100, 255, 256, 257 and 1000: CTAs over many blocks, within one block, ending partly invalid;
  * block parameters: exponent logits at +-6, log-scales -5 .. 3, unnormalised 6D vectors, small blocks far from the others
    whose points lie beyond the +-5 clamp in the other blocks' frames;
  * TV sizes whose background | ground | blocks boundaries fall inside a forward CTA, inside one thread's four strided
    texels and inside a backward CTA; sides 2 and 3 (the u-wrap's two neighbours are one texel); an environment smaller than
    the blocks' maps; the shipped DTU and configs[4] shapes; every norm, both phases; plateau maps (equal logits over 8 x 8
    cells: exact zero differences) and logits up to +-20;
  * all seven term subsets with distinct weights including 0, and each gradient output NULL on its own.
Outputs and gradients are prefilled with NaN (every element is written, include/dbw_render.h: "written, not accumulated"),
outputs of terms that are off keep their NaN, and the workspace is the reported size followed by a sentinel tail no call
touches.

The inputs keep every discrete decision of the function far from float32 rounding (reg_inputs redraws points that are not,
the texture logits lie on a grid): the overlap excess occ - 1.95, the +-5 clamp of block-frame coordinates, l2's 1e-6 clamp
and l1's sign(0).  Bars are fractions of each array's largest float64 magnitude, BAR_FACTOR times what the oracle's own
float32 evaluation shows against float64 over the same cases (tests/test_reg_matrix_host.py measures it on the CPU).

This module is importable without a GPU: the host module reuses its case tables and oracle."""
import ctypes
import functools
import json
import math
import os

import pytest
import torch

from oracle import dbw_path as D
from oracle import pt3d

pytestmark = pytest.mark.gpu

PAR, TV, OV = 1, 2, 4                                   # DBW_REG_* of include/dbw_render.h
TERMS = ((PAR, 'parsimony'), (TV, 'tv'), (OV, 'overlap'))
TV_CODES = {'l2': 0, 'l1': 1, 'l2sq': 2}
TV_NORMS = {'l1': lambda t: t.abs().sum(-1), 'l2': lambda t: D.safe_pow(t.pow(2).sum(-1), 0.5), 'l2sq': lambda t: t.pow(2).sum(-1)}
RATIO, SCALE_MIN = 0.25, 0.2
TEMPERATURE, OCC_LIMIT, CLAMP = 0.005, 1.95, 5.0
LEAVES = ('texture_bkg', 'texture_ground', 'textures', 'S', 'R_6d', 'T', 'sq_eps', 'alpha_full')
# the terms that read (and whose gradient writes) each leaf
READ_BY = {'texture_bkg': TV, 'texture_ground': TV, 'textures': TV, 'S': OV, 'R_6d': OV, 'T': OV, 'sq_eps': OV,
           'alpha_full': PAR | OV}

# every discrete decision stays this far from its threshold (asserted by tests/test_reg_matrix_host.py)
OCC_MARGIN = 0.01           # |occ - 1.95| of every point
CLAMP_MARGIN = 1e-3         # ||local| - 5| of every point in every block's frame
L2_MARGIN = 0.1             # |sum d^2 / 1e-6 - 1| of every texel pair
L1_MARGIN = 1e-4            # |d| of every nonzero channel difference
# texture logits: a grid of steps 1/4 over +-4, and +-20 (sigmoid 1 - 2e-9: saturated); neighbouring grid values differ by
# at least 5e-3 after the sigmoid
LOGIT_GRID = torch.cat([torch.arange(-16, 17, dtype=torch.float32) / 4, torch.tensor([-20., 20.])])

BAR_FACTOR = 8
# Each bar is about BAR_FACTOR times the worst deviation of the oracle's own float32 evaluation from float64 over this module's
# cases (fraction of each array's largest magnitude; tests/test_reg_matrix_host.py measures it on the CPU and keeps the two
# consistent).  Bars above 2e-6 are explained in BAR_NOTES.
BARS = {
    'val.parsimony': 1.2e-6, 'val.tv': 6e-7, 'val.overlap': 6e-6,
    'g.texture_bkg': 2e-6, 'g.texture_ground': 2e-6, 'g.textures': 2e-6,
    'g.S': 3e-4, 'g.R_6d': 1.5e-3, 'g.T': 5e-4, 'g.sq_eps': 1.7e-4, 'g.alpha_full': 3e-6,
}
_AMPLIFIED = ('the overlap term takes sigmoid(-sdf / 0.005) of every point in every block: the float32 rounding of a point and '
              'of its block-frame coordinates reaches the sigmoid 200x larger')
BAR_NOTES = {
    'val.overlap': 'the mean of each point\'s clamped excess, a sum of sigmoids: ' + _AMPLIFIED,
    'g.alpha_full': 'sums of sigmoid(-sdf / 0.005) over all points: ' + _AMPLIFIED,
    'g.S': _AMPLIFIED + '; log-scales of -5 .. 3 make blocks 100x apart in size, and exponents at e = 0.1 raise the '
                        'coordinates to the power 10',
    'g.T': _AMPLIFIED + '; the translation gradient sums those of every point the block reaches, of both signs',
    'g.R_6d': _AMPLIFIED + '; the 6D vectors span 0.1 .. 10 in magnitude (gradients ~1/|a|), and Gram-Schmidt loses bits on '
                           'nearly parallel pairs',
    'g.sq_eps': _AMPLIFIED + '; d/d e sums |x|^(2/e) ln|x| terms of both signs',
}

WORST = {}          # bar name -> worst error seen in this session (written out when DBW_REG_MATRIX_REPORT names a file)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    path = os.environ.get('DBW_REG_MATRIX_REPORT')
    if path:
        with open(path, 'w') as f:
            json.dump({k: {'worst_rel_err': v, 'bar': BARS[k]} for k, v in sorted(WORST.items())}, f, indent=1)


def rel_err(got, want):
    """max |got - want| over max |want| (0 when both are all zero, inf when only `got` is not, or on a NaN)"""
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
    return torch.rand(shape, generator=g, dtype=torch.float64) * (hi - lo) + lo


# ---------------------------------------------------------------------------------------------------------- cases
def _case(name, n_blocks, n_points, env, txt, norm, coarse=True, terms=PAR | TV | OV, w=(0.01, 0.1, 1.0), blocks='packed',
          maps='grid', kill='some', zero=0):
    """blocks: 'packed' (overlapping blocks of moderate size) or 'wide' (log-scales -5 .. 3, exponent logits at +-6, small blocks
    far away); maps: 'grid' (a grid logit per texel) or 'plateau' (one per 8 x 8 cell); kill: 'none', 'some' (every fifth
    block at opacity 0), 'all'; zero: the term whose upstream gradient is 0"""
    return dict(name=name, n_blocks=n_blocks, n_points=n_points, env=env, txt=txt, norm=norm, coarse=coarse, terms=terms, w=w,
                blocks=blocks, maps=maps, kill=kill, zero=zero)


CASES = [
    # overlap chunks and point counts (TV boundaries inside CTAs and strides: 20^2 = 400, 30^2 = 900, ...)
    _case('n1-p1000', 1, 1000, 20, 12, 'l2', kill='none'),
    _case('n2-p257', 2, 257, 30, 7, 'l1', kill='none', zero=PAR),
    _case('n127-p100-wide', 127, 100, 16, 8, 'l2sq', blocks='wide'),
    _case('n128-p255', 128, 255, 20, 12, 'l1', maps='plateau'),
    _case('n129-p256-wide', 129, 256, 30, 7, 'l2', blocks='wide', zero=TV),
    _case('n256-p1', 256, 1, 8, 4, 'l2sq'),
    _case('n257-p100-wide', 257, 100, 3, 2, 'l1', blocks='wide'),
    _case('n257-p1-all-killed', 257, 1, 2, 3, 'l2', kill='all'),
    _case('n40-p257-wide', 40, 257, 5, 16, 'l2', blocks='wide'),
    # the shipped shapes, every norm, both phases
    _case('dtu-coarse-l2', 10, 1000, 256, 256, 'l2', maps='plateau'),
    _case('dtu-fine-l2sq', 10, 1000, 256, 256, 'l2sq', coarse=False, terms=TV),
    _case('configs4-coarse-l1', 50, 1000, 256, 128, 'l1', maps='plateau'),
    _case('configs4-fine-l1', 50, 1000, 256, 128, 'l1', coarse=False, terms=TV),
    _case('e20-t12-fine-l2', 6, 100, 20, 12, 'l2', coarse=False, terms=TV, maps='plateau'),
    _case('e3-t2-fine-l1', 3, 100, 3, 2, 'l1', coarse=False, terms=TV),
    # every term subset, distinct weights including 0 (the weights of terms that are off are NaN on the C-ABI)
    _case('P', 9, 64, 12, 10, 'l2', terms=PAR, w=(0.7, None, None)),
    _case('T', 9, 64, 12, 10, 'l1', terms=TV, w=(None, 0.35, None)),
    _case('O', 12, 300, 12, 10, 'l2', terms=OV, w=(None, None, 2.5)),
    _case('PT', 9, 64, 30, 7, 'l2sq', terms=PAR | TV, w=(0., 0.2, None)),
    _case('PO', 12, 300, 12, 10, 'l2', terms=PAR | OV, w=(0.05, None, 0.)),
    _case('TO', 12, 300, 20, 12, 'l2', terms=TV | OV, w=(None, 0., 1.3), blocks='wide'),
    _case('PTO', 12, 300, 20, 12, 'l1', w=(0.45, 0.9, 0.6), zero=OV),
]
CASE_IDS = [c['name'] for c in CASES]
BY_NAME = {c['name']: c for c in CASES}


def cotangents(case):
    """one upstream gradient per term, distinct, +- and 0 for case['zero']"""
    g = _gen(sum(map(ord, case['name'])))
    vals = torch.tensor([-2.5, -1.25, -0.4, 0.3, 0.9, 1.7])[torch.randperm(6, generator=g)[:3]]
    return {name: 0. if case['zero'] == bit else float(v) for (bit, name), v in zip(TERMS, vals)}


def _maps(g, n, side, kind):
    """(n, side, side, 3) grid logits, 10% of them +-20; 'plateau': equal over 8 x 8 cells"""
    cell = 8 if kind == 'plateau' else 1
    cs = -(-side // cell)
    idx = torch.randint(0, 33, (n, cs, cs, 3), generator=g)
    sat = torch.rand(n, cs, cs, 3, generator=g) < 0.1
    idx = torch.where(sat, 33 + torch.randint(0, 2, (n, cs, cs, 3), generator=g), idx)
    x = LOGIT_GRID[idx]
    if cell > 1:
        x = x.repeat_interleave(cell, 1).repeat_interleave(cell, 2)[:, :side, :side]
    return x.contiguous()


def _blocks(g, case):
    N, kind = case['n_blocks'], case['blocks']
    if kind == 'packed':
        S = _uniform(g, (N, 3), -1.2, 0.3)
        T = torch.randn(N, 3, generator=g, dtype=torch.float64) * (0.15 if N > 2 else 0.02)     # two blocks: overlapping
        sq_eps = _uniform(g, (N, 2), -3, 3)
    else:
        S = _uniform(g, (N, 3), -5, 3)
        T = torch.randn(N, 3, generator=g, dtype=torch.float64) * 0.3
        sq_eps = torch.where(torch.rand(N, 2, generator=g) < 0.5, torch.where(torch.rand(N, 2, generator=g) < 0.5, 6., -6.),
                             _uniform(g, (N, 2), -3, 3))
        far = torch.arange(N) % 8 == 7                                    # small blocks away from the cluster
        d = torch.randn(N, 3, generator=g, dtype=torch.float64)
        T = torch.where(far[:, None], 2.5 * d / d.norm(dim=1, keepdim=True), T)
        S = torch.where(far[:, None], _uniform(g, (N, 3), -5, -3), S)
    R_6d = torch.randn(N, 6, generator=g, dtype=torch.float64) * 10 ** _uniform(g, (N, 1), -1, 1)
    alpha = _uniform(g, (N,), 0.985, 0.9995)                # two overlapping blocks can pass 1.95
    if case['kill'] == 'some':
        alpha[torch.arange(N) % 5 == 4] = 0.
    elif case['kill'] == 'all':
        alpha[:] = 0.
    return {'S': S, 'R_6d': R_6d, 'T': T, 'sq_eps': sq_eps, 'alpha_full': alpha}


def _frames(lv):
    """(S, R, T, e1, e2) of every block from its leaves: S = exp(S) + scale_min, R = rotation_6d_to_matrix(R_6d),
    (e1, e2) = sigmoid(sq_eps) * 1.8 + 0.1"""
    e1, e2 = (torch.sigmoid(lv['sq_eps']) * 1.8 + 0.1).split([1, 1], dim=-1)
    return lv['S'].exp() + SCALE_MIN, pt3d.rotation_6d_to_matrix(lv['R_6d']), lv['T'], e1, e2


def sample_points(S, R, T, unit_samples):
    """((2 u - 1) ratio S_b) R_b + T_b of every block b, (N * n_points, 3), no grad"""
    with torch.no_grad():
        u = unit_samples.to(S)
        return ((u * 2 - 1) * RATIO * S[:, None]) @ R + T[:, None]


CHUNK_PAIRS = 1 << 20       # (block, point) pairs the oracle holds at a time


def _chunk(n_pts):
    return max(1, CHUNK_PAIRS // n_pts)


def block_local(pts, S, R, T, k0, k1):
    """the points in the frames of blocks k0 .. k1 - 1: (k1 - k0, n_pts, 3), as D.regularisers writes it"""
    return ((pts[None] - T[k0:k1, None]) @ R[k0:k1].transpose(1, 2)) / (S[k0:k1, None] * RATIO)


def overlap_decisions(x, idx=None):
    """float64, no grad: (occ - 1.95 per point, min over blocks of ||local| - 5| per point), for the points `idx` or all"""
    with torch.no_grad():
        S, R, T, e1, e2 = _frames({k: x[k].double() for k in ('S', 'R_6d', 'T', 'sq_eps')})
        pts = sample_points(S, R, T, x['unit_samples'].double()).reshape(-1, 3)
        if idx is not None:
            pts = pts[idx]
        a = x['alpha_full'].double()
        N, C = S.shape[0], _chunk(pts.shape[0])
        occ = torch.zeros(pts.shape[0], dtype=torch.float64)
        gap = torch.full((pts.shape[0],), math.inf, dtype=torch.float64)
        for k0 in range(0, N, C):
            k1 = min(N, k0 + C)
            loc = block_local(pts, S, R, T, k0, k1)
            occ += (torch.sigmoid(-D.implicit_sq(loc, e1[k0:k1], e2[k0:k1]) / TEMPERATURE) * a[k0:k1, None]).sum(0)
            gap = torch.minimum(gap, (loc.abs() - CLAMP).abs().amin(dim=(0, 2)))
        return occ - OCC_LIMIT, gap


def sigmoid_maps(logits):
    """sigmoid with equal logits mapped to equal values, as the kernels compute them: torch's CPU float32 sigmoid can round
    one logit differently in its vectorised body and in its scalar tail, which would turn a plateau's exact zero differences
    into one-ulp ones"""
    u, inv = torch.unique(logits.detach(), return_inverse=True)
    s = torch.sigmoid(logits)
    return s + (torch.sigmoid(u)[inv] - s).detach()


def tv_pairs(maps, wrap):
    """the (v, u) neighbour differences TV takes of (M, H, W, 3) sigmoid maps, as two tensors (..., 3)"""
    dv = torch.diff(maps, dim=1)
    du = torch.diff(maps, dim=2, append=maps[:, :, 0:1]) if wrap else torch.diff(maps, dim=2)
    return dv, du


@functools.lru_cache(maxsize=None)
def reg_inputs(name):
    """float32 CPU leaves of case `name` (and its U(0,1) points when overlap is on), the points redrawn until every decision
    of the overlap term is clear of float32 rounding"""
    case = BY_NAME[name]
    g = _gen(7 + sum(map(ord, name)))
    N, P, E, B = case['n_blocks'], case['n_points'], case['env'], case['txt']
    x = {'texture_bkg': _maps(g, 1, E, case['maps']), 'texture_ground': _maps(g, 1, E, case['maps']),
         'textures': _maps(g, N, B, case['maps'])}
    x.update({k: v.float() for k, v in _blocks(g, case).items()})
    x['unit_samples'] = None
    if case['terms'] & OV:
        u = torch.rand(N * P, 3, generator=g)
        x['unit_samples'] = u.view(N, P, 3)
        idx = None
        for _ in range(100):
            exc, gap = overlap_decisions(x, idx)
            bad = (exc.abs() < OCC_MARGIN) | (gap < CLAMP_MARGIN)
            if not bad.any():
                break
            idx = (torch.arange(N * P) if idx is None else idx)[bad]
            u[idx] = torch.rand(len(idx), 3, generator=g)
        else:
            raise AssertionError(f'{name}: points near a decision after 100 redraws')
    return x


# ---------------------------------------------------------------------------------------------------------- the oracle
def _total_variation(bkg, ground, blocks, norm, coarse):
    f = 1.0 if coarse else 0.1
    n = TV_NORMS[norm]
    tv = sum(n(d).mean() for d in tv_pairs(sigmoid_maps(bkg), False))
    dv, du = tv_pairs(sigmoid_maps(blocks), True)
    tv = tv + n(du).sum(0).mean() + n(dv).sum(0).mean()
    tv = tv + sum(n(d).mean() for d in tv_pairs(sigmoid_maps(ground), False)) * f
    return f * tv


def oracle(case, x, dtype, device='cpu'):
    """(values {term: 0-d}, grads {leaf: tensor}) of the terms that are on, in `dtype` on `device`: the gradients of
    sum_term cotangent * value, for the leaves some term that is on reads.  The overlap term goes over chunks of blocks: the
    per-point occupancy without grad, then its gradient chunk by chunk."""
    cot, terms = cotangents(case), case['terms']
    wp, wt, wo = case['w']
    lv = {k: x[k].to(device, dtype).clone().requires_grad_(True) for k in LEAVES if READ_BY[k] & terms}
    vals, loss = {}, 0.
    if terms & PAR:
        vals['parsimony'] = wp * D.safe_pow(lv['alpha_full'], 0.5).mean()
    if terms & TV:
        vals['tv'] = wt * _total_variation(lv['texture_bkg'], lv['texture_ground'], lv['textures'], case['norm'], case['coarse'])
    for k, v in vals.items():
        loss = loss + cot[k] * v
    grads = dict(zip(lv, torch.autograd.grad(loss, list(lv.values()), allow_unused=True))) if vals else {k: None for k in lv}
    if terms & OV:
        val, g_ov = _overlap(lv, x['unit_samples'], wo, cot['overlap'])
        vals['overlap'] = val
        for k, g in g_ov.items():
            grads[k] = g if grads[k] is None else grads[k] + g
    grads = {k: torch.zeros_like(lv[k]) if g is None else g for k, g in grads.items()}
    return {k: v.detach() for k, v in vals.items()}, grads


def _overlap(lv, unit_samples, w, cot):
    S, R, T, e1, e2 = _frames(lv)
    a = lv['alpha_full']
    pts = sample_points(S, R, T, unit_samples).reshape(-1, 3)
    N, M = S.shape[0], pts.shape[0]
    C = _chunk(M)

    def occ(k0, k1):
        loc = block_local(pts, S, R, T, k0, k1)
        return (torch.sigmoid(-D.implicit_sq(loc, e1[k0:k1], e2[k0:k1]) / TEMPERATURE) * a[k0:k1, None]).sum(0)

    with torch.no_grad():
        excess = sum(occ(k0, min(N, k0 + C)) for k0 in range(0, N, C)) - OCC_LIMIT
        val = w * excess.clamp(min=0).mean()
    g_pt = (excess >= 0).to(excess) * (cot * w / M)                     # clamp(min=0), then the mean
    names = ('S', 'R_6d', 'T', 'sq_eps', 'alpha_full')
    grads = {k: torch.zeros_like(lv[k]) for k in names}
    for k0 in range(0, N, C):
        gs = torch.autograd.grad((occ(k0, min(N, k0 + C)) * g_pt).sum(), [lv[k] for k in names], retain_graph=True,
                                 allow_unused=True)
        for k, g in zip(names, gs):
            if g is not None:
                grads[k] += g
    return val, grads


@functools.lru_cache(maxsize=None)
def oracle64(name):
    """the float64 oracle of case `name` (on the device when there is one), on the CPU"""
    dev = 'cuda' if torch.cuda.is_available() else 'cpu'
    vals, grads = oracle(BY_NAME[name], reg_inputs(name), torch.float64, dev)
    return {k: v.cpu() for k, v in vals.items()}, {k: v.cpu() for k, v in grads.items()}


# ---------------------------------------------------------------------------------------------------------- the C-ABI
def reg_struct(case, ptrs):
    """DbwRegularisers of `case` with device pointers `ptrs` (leaf name or 'unit_samples' -> int or None); the weights of
    terms that are off are NaN: no kernel reads them"""
    from dbw_b200 import _lib
    wp, wt, wo = (float('nan') if v is None else v for v in case['w'])
    return _lib.DbwRegularisers(*[ptrs.get(k) for k in LEAVES + ('unit_samples',)], n_blocks=case['n_blocks'],
                                n_points=case['n_points'], env_size=case['env'], txt_size=case['txt'], terms=case['terms'],
                                tv_norm=TV_CODES[case['norm']], coarse=int(case['coarse']), ratio_block_scene=RATIO,
                                scale_min=SCALE_MIN, w_parsimony=wp, w_tv=wt, w_overlap=wo)


TAIL, SENTINEL = 256, 0x5A


def run_cabi(case, x, dev, drop=None):
    """forward and backward through the raw entries on NaN-prefilled outputs, the gradient output `drop` NULL.  Inputs no term
    that is on reads are NULL; the workspace is exactly the reported size, followed by a sentinel tail.
    Returns ({term: value}, {leaf: gradient buffer}, the three forward outputs, the workspace buffer, its reported size)."""
    from dbw_b200 import _lib
    from dbw_b200.renderer import _stream
    L = _lib.lib()
    terms = case['terms']
    ins = {k: x[k].to(dev).contiguous() for k in LEAVES if READ_BY[k] & terms}
    if terms & OV:
        ins['unit_samples'] = x['unit_samples'].to(dev).contiguous()
    r = reg_struct(case, {k: t.data_ptr() for k, t in ins.items()})
    nbytes = ctypes.c_size_t(0)
    _lib.check(L.dbw_regularisers_workspace_bytes(ctypes.byref(r), ctypes.byref(nbytes)), 'dbw_regularisers_workspace_bytes')
    ws = torch.full((nbytes.value + TAIL,), SENTINEL, dtype=torch.uint8, device=dev)
    out = torch.full((3,), float('nan'), device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(L.dbw_regularisers_forward(ctypes.byref(r), p(out[0:1]), p(out[1:2]), p(out[2:3]), p(ws), nbytes.value, _stream()),
               'dbw_regularisers_forward')
    cot = cotangents(case)
    g_up = torch.tensor([cot[n] for _, n in TERMS], device=dev)
    grads = {k: torch.full(x[k].shape, float('nan'), device=dev) for k in LEAVES}
    _lib.check(L.dbw_regularisers_backward(ctypes.byref(r), *[p(g_up[i:i + 1]) if terms & bit else None for i, (bit, _) in enumerate(TERMS)],
                                           *[p(grads[k]) if k != drop else None for k in LEAVES], p(ws), nbytes.value, _stream()),
               'dbw_regularisers_backward')
    torch.cuda.synchronize()
    vals = {n: out[i] for i, (bit, n) in enumerate(TERMS) if terms & bit}
    return vals, grads, out, ws, nbytes.value


@pytest.mark.parametrize('name', CASE_IDS)
def test_cabi_matches_the_float64_oracle(name):
    """dbw_regularisers_forward / _backward: every value and every leaf gradient; the outputs of terms that are off and the
    workspace tail keep what the caller left there"""
    case, dev = BY_NAME[name], torch.device('cuda:0')
    x = reg_inputs(name)
    want_vals, want_grads = oracle64(name)
    vals, grads, out, ws, nbytes = run_cabi(case, x, dev)
    assert (ws[nbytes:] == SENTINEL).all(), 'the kernels wrote past the reported workspace'
    for i, (bit, n) in enumerate(TERMS):
        if case['terms'] & bit:
            check(f'val.{n}', vals[n], want_vals[n], name)
        else:
            assert torch.isnan(out[i]), (name, n)
    for k in LEAVES:
        if READ_BY[k] & case['terms']:
            check(f'g.{k}', grads[k], want_grads[k], name)
        else:
            assert torch.isnan(grads[k]).all(), (name, k)


@pytest.mark.parametrize('name', CASE_IDS)
def test_library_call_matches_the_float64_oracle(name):
    """losses.regularisers: the weighted terms of `weights` and, through autograd, every leaf gradient (None for the leaves
    no term that is on reads)"""
    from dbw_b200 import losses as L
    case, dev = BY_NAME[name], torch.device('cuda:0')
    x = reg_inputs(name)
    want_vals, want_grads = oracle64(name)
    q = {k: x[k].to(dev).requires_grad_(True) for k in LEAVES}
    weights = {n: case['w'][i] for i, (bit, n) in enumerate(TERMS) if case['terms'] & bit}
    u = x['unit_samples'].to(dev) if x['unit_samples'] is not None else None
    got = L.regularisers(*[q[k] for k in LEAVES], weights, case['norm'], case['coarse'], RATIO, SCALE_MIN, unit_samples=u)
    assert list(got) == list(weights)
    cot = cotangents(case)
    for n in got:
        check(f'val.{n}', got[n], want_vals[n], name)
    grads = torch.autograd.grad(sum(cot[n] * v for n, v in got.items()), [q[k] for k in LEAVES], allow_unused=True)
    for k, g in zip(LEAVES, grads):
        if READ_BY[k] & case['terms']:
            assert g is not None, (name, k)
            check(f'g.{k}', g, want_grads[k], name)
        else:
            assert g is None, (name, k)


@pytest.mark.parametrize('name', ['n129-p256-wide', 'n2-p257', 'PO'])
def test_each_null_gradient_output_leaves_the_others_bits(name):
    """every gradient output NULL on its own: it is skipped, and the others are the bits of the call with all of them"""
    case, dev = BY_NAME[name], torch.device('cuda:0')
    x = reg_inputs(name)
    _, full, _, _, _ = run_cabi(case, x, dev)
    for drop in LEAVES:
        if not READ_BY[drop] & case['terms']:
            continue
        _, grads, _, _, _ = run_cabi(case, x, dev, drop=drop)
        assert torch.isnan(grads[drop]).all(), (name, drop)
        for k in LEAVES:
            if k != drop and READ_BY[k] & case['terms']:
                assert torch.equal(grads[k], full[k]), (name, drop, k)
