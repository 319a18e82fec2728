"""GPU: the loss-epilogue raster kernel and the blocks backward it runs itself, against the float64 oracle of one step.

Every training step renders its blocks pass through `raster_forward_kernel<NT, true>` (fused_loss.scene_mse): the kernel
composites over the environment render, takes the squared error and, in the coarse phase (detach_bary over cell maps), also
differentiates the pass on the fragment lists still in shared memory (`epilogue_backward`, folded later by
dbw_render_backward_deferred).  The cases below pin that path to the oracle of the same step, element by element:

    env  = D.render(environment, K = 1, sigma = 0)
    fg   = D.render(blocks, K, sigma, detach_bary, faces_alpha)
    rec  = fg_rgb * a + (1 - a) * env_rgb
    loss = sum((rec - imgs)^2) / (n_views * 3 * H * W)                         all in float64 autograd

with the env vertices and maps, the block vertices, the block CELLS (expanded to the atlas as test_raster_matrix_gpu's
test_map_layouts does), the opacities and, where a case asks, R and T as leaves.  Each case runs twice, with
fused_loss.FUSE_BLOCKS_BACKWARD on and off; both runs must meet the oracle bar, and a case that is not eligible for the
fused path (atlas maps, a pass that is not detached) asserts that it did not take it.

Decisions: the kept face ids of each pass come from render_scene with the pass's settings; scene_mse's `rec` must equal the
composite of those two renders (so both took the same decisions).  Where either pass's ids differ from the oracle's, each side's
target is its own `rec`: zero residual and zero gradient on both sides.  Their share is bounded and printed.

Bars (those of test_raster_matrix_gpu): `rec` within 1e-4 on the other pixels, the loss within 1e-5 relative, every leaf
within 1e-3 relative L2 and 2e-3 of its largest magnitude.  Only the fine-phase and the benched-shape cases widen them,
and only to what the oracle's own float32 evaluation of the step shows against float64 (see their docstrings).

Each case also asserts the kernel branch it exists for: the forward entry fused_loss called (spied), the number of opacity
entries per view against the 512 the kernel sums in shared memory (DBW_ALPHA_SMEM_MAX; more go through global atomics and
the deferred fold's scale_add_kernel), and for the crowded scenes a host-side lower bound on the faces some tile lists,
against the list capacity beyond which the kernel takes its chunked path."""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import dbw_path as D
from oracle import pt3d
from tests.helpers import decision_mask
from tests.test_fused_blocks_grad_gpu import _Spy
from tests.test_raster_matrix_gpu import (BANDS, GRAD_ELEM, GRAD_REL, IMG_TOL, SHAPES, _alpha, _away_views, _cams,
                                          _close_to_cuda, _close_to_oracle, _expand, _pack_maps, _rel, _split_maps)

pytestmark = pytest.mark.gpu

LOSS_REL = 1e-5
REC_EQ = 1e-6                # scene_mse's rec vs the composite of the two id renders
ALPHA_SMEM_MAX = 512         # DBW_ALPHA_SMEM_MAX: opacity entries per view summed in shared memory
LEAVES = ('ev', 'em', 'bv', 'bm', 'ba', 'R', 'T')
NAMES = {'ev': 'env verts', 'em': 'env maps', 'bv': 'blocks verts', 'bm': 'blocks cells', 'ba': 'alpha', 'R': 'R', 'T': 'T'}


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _nt(Kf):
    """block size of the forward kernel (DBW_FWD_NT_SMALLK for K <= 4) and its tile-list capacity CAP"""
    return (256, 256) if Kf <= 4 else (128, 64)


def _case(**kw):
    c = dict(nb=4, txt=16, seed=13, boxy=False, crowd=None, cells=(4, 3, 1), Kf=10, sigma=1e-4, detach=True, alpha='batch',
             size=(40, 56), n_views=2, dist=2.0, fx=None, ring49=False, away=False, z_clip=0.001, zero_area=False, scale=1.0,
             poses=False, bands=False, max_amb=2e-3, big_alpha=None, fp32_model=False, model_cells=False, yaw=0.0)
    assert set(kw) <= set(c), set(kw) - set(c)
    c.update(kw)
    return c


# ------------------------------------------------------------------------------------------------ the step, both sides
def _world(c):
    """scene, opacities, cameras and target of one case (float64, CPU)"""
    nb, TS = c['nb'], c['txt']
    tpl = D.SceneTemplate(n_blocks=nb, txt_size=TS)
    p = D.init_params(nb, TS, seed=c['seed'], boxy=c['boxy'], dtype=torch.float64)
    if c['crowd']:
        p['T'] = p['T'] * c['crowd']
    env = tpl.build_env(p)
    blocks, _ = tpl.build_blocks(p)
    w = {'tpl': tpl, 'env': env, 'n_bkg_v': tpl.bkg_verts.shape[0], 'n_bkg_f': tpl.bkg_faces.shape[0]}
    faces, fvu, fmap = blocks['faces'], blocks['faces_verts_uvs'], blocks['face_map']
    if c['cells']:
        f, pl, pr = c['cells']
        CS, Wt = TS // f, TS + pl + pr
        faces_uvs, verts_uvs = D.get_icosphere_uvs(1)
        fvu = torch.stack([(verts_uvs[:, 0].double() * TS + pl) / Wt, verts_uvs[:, 1].double()], -1)[faces_uvs].repeat(nb, 1, 1)
        fmap = torch.arange(nb).repeat_interleave(tpl.BNF)
        if c['model_cells']:        # the model's: its texture parameters through the sigmoid, box-decimated f times
            w['bm'] = F.avg_pool2d(torch.sigmoid(p['textures']).permute(0, 3, 1, 2), f).permute(0, 2, 3, 1).contiguous()
        else:
            w['bm'] = torch.rand(nb, CS, CS, 3, generator=torch.Generator().manual_seed(c['seed'] + f + pl), dtype=torch.float64)
    else:
        w['bm'] = [m.detach() for m in blocks['maps']]
    if c['zero_area']:            # as test_raster_matrix_gpu.test_zero_area_faces: a repeated vertex, at face ids 100 and 101
        faces = torch.cat([faces[:100], torch.tensor([[5, 5, 60], [7, 30, 30]]), faces[100:]])
        fvu = torch.cat([fvu[:100], fvu[:2], fvu[100:]])
        fmap = torch.cat([fmap[:100], torch.tensor([1, 2]), fmap[100:]])
    w['blk'] = {'verts': blocks['verts'].detach(), 'faces': faces, 'faces_verts_uvs': fvu.detach(), 'face_map': fmap}
    if c['ring49']:
        R, T, K = D.ring_cameras(49, dtype=torch.float64)
        R, T = R[[0, 24, 48]], T[[0, 24, 48]]
    else:
        R, T, K = _cams(c['n_views'], seed=c['seed'], dist=c['dist'])
    if c['yaw']:                   # the ring turned about the world's vertical axis (the cameras still look at the origin)
        cy, sy = math.cos(c['yaw']), math.sin(c['yaw'])
        R = torch.tensor([[cy, 0., -sy], [0., 1., 0.], [sy, 0., cy]], dtype=R.dtype) @ R
    if c['away']:
        R, T = _away_views(R, T)
    if c['fx']:
        K = K.clone()
        K[0, 0] = K[1, 1] = c['fx']
    B = R.shape[0]
    bnf = 1 if c['zero_area'] else tpl.BNF
    w['ba'], fa_ref, w['group'] = _alpha(c['alpha'], B, faces.shape[0], bnf, seed=c['seed'] + c['Kf'])
    if fa_ref is not None:        # the layout as an index into the opacity leaf, whose entries are distinct random draws
        w['alpha_idx'] = (fa_ref.detach()[:, None] == w['ba'].detach()[None]).int().argmax(1)
        assert torch.equal(w['ba'].detach()[w['alpha_idx']], fa_ref.detach())
    w.update(R=R, T=T, K=K, B=B, imgs=torch.rand(B, 3, *c['size'], generator=torch.Generator().manual_seed(c['seed']),
                                                dtype=torch.float64))
    return w


def _leaves(w, c, dtype=torch.float64):
    """fresh oracle leaves of one evaluation"""
    leaf = lambda t, on=True: t.detach().to(dtype).clone().requires_grad_(on)
    return {'ev': leaf(w['env']['verts']), 'em': [leaf(m) for m in w['env']['maps']], 'bv': leaf(w['blk']['verts']),
            'bm': leaf(w['bm']) if c['cells'] else [leaf(m) for m in w['bm']], 'ba': None if w['ba'] is None else leaf(w['ba']),
            'R': leaf(w['R'], c['poses']), 'T': leaf(w['T'], c['poses'])}


def _oracle_rec(w, c, L):
    """(rec, env fragments, blocks fragments) of the oracle step"""
    dt = L['ev'].dtype
    ev = L['ev']
    if not c['poses']:
        # the background sphere is static (n_static_faces): its vertices reach the oracle as constants.  With pose gradients
        # the library differentiates it too (it moves in the image when the camera moves)
        keep = torch.ones(ev.shape[0], 1, dtype=dt)
        keep[:w['n_bkg_v']] = 0
        ev = ev * keep + ev.detach() * (1 - keep)
    env = dict(w['env'], verts=ev, maps=L['em'], faces_verts_uvs=w['env']['faces_verts_uvs'].to(dt))
    K = w['K'].to(dt)
    env_rgba, fe = D.render(env, L['R'], L['T'], K, c['size'], sigma=0, faces_per_pixel=1, z_clip=0.001, return_fragments=True)
    maps = list(_expand(L['bm'], *c['cells']).unbind(0)) if c['cells'] else L['bm']
    blk = dict(w['blk'], verts=L['bv'], maps=maps, faces_verts_uvs=w['blk']['faces_verts_uvs'].to(dt))
    fa = None if L['ba'] is None else L['ba'][w['alpha_idx']]
    fg, fb = D.render(blk, L['R'], L['T'], K, c['size'], sigma=c['sigma'], faces_per_pixel=c['Kf'], z_clip=c['z_clip'],
                      detach_bary=c['detach'], faces_alpha=fa, return_fragments=True)
    a = fg[:, 3:]
    return fg[:, :3] * a + (1 - a) * env_rgba[:, :3], fe, fb


def _flat(L):
    keys, out = [], []
    for k in LEAVES:
        v = L[k]
        if v is None or (k in ('R', 'T') and not v.requires_grad):
            continue
        for i, t in enumerate(v if isinstance(v, list) else [v]):
            keys.append((k, i))
            out.append(t)
    return keys, out


def _oracle_grads(w, c, L, rec, amb):
    """loss and {(leaf, part): gradient} of the oracle step whose target is its own rec on the `amb` pixels"""
    target = torch.where(amb, rec.detach(), w['imgs'].to(rec.dtype))
    loss = ((rec - target) ** 2).sum() / rec.numel()
    keys, leaves = _flat(L)
    g = torch.autograd.grad(loss * c['scale'], leaves, allow_unused=True)
    return loss.item(), {k: (torch.zeros_like(t) if gi is None else gi).double() for k, t, gi in zip(keys, leaves, g)}


def _device_step(w, c, dev):
    """CUDA inputs and the two ScenePass descriptions of the step (as DifferentiableBlocksWorld._scene_mse_fused builds them)"""
    from dbw_b200 import Renderer
    from dbw_b200.fused_loss import ScenePass
    H, W = c['size']

    def renderer(z_clip, **kw):
        r = Renderer((H, W), z_clip=z_clip, cameras={'name': 'perspective'}, **kw).to(dev)
        r.update_cameras(device=dev, K=w['K'].float()[None].to(dev))
        return r

    env, blk = w['env'], w['blk']
    em, et = _pack_maps(env['maps'], True)
    if c['cells']:
        f, pl, pr = c['cells']
        nb, CS = w['bm'].shape[:2]
        bm = F.pad(w['bm'].float(), (0, 1)).reshape(-1)
        tb = [(i * CS * CS * 3, c['txt'], c['txt'] + pl + pr, (pl << 8) | f) for i in range(nb)]
    else:
        bm, tb = _pack_maps(w['bm'], True)
    i32 = lambda t: t.to(dev).to(torch.int32)
    leaf = lambda t, on=True: t.detach().float().to(dev).contiguous().requires_grad_(on)
    x = dict(ev=leaf(env['verts']), em=leaf(em), bv=leaf(blk['verts']), bm=leaf(bm),
             ba=None if w['ba'] is None else leaf(w['ba']), R=leaf(w['R'], c['poses']), T=leaf(w['T'], c['poses']),
             fmap=i32(blk['face_map']), et=et, tb=tb)
    env_pass = ScenePass(i32(env['faces']), env['faces_verts_uvs'].to(dev), i32(env['face_map']), et,
                         renderer(0.001, faces_per_pixel=1, sigma=0), n_static_faces=w['n_bkg_f'])
    blk_pass = ScenePass(i32(blk['faces']), blk['faces_verts_uvs'].to(dev), i32(blk['face_map']), tb,
                         renderer(c['z_clip'], faces_per_pixel=c['Kf'], sigma=c['sigma'], detach_bary=c['detach']),
                         alpha_group=w['group'])
    return x, env_pass, blk_pass


def _pass_ids(x, p, verts, maps, fa, fmap):
    """(RGBA, kept slot ids) of one pass, rendered on its own with the pass's settings"""
    from dbw_b200 import render_scene
    r = p.r
    with torch.no_grad():
        return render_scene(verts, p.faces, p.faces_uvs, fmap, maps, p.map_table_host, x['R'], x['T'], r.cameras.intrinsics(),
                            r.img_size, r.sigma, r.faces_per_pixel, r.z_clip, r.detach_bary, r.clip_inside, r.background_color,
                            fa, r.perspective_correct, blur_radius=r.blur_radius, return_ids=True, maps_are_texels4=True,
                            alpha_group=p.alpha_group, n_static_faces=p.n_static_faces)


@contextlib.contextmanager
def _spying():
    """records (entry, args) of every library call, fused_loss's included"""
    from dbw_b200 import _lib
    real = _lib.lib
    spy = _Spy(real())
    _lib.lib = lambda: spy
    try:
        yield spy
    finally:
        _lib.lib = real


def _scene_mse(x, env_pass, blk_pass, imgs, fused, view_rows=None, scale=1.0):
    """(loss, rec, {leaf: gradient}, library calls) of one CUDA step with fused_loss.FUSE_BLOCKS_BACKWARD = `fused`"""
    from dbw_b200 import fused_loss
    old, fused_loss.FUSE_BLOCKS_BACKWARD = fused_loss.FUSE_BLOCKS_BACKWARD, fused
    try:
        with _spying() as spy:
            loss, rec = fused_loss.scene_mse(x['ev'], x['em'], x['bv'], x['bm'], x['ba'], x['R'], x['T'], imgs, env_pass, blk_pass,
                                             x['fmap'], return_rec=True, view_rows=view_rows)
            keys = [k for k in LEAVES if x[k] is not None and x[k].requires_grad]
            g = torch.autograd.grad(loss * scale, [x[k] for k in keys])
            torch.cuda.synchronize()
    finally:
        fused_loss.FUSE_BLOCKS_BACKWARD = old
    return loss.item(), rec, dict(zip(keys, g)), spy.calls


def _to_oracle_layout(x, c, k, g):
    """a CUDA gradient as the list of tensors shaped like the oracle's leaf parts"""
    g = g.detach().cpu().double()
    if k == 'em':
        return _split_maps(g, x['et'], True)
    if k == 'bm':
        if c['cells']:
            nb, CS = len(x['tb']), c['txt'] // c['cells'][0]
            return [g.reshape(nb, CS, CS, 4)[..., :3]]
        return _split_maps(g, x['tb'], True)
    return [g]


def _check_branch(calls, c, w, fused_on):
    """the entry fused_loss called and the opacity-sum branch the kernel takes"""
    names = [n for n, _ in calls]
    eligible = c['detach'] and bool(c['cells'])
    fused = 'dbw_render_forward_loss_grad' in names
    assert fused == (fused_on and eligible), (fused_on, eligible, names)
    assert ('dbw_render_forward_loss' in names) == (not fused), names
    assert ('dbw_render_backward_deferred' in names) == fused, names
    (cfg,) = [a[0]._obj for n, a in calls if n in ('dbw_render_forward_loss_grad', 'dbw_render_forward_loss')]
    n_alpha = cfg.n_faces // cfg.alpha_group
    assert cfg.faces_per_pixel == c['Kf'] and bool(cfg.detach_bary) == c['detach']
    if c['big_alpha'] is not None:
        assert w['ba'] is not None and (n_alpha > ALPHA_SMEM_MAX) == c['big_alpha'], (n_alpha, c['big_alpha'])
    return fused, n_alpha


def _run(c, tag, dev=None):
    """the oracle step once, the CUDA step with the fused path on and off; returns the world, the CUDA inputs and passes, the
    ambiguous pixels, the oracle's blocks fragments, the CUDA blocks ids and each run's (rec, gradients)"""
    dev = dev or _dev()
    w = _world(c)
    L = _leaves(w, c)
    rec_ref, fe, fb = _oracle_rec(w, c, L)
    x, env_pass, blk_pass = _device_step(w, c, dev)
    env_rgba, ids_e = _pass_ids(x, env_pass, x['ev'], x['em'], None, env_pass.face_map)
    fg_rgba, ids_b = _pass_ids(x, blk_pass, x['bv'], x['bm'], x['ba'], x['fmap'])
    a = fg_rgba[:, 3:]
    rec_ids = fg_rgba[:, :3] * a + (1 - a) * env_rgba[:, :3]
    same = decision_mask(ids_e, fe, w['env']['faces'].shape[0]) * decision_mask(ids_b, fb, w['blk']['faces'].shape[0])
    amb = same == 0
    share = amb.double().mean().item()
    B, _, H, W = rec_ref.shape
    assert share <= max(c['max_amb'], 1.5 / (B * H * W)), f'{tag}: {share * 100:.3f}% of pixels take a different discrete decision'
    loss_ref, g_ref = _oracle_grads(w, c, L, rec_ref, amb)
    rec_tol, bars = IMG_TOL, {}
    if c['fp32_model']:
        rec_tol, bars = _fp32_model(w, c, rec_ref, fe, fb, amb)
    imgs = w['imgs'].float().to(dev)
    amb_d = amb.to(dev)
    results = {}
    for fused_on in (True, False):
        # first pass: this side's own rec (the target of its ambiguous pixels)
        _, rec, _, calls = _scene_mse(x, env_pass, blk_pass, imgs, fused_on)
        assert (rec - rec_ids).abs().max().item() <= REC_EQ, f'{tag}: scene_mse rec differs from the composite of the id renders'
        fused, n_alpha = _check_branch(calls, c, w, fused_on)
        target = torch.where(amb_d, rec, imgs)
        if c['bands']:
            loss, g = 0.0, None
            for rows in BANDS:
                l, _, gb, _ = _scene_mse(x, env_pass, blk_pass, target, fused_on, torch.tensor(rows, dtype=torch.int32, device=dev),
                                         c['scale'])
                loss += l
                g = gb if g is None else {k: g[k] + gb[k] for k in g}
        else:
            loss, _, g, _ = _scene_mse(x, env_pass, blk_pass, target, fused_on, scale=c['scale'])
        err = ((rec.cpu().double() - rec_ref.detach()).abs() * (~amb)).max().item()
        assert err <= rec_tol, f'{tag}: rec max err {err:.3e}'
        lrel = abs(loss - loss_ref) / abs(loss_ref)
        assert lrel <= LOSS_REL, f'{tag}: loss {loss:.9e} vs oracle {loss_ref:.9e}'
        worst = []
        for k, gk in g.items():
            for i, gi in enumerate(_to_oracle_layout(x, c, k, gk)):
                ref = g_ref[(k, i)]
                name = 'blocks maps' if k == 'bm' and not c['cells'] else NAMES[k]
                name += f'[{i}]' if k == 'em' or (k == 'bm' and not c['cells']) else ''
                scale = ref.abs().max().item()
                worst.append((name, _rel(gi, ref) if scale else 0.0, (gi - ref).abs().max().item() / scale if scale else 0.0))
                _close_to_oracle(gi, ref, f'{tag} fused={fused} {name}', *bars.get((k, i), (GRAD_REL, GRAD_ELEM)))
        print(f'\n{tag} [fused={fused} NT={_nt(c["Kf"])[0]} n_alpha={n_alpha if w["ba"] is not None else 0}]: ambiguous {share * 100:.3f}%, '
              f'rec err {err:.1e}, loss rel {lrel:.1e}; worst rel / elem: '
              + ', '.join(f'{n} {r:.1e}/{e:.1e}' for n, r, e in sorted(worst, key=lambda t: -t[1])[:3]))
        results[fused_on] = (rec, g)
    return {'w': w, 'x': x, 'passes': (env_pass, blk_pass), 'amb': amb, 'fb': fb, 'ids_b': ids_b, 'results': results}


def _fp32_model(w, c, rec64, fe64, fb64, amb):
    """what float32 can deliver on this step: the oracle's own float32 evaluation against its float64 one, on the pixels where
    both take the float64 decisions.  rec bar: 2x its deviation (test_baseline_shapes_gpu.test_cfg2_blocks_pass_fine_400x400);
    gradient bars, per leaf: 3x its deviation (test_raster_matrix_gpu.test_z_clipped_scene_with_and_without_perspective_correction),
    never below the default bars"""
    L32 = _leaves(w, c, torch.float32)
    rec32, fe32, fb32 = _oracle_rec(w, c, L32)
    same32 = ((fe32.pix_to_face == fe64.pix_to_face).all(-1) & (fb32.pix_to_face == fb64.pix_to_face).all(-1))[:, None]
    amb32 = amb | ~same32
    _, g32 = _oracle_grads(w, c, L32, rec32, amb32)
    L64 = _leaves(w, c)
    rec64b, _, _ = _oracle_rec(w, c, L64)
    _, g64 = _oracle_grads(w, c, L64, rec64b, amb32)
    rec_dev = ((rec32.detach().double() - rec64.detach()).abs() * (~amb32)).max().item()
    bars = {}
    for k, g in g64.items():
        scale = g.abs().max().item()
        if scale > 0:
            rel, elem = _rel(g32[k], g), (g32[k] - g).abs().max().item() / scale
            bars[k] = (max(GRAD_REL, 3 * rel), max(GRAD_ELEM, 3 * elem))
            print(f'\nfloat32 oracle vs float64: {NAMES[k[0]]}[{k[1]}] rel {rel:.2e}, elem {elem:.2e}', end='')
    print(f'\nfloat32 oracle vs float64: rec {rec_dev:.2e}')
    return max(IMG_TOL, 2 * rec_dev), bars


# ------------------------------------------------------------------------------------------------ 1. K x opacity layout
# 7 blocks = 560 faces: per-face layouts have more than 512 entries per view (global atomics + scale_add_kernel), per-block
# layouts 7 (shared-memory sums).  6 blocks = 480 per-face entries: the shared-memory path with per-face opacities.
K_LAYOUT = [
    (1, None, 7), (1, 'face', 7), (2, 'batch_face', 7), (3, 'block', 7), (3, 'face', 6), (4, 'face', 7), (4, 'batch', 7),
    (5, 'face', 7), (5, 'block', 7), (9, 'batch_face', 7), (10, 'face', 6), (10, 'batch', 7), (16, 'face', 7),
    (25, 'batch_face', 7), (26, 'block', 7), (40, 'face', 7), (64, 'batch_face', 7), (64, None, 7),
]


def _big_alpha(alpha, nb):
    return None if alpha is None else (alpha in ('face', 'batch_face') and nb * 80 > ALPHA_SMEM_MAX)


def test_k_layout_table_covers_both_opacity_branches_at_both_block_sizes():
    """on each side of the K = 4 / 5 switch of the forward block size there are per-face cases above and at most 512 entries"""
    for nt in (256, 128):
        kinds = {_big_alpha(a, nb) for k, a, nb in K_LAYOUT if _nt(k)[0] == nt and a in ('face', 'batch_face')}
        assert kinds == {True, False}, (nt, kinds)
        assert any(_nt(k)[0] == nt and a in ('block', 'batch') for k, a, nb in K_LAYOUT), nt


@pytest.mark.parametrize('Kf,alpha,nb', K_LAYOUT)
def test_faces_per_pixel_and_opacity_layout(Kf, alpha, nb):
    r = _run(_case(nb=nb, seed=3, Kf=Kf, alpha=alpha, size=(48, 64), big_alpha=_big_alpha(alpha, nb)),
             f'K={Kf} alpha={alpha} blocks={nb}')
    if Kf in (3, 16):
        assert (r['fb'].pix_to_face[..., -1] >= 0).any(), 'K is never exceeded'


# ------------------------------------------------------------------------------------------------ 2. map layouts
@pytest.mark.parametrize('f,p_left,p_right', [(2, 0, 0), (2, 3, 4), (4, 3, 1), (8, 0, 5), (16, 3, 2)])
def test_cell_map_layouts(f, p_left, p_right):
    """float4 cell maps of 32 x 32 textures decimated f times, circularly padded by (p_left, p_right) texels, p_left not
    always a multiple of f; the gradient is compared in cell space"""
    _run(_case(txt=32, seed=10, cells=(f, p_left, p_right), alpha='face', size=(64, 64), big_alpha=False),
         f'cells f={f} p=({p_left},{p_right})')


def test_float4_atlas_maps_are_never_fused():
    _run(_case(txt=32, seed=10, cells=None, alpha='face', size=(64, 64)), 'float4 atlas')


# ------------------------------------------------------------------------------------------------ 3. the benched shape
def test_model_shape_400x400():
    """3 ring views at 400 x 400, 10 blocks with 256^2 textures as 8x decimated cells padded like the model's (23 columns:
    256 x 279), K = 10, one opacity per (view, block).  The cells are the model's own (its initial textures, box-decimated):
    with cells drawn uniformly in [0, 1] instead, the float32 rounding of a few halo opacities shows at 400 x 400 -- the
    oracle's own float32 evaluation deviates from float64 by up to 7.6e-4 at the pixels where this path deviates by 2.8e-4.
    The ground passes under these cameras: its z-clipped faces have vertices at z = z_clip, ~1e3 NDC units off screen, and
    the environment vertex gradient carries ~1e-3 relative rounding noise in any float32 evaluation
    (test_baseline_shapes_gpu._leaf_gradient_parity), so each leaf's bar is 3x what the float32 oracle shows for it"""
    tpl = D.SceneTemplate(n_blocks=10, txt_size=256)
    assert tpl.txt_padding == (0, 23)
    _run(_case(nb=10, txt=256, seed=5, cells=(8, *tpl.txt_padding), model_cells=True, alpha='batch', size=(400, 400),
               ring49=True, big_alpha=False, fp32_model=True), 'model shape 400x400')


# ------------------------------------------------------------------------------------------------ 4. not detached, fine phase
@pytest.mark.parametrize('Kf', [3, 10])
def test_not_detached_is_never_fused(Kf):
    """detach_bary = False over cell maps: the barycentric vertex gradient needs the two-kernel path"""
    _run(_case(seed=4, Kf=Kf, detach=False, alpha='face', size=(48, 64)), f'not detached K={Kf}')


def test_fine_phase_over_atlas_maps():
    """fine phase: sigma = 5e-6, full-resolution atlas maps, no opacities.  The opacity exp(-d / sigma) of a halo pixel
    amplifies the float32 rounding of the squared distance by 1 / sigma; the oracle's own float32 evaluation of the step
    deviates from its float64 one by more than the default bars, so the bars are 2x its rec deviation and 3x its gradient
    deviation (computed here, on the pixels where float32 and float64 take the same decisions)"""
    _run(_case(nb=5, txt=32, seed=6, boxy=True, cells=None, alpha=None, sigma=5e-6, size=(96, 128), fp32_model=True),
         'fine sigma=5e-6')


# ------------------------------------------------------------------------------------------------ 5. image shapes
@pytest.mark.parametrize('mode', ['soft', 'k3'])
@pytest.mark.parametrize('size', SHAPES)
def test_image_shapes(size, mode):
    """images narrower or shorter than one tile, 1 x N and N x 1, not multiples of the tile: lanes that are not live take
    part in the warp-uniform loops of epilogue_backward.  The ring is turned by 0.1 rad: unturned, both cameras look along the
    world plane x = 0, which holds edges of the ground's grid, and at odd widths the middle pixel column lies exactly on them
    (a tie that float32 and float64 break differently at every pixel of the column)"""
    Kf, alpha = (10, 'batch') if mode == 'soft' else (3, 'face')
    _run(_case(seed=15, Kf=Kf, alpha=alpha, size=size, yaw=0.1), f'{size} {mode}')


# ------------------------------------------------------------------------------------------------ 6. views that see nothing
def test_many_views_and_views_that_see_nothing():
    """17 views: 15 on a ring, one turned away from the scene and one whose frustum misses it.  On the last two `rec` is the
    environment render exactly, and a residual there gives the blocks leaves exactly zero gradient"""
    dev = _dev()
    r = _run(_case(seed=16, alpha='batch', size=(24, 32), n_views=15, away=True), '17 views')
    x, (env_pass, blk_pass) = r['x'], r['passes']
    assert r['w']['B'] == 17
    env_rgba, _ = _pass_ids(x, env_pass, x['ev'], x['em'], None, env_pass.face_map)
    for fused_on in (True, False):
        rec, _ = r['results'][fused_on]
        assert torch.equal(rec[15:], env_rgba[15:, :3]), fused_on
        target = rec.clone()
        target[15:] = torch.rand(2, *target.shape[1:], generator=torch.Generator().manual_seed(16)).to(dev)
        _, _, g, _ = _scene_mse(x, env_pass, blk_pass, target, fused_on)
        for k in ('bv', 'bm', 'ba'):
            assert torch.isfinite(g[k]).all() and g[k].abs().max() == 0, (fused_on, k)
        assert g['em'].abs().max() > 0, fused_on


# ------------------------------------------------------------------------------------------------ 7. row bands
@pytest.mark.parametrize('Kf,alpha', [(10, 'batch'), (3, 'face')])
def test_row_bands_sum_to_the_oracle_gradient(Kf, alpha):
    """view_rows: the gradients of a partition of the rows (an empty and a one-row band among them) sum to the oracle's
    gradient of the whole image, and the band losses to its loss"""
    _run(_case(seed=12, Kf=Kf, alpha=alpha, size=(72, 40), bands=True), f'row bands K={Kf}')


# ------------------------------------------------------------------------------------------------ 8. z-clipping
def test_z_clipped_block_faces():
    """the camera among the blocks: block faces straddle z_clip and are split (second-triangle slots, conversion matrices);
    face_setup_backward_kernel folds their gradients back"""
    r = _run(_case(nb=3, txt=32, seed=5, Kf=8, alpha='block', size=(48, 48), dist=0.3, fx=1.2, z_clip=0.05, max_amb=1e-2),
             'z-clipped blocks')
    assert r['fb'].unclipped_to_clipped is not None


# ------------------------------------------------------------------------------------------------ 9. zero-area faces
@pytest.mark.parametrize('Kf', [3, 10])
def test_zero_area_faces(Kf):
    r = _run(_case(seed=17, Kf=Kf, alpha='face', size=(48, 48), zero_area=True), f'zero-area K={Kf}')
    assert not ((r['ids_b'] == 100) | (r['ids_b'] == 101)).any()


# ------------------------------------------------------------------------------------------------ 10. crowded tiles
def _listed_faces_lower_bound(scene, R, T, K, size, nt, z_clip):
    """most faces some forward tile (16 x nt/16 pixels) lists, at least: faces in front of z_clip whose projected triangle
    contains a pixel centre of the tile pass both the box test and tri_overlaps_rect"""
    H, W = size
    th = nt // 16

    def pix_to_ndc(i, s1, s2):               # csrc/dbw_math.cuh (+X is left, +Y is up)
        rng = 2.0 * s1 / s2 if s1 > s2 else 2.0
        return -rng / 2 + (rng * i + rng / 2) / s1

    px = pix_to_ndc(W - 1 - torch.arange(W, dtype=torch.float64), W, H)
    py = pix_to_ndc(H - 1 - torch.arange(H, dtype=torch.float64), H, W)
    ndc = pt3d.world_to_ndc(scene['verts'].detach(), R, T, K)
    most = 0
    for b in range(R.shape[0]):
        fv = ndc[b][scene['faces']]
        tri = fv[(fv[..., 2] > z_clip).all(-1), :, :2]
        count = torch.zeros((H + th - 1) // th, (W + 15) // 16, dtype=torch.long)
        for t in tri.split(256):
            e = []
            for i in range(3):
                a, c = t[:, i], t[:, (i + 1) % 3]
                e.append((px[None, None] - a[:, 0, None, None]) * (c[:, 1] - a[:, 1])[:, None, None]
                         - (py[None, :, None] - a[:, 1, None, None]) * (c[:, 0] - a[:, 0])[:, None, None])
            e = torch.stack(e)
            inside = (e > 1e-12).all(0) | (e < -1e-12).all(0)                    # (faces, H, W)
            inside = F.pad(inside, (0, -W % 16, 0, -H % th))
            hit = inside.view(len(t), inside.shape[1] // th, th, inside.shape[2] // 16, 16).any(4).any(2)
            count += hit.sum(0)
        most = max(most, int(count.max()))
    return most


@pytest.mark.parametrize('Kf,alpha', [(10, 'face'), (3, 'batch')])
def test_crowded_tiles_take_the_chunked_path(Kf, alpha):
    """test_render_parity.test_stress_shape_many_faces's crowded 50-block scene: some tile lists more faces than the forward
    kernel's list holds (CAP = 64 at K > 4, 256 at K <= 4), with the loss epilogue and its backward.  At K > 4 ordinary scenes
    take the chunked path too (back faces are listed: the 7-block scenes above list at least 137 faces in some 16 x 8 tile);
    at K <= 4 only crowded scenes and images small enough for the whole scene to fall into one tile do"""
    c = _case(nb=50, seed=7, boxy=True, crowd=0.35, Kf=Kf, alpha=alpha, size=(96, 128), big_alpha=alpha == 'face')
    w = _world(c)
    nt, cap = _nt(Kf)
    most = _listed_faces_lower_bound(w['blk'], w['R'], w['T'], w['K'], c['size'], nt, c['z_clip'])
    print(f'\ncrowded K={Kf}: some tile lists at least {most} faces (CAP {cap})')
    assert most > cap
    _run(c, f'crowded K={Kf}')


# ------------------------------------------------------------------------------------------------ 11. upstream gradient, poses
def test_upstream_scale_and_pose_gradients():
    """loss x 0.37, and R / T requiring grad: the deferred fold multiplies by the upstream gradient and its camera_grad_kernel
    gives d/dR and d/dT"""
    _run(_case(seed=14, alpha='batch', scale=0.37, poses=True, size=(48, 64)), 'upstream 0.37 + poses')


# ------------------------------------------------------------------------------------------------ 12. the model, per-face opacities
def test_model_with_per_face_opacities():
    """DifferentiableBlocksWorld in the coarse phase with one opacity entry per face (alpha_group_faces = 1): 10 blocks, 800
    entries per view, above the 512 the kernel sums in shared memory.  Every leaf against the oracle (test_baseline_shapes_gpu's
    scheme), then against the same model with one entry per block, within the spread of the atomics"""
    from tests.test_baseline_shapes_gpu import _bench_model, _leaf_gradient_parity, _ring
    dev = _dev()
    size = (96, 128)
    tpl = D.SceneTemplate(n_blocks=10, txt_size=256)
    R, T, K = _ring([0, 24, 48])
    model = _bench_model(size)
    model.alpha_group_faces = 1
    with _spying() as spy:
        _leaf_gradient_parity(model, tpl, size, R, T, K, 10, 1e-4, False)
    fwd = [a for n, a in spy.calls if n == 'dbw_render_forward_loss_grad']
    assert len(fwd) == 1, [n for n, _ in spy.calls]
    cfg = fwd[0][0]._obj
    assert cfg.alpha_group == 1 and cfg.n_faces == 800 > ALPHA_SMEM_MAX

    g = torch.Generator().manual_seed(8)
    inp = {'imgs': torch.rand(3, 3, *size, generator=g).to(dev), 'R': R.float().to(dev), 'T': T.float().to(dev),
           'K': K.float()[None].expand(3, -1, -1).to(dev)}
    noise = torch.randn(10, generator=g).to(dev)

    def grads(group):
        m = _bench_model(size)
        m.alpha_group_faces = group
        m.opacity_noise_buffer = noise
        m(inp, None)['total'].backward()
        return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}
    per_face, per_block, per_block2 = grads(1), grads(None), grads(None)
    assert per_face.keys() == per_block.keys()
    for n in per_block:
        if per_block[n].abs().max() > 0:
            _close_to_cuda(per_face[n], per_block[n], per_block2[n], f'per-face vs per-block opacities: {n}')
