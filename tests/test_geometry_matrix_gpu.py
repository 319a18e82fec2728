"""GPU: the geometry end of the render backward against a float64 autograd oracle, element by element.

Everything in csrc/dbw_render.cu between the rasterizer's per-slot triangle gradients and the leaves:
  * the standalone projection -- dbw_camera_project / dbw_camera_project_backward (camera_project_*_kernel): each view with its
    own (fx, fy, px, py), 1 .. 33 views, 1 .. 3000 vertices around the 32-lane warp, vertices at |z| < eps, at exactly 0 and at
    +-eps (1 +- 1e-3), rotations far from the identity and large translations; outputs accumulate into random prefills, and
    each output may be NULL on its own;
  * the deferred fold -- dbw_render_backward_deferred after a dbw_render_forward_loss_grad: the forward sets up the workspace,
    then the scratch's g_tri, g_conv, cell-gradient copies and opacity partials are overwritten with chosen cotangents
    (the scratch layout is mirrored from carve_bwd) and folded: fold_gcells_kernel, scale_add_kernel, and
    face_setup_backward_kernel's z-clip branch (lerp_clip_backward, the w2 / w3 chain, the conversion rows b4 / b5, both
    slot layouts) through project_verts_backward_kernel and camera_grad_kernel.  The oracle differentiates
        L = sum_slots <g_tri, tri_slot(verts, R, T, K)> + sum_clipped slots <g_conv, conv_slot(verts, R, T, K)>
    built from oracle.pt3d.world_to_ndc and clip_faces, mapped to the kernel's (view, slot) layout as
    tests/test_device_math_host.py maps clip_face to clip_faces (slot f: clipped face u2c[f], slot F + f: u2c[f] + 1);
  * what the real forward leaves in the scratch where the fold reads without looking (slots that do not exist, static and
    killed faces, g_conv of unclipped slots), the fold of a real forward at the training's 400 x 400 shape with z-clipped
    ground quads, and dbw_render_backward's geometry end against the deferred one on the same slot gradients.

Every clip decision (z against z_clip, |z| against eps) is exact: the cameras' depth axis is a signed unit vector and the
vertices' depth coordinates lie on a 2^-16 grid, so the float32 view depth equals the float64 one and sits where the case
puts it -- clear of z_clip by many ulps, or exactly at 0, or at eps (1 +- 1e-3).

Bars are fractions of each array's largest float64 magnitude: BAR_FACTOR times the deviation of the oracle's own float32
evaluation from float64 over the same cases (tests/test_geometry_matrix_host.py measures it on the CPU), floored at 4x the
spread of two identical runs (the order of the atomics).  This module is importable without a GPU: the host module reuses
its case tables and oracle."""
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import pt3d

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAR_FACTOR = 8
BAR_CAP = 1e-5                # no bar is looser than this fraction of the largest magnitude
BARS = {
    'proj.ndc': 1e-6, 'proj.g_verts': 4.5e-6, 'proj.g_R': 5.5e-6, 'proj.g_T': 2.5e-6, 'proj.g_intr': 3.7e-6,
    'fold.g_verts': 3.7e-6, 'fold.g_R': 8.7e-6, 'fold.g_T': 2e-6, 'fold.g_maps': 1.4e-6, 'fold.g_alpha': 1.4e-6,
}
WORST = {}          # bar name -> worst error seen in this session (written out when DBW_GEOMETRY_MATRIX_REPORT names a file)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    path = os.environ.get('DBW_GEOMETRY_MATRIX_REPORT')
    if path:
        with open(path, 'w') as f:
            json.dump({k: {'worst_rel_err': v[0], 'bar': v[1]} for k, v in sorted(WORST.items())}, f, indent=1)


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


def check(name, got, want, what='', floor=0.):
    """got vs want against BARS[name] (or `floor`, 4x the spread of two identical runs, when that is larger)"""
    bar = max(BARS[name], floor)
    e = rel_err(got, want)
    w = WORST.get(name, (0., bar))
    WORST[name] = (max(w[0], e), max(w[1], bar))
    print(f'{name} {what}: {e:.3g} of max |oracle| (bar {bar:.3g})')
    assert e <= bar, f'{name} {what}: max error {e:.3g} of max |oracle| > bar {bar:.3g}'


# ---------------------------------------------------------------------------------------------------------- constants
def _source_constants():
    cu = open(os.path.join(ROOT, 'differentiable-blocksworld_b200', 'csrc', 'dbw_render.cu')).read()
    h = open(os.path.join(ROOT, 'include', 'dbw_render.h')).read()
    c = {n: int(re.search(rf'#define {n} (\d+)', cu).group(1)) for n in ('DBW_BWD_NT', 'TILE_W', 'DBW_BWD_TILES_K1', 'DBW_BWD_TILES_KN')}
    c['DBW_CELL_GRAD_COPIES'] = int(re.search(r'#define DBW_CELL_GRAD_COPIES (\d+)', h).group(1))
    return c


CONST = _source_constants()
COPIES = CONST['DBW_CELL_GRAD_COPIES']
GRAD_VERTS, GRAD_MAPS, GRAD_ALPHA = 1, 2, 4          # DBW_GRAD_* of include/dbw_render.h


def _align(x, a=256):
    return (x + a - 1) // a * a


def bwd_layout(s):
    """{region: (byte offset, bytes)} and the total of the backward scratch, region for region as carve_bwd lays it out"""
    B, V, S = s.n_views, s.n_verts, 2 * s.n_faces
    n_entries = s.n_map_floats // 3
    strip_rows = (CONST['DBW_BWD_TILES_K1'] if s.faces_per_pixel == 1 else CONST['DBW_BWD_TILES_KN']) * (CONST['DBW_BWD_NT'] // 16)
    n_flags = 0 if (s.faces_per_pixel != 1 or s.detach_bary) else \
        B * -(-s.width // CONST['TILE_W']) * -(-s.height // strip_rows)
    n_alpha = s.n_faces // (s.alpha_group if s.alpha_group > 0 else 1)
    sizes = [('g_tri', B * S * 9 * 4), ('g_conv', B * S * 9 * 4), ('g_verts_ndc', B * V * 3 * 4),
             ('g_maps4', 0 if s.maps_are_texels4 else n_entries * 16),
             ('g_cells', COPIES * n_entries * 16 if s.maps_are_texels4 == 2 else 0),
             ('bary_flags', n_flags * 4), ('g_alpha', B * n_alpha * 4)]
    out, off = {}, 0
    for name, n in sizes:
        out[name] = (off, n)
        off += _align(n)
    return out, off


def workspace_bytes(s):
    from dbw_b200 import _lib
    fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(_lib.lib().dbw_workspace_bytes(ctypes.byref(s), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
    return fwd.value, bwd.value


# ---------------------------------------------------------------------------------------------------------- oracle
def K4(intr):
    """the (4,4) K of oracle.pt3d.world_to_ndc from (fx, fy, px, py), differentiable in them"""
    z, o = intr.new_zeros(()), intr.new_ones(())
    return torch.stack([torch.stack([intr[0], z, intr[2], z]), torch.stack([z, intr[1], intr[3], z]),
                        torch.stack([z, z, z, o]), torch.stack([z, z, o, z])])


def _leaf(t, dtype):
    return t.detach().to(dtype).clone().requires_grad_(True)


def proj_oracle(x, dtype):
    """(verts_ndc, {g_verts, g_R, g_T, g_intr}) of sum <g_ndc, world_to_ndc>, each view with its own K"""
    v, R, T, intr = (_leaf(x[k], dtype) for k in ('verts', 'R', 'T', 'intr'))
    ndc = torch.cat([pt3d.world_to_ndc(v, R[b:b + 1], T[b:b + 1], K4(intr[b]), eps=x['eps']) for b in range(R.shape[0])])
    loss = (ndc * x['g_ndc'].to(dtype)).sum()
    g = torch.autograd.grad(loss, [v, R, T, intr])
    return ndc.detach(), dict(zip(('g_verts', 'g_R', 'g_T', 'g_intr'), g))


def clip_slots(fv, z_clip):
    """per face (packed over views): number of vertices behind z_clip and number of triangle slots (0, 1 or 2)"""
    nb = (fv[:, :, 2] < z_clip).sum(1) if z_clip >= 0 else torch.zeros(fv.shape[0], dtype=torch.long)
    return nb, torch.tensor([1, 2, 1, 0])[nb]


def fold_oracle(x, g_tri, g_conv, dtype):
    """{g_verts[, g_R, g_T]} (unscaled) of L = sum_slots <g_tri, tri_slot> + sum_clipped slots <g_conv, conv_slot>.
    g_tri / g_conv (B, 2F, 9): slot f is the first triangle of face f, slot F + f the second one of a split face."""
    ndc_in = x['ndc']
    B, F = x['R'].shape[0], x['faces'].shape[0]
    faces = x['faces'].long()
    if ndc_in:
        v = _leaf(x['verts'], dtype)
        leaves, ndc = [v], v
    else:
        v, R, T = (_leaf(x[k], dtype) for k in ('verts', 'R', 'T'))
        leaves = [v, R, T]
        ndc = pt3d.world_to_ndc(v, R, T, K4(torch.tensor(x['intr'], dtype=dtype)), eps=x['eps'])
    fv = ndc[:, faces].reshape(B * F, 3, 3)
    gt = g_tri.to(dtype).reshape(B, 2, F, 9).transpose(0, 1).reshape(2, B * F, 9)
    gc = g_conv.to(dtype).reshape(B, 2, F, 9).transpose(0, 1).reshape(2, B * F, 9)
    nb, ntri = clip_slots(fv.detach(), x['z_clip'])
    if int(nb.sum()) == 0:
        loss = (fv.reshape(B * F, 9) * gt[0]).sum()
    else:
        cl = pt3d.clip_faces(fv, torch.arange(B) * F, torch.full((B,), F), x['z_clip'], x['persp'])
        clipped = (nb == 1) | (nb == 2)
        loss = fv.new_zeros(())
        for k in range(2):
            sel = ntri > k
            loss = loss + (cl.face_verts[cl.u2c[sel] + k].reshape(-1, 9) * gt[k][sel]).sum()
            sel = sel & clipped
            loss = loss + (cl.conversion[cl.u2c[sel] + k].reshape(-1, 9) * gc[k][sel]).sum()
    g = torch.autograd.grad(loss, leaves)
    return dict(zip(('g_verts', 'g_R', 'g_T'), g))


def fold_maps_alpha(g_cells, g_alpha, n_alpha_out, dtype):
    """sum of the cell-gradient copies (xyz; w untouched) and the opacity partials a fold adds, unscaled"""
    cells = g_cells.to(dtype).reshape(COPIES, -1, 4)
    t = cells[0, :, :3].clone()
    for r in range(1, COPIES):
        t = t + cells[r, :, :3]
    return t, g_alpha.to(dtype).reshape(-1)[:n_alpha_out]


# ---------------------------------------------------------------------------------------------------------- inputs
GRID = 2.0 ** -16


def _on_grid(a):
    return np.round(np.asarray(a, np.float64) / GRID) * GRID


def _cyclic_rotation(theta):
    """P @ Rz(theta), P the cyclic permutation: its depth column is exactly (0, 1, 0), so z_view = Y_world + T_z"""
    c, s = math.cos(theta), math.sin(theta)
    Rz = np.array([[c, -s, 0.], [s, c, 0.], [0., 0., 1.]])
    P = np.array([[0., 1., 0.], [0., 0., 1.], [1., 0., 0.]])
    return P @ Rz


def _random_rotation(g):
    q, r = np.linalg.qr(g.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


PROJ_EPS = 0.05                 # eps of the projection cases: vertices sit at and around it
PROJ_CASES = [dict(name=f'B{B}-V{V}', B=B, V=V, seed=100 * B + V) for B in (1, 7, 33) for V in (1, 31, 32, 33, 3000)]
PROJ_BY_NAME = {c['name']: c for c in PROJ_CASES}
SPECIAL_Z = [0.0, 0.3 * PROJ_EPS, -0.3 * PROJ_EPS, PROJ_EPS * (1 + 1e-3), PROJ_EPS * (1 - 1e-3), -PROJ_EPS * (1 + 1e-3),
             -PROJ_EPS * (1 - 1e-3)]


def proj_inputs(name):
    """float32 inputs of one projection case.  Even views: random rotations, translations up to 40.  Odd views: exact-depth
    cameras (_cyclic_rotation, T_z = 0) in which the first vertices sit at z = 0, |z| < eps and +-eps (1 +- 1e-3)."""
    c = PROJ_BY_NAME[name]
    g = np.random.default_rng(c['seed'])
    B, V = c['B'], c['V']
    verts = g.uniform(-2, 2, (V, 3))
    y = verts[:, 1]
    y[np.abs(y) < 0.2] += 0.4                                      # ordinary vertices stay far from the clamp in every view
    n_sp = min(V, len(SPECIAL_Z))
    y[:n_sp] = SPECIAL_Z[:n_sp]
    R, T = np.zeros((B, 3, 3)), np.zeros((B, 3))
    for b in range(B):
        if b % 2 == 0:
            R[b] = _random_rotation(g)
            T[b] = [g.uniform(-30, 30), g.uniform(-30, 30), g.uniform(10, 40)]
        else:
            R[b] = _cyclic_rotation(g.uniform(0, 2 * math.pi))
            T[b] = [g.uniform(-30, 30), g.uniform(-30, 30), 0.]
    intr = np.stack([g.uniform(0.5, 5, B), g.uniform(0.5, 5, B), g.uniform(-0.5, 0.5, B), g.uniform(-0.5, 0.5, B)], 1)
    f32 = lambda a: torch.from_numpy(np.asarray(a, np.float32))
    x = dict(verts=f32(verts), R=f32(R), T=f32(T), intr=f32(intr), eps=PROJ_EPS)
    x['g_ndc'] = f32(g.standard_normal((B, V, 3)))
    return x


def proj_depths(x):
    """float64 view depth of every (view, vertex) of the float32 inputs"""
    v, R, T = x['verts'].double(), x['R'].double(), x['T'].double()
    return (v[None] @ R + T[:, None])[..., 2]


# Fold cases: a covering set.  z_clip < 0: clipping off.  hub: one vertex shared by that many faces.  static / killed: leading
# faces with constant vertices / faces whose face_map is -1.  small_den: the isolated vertex and one other sit 2.5e-4 (in units
# of the depth) on either side of z_clip.  eps_verts: z_clip off and vertices within proj_eps of z = 0.
FOLD_CASES = [
    dict(name='persp-B1', B=1, F=160, persp=True, z_clip=0.3, scale=1.0, seed=1),
    dict(name='affine-B33', B=33, F=37, persp=False, z_clip=0.3, scale=-0.37, seed=2, alpha='view', group=1),
    dict(name='persp-B33-group', B=33, F=40, persp=True, z_clip=0.3, scale=2.5, seed=3, alpha='view', group=4),
    dict(name='small-den-persp', B=3, F=96, persp=True, z_clip=0.5, scale=0.7, seed=4, small_den=True),
    dict(name='small-den-affine', B=2, F=96, persp=False, z_clip=0.5, scale=-1.3, seed=5, small_den=True),
    dict(name='hub500', B=2, F=520, persp=True, z_clip=0.3, scale=0.9, seed=6, hub=500),
    dict(name='static-killed', B=4, F=90, persp=True, z_clip=0.3, scale=1.7, seed=7, static=20, killed=13, group=2),
    dict(name='zclip-off-eps', B=2, F=64, persp=True, z_clip=-1.0, scale=0.45, seed=8, eps_verts=True),
    dict(name='ndc-B3', B=3, F=80, persp=True, z_clip=0.3, scale=1.1, seed=9, ndc=True),
    dict(name='ndc-affine-B5', B=5, F=70, persp=False, z_clip=0.3, scale=-0.8, seed=10, ndc=True, alpha='view'),
]
FOLD_BY_NAME = {c['name']: c for c in FOLD_CASES}
FOLD_EPS = 0.05                  # proj_eps of the eps_verts case (1e-8, the renderer's, elsewhere)
N_MAPS, MAP_H, MAP_F = 3, 8, 2   # cell maps of the fold scenes: 3 maps of (8/2)^2 cells
H_IMG = W_IMG = 40


def _face_depths(g, c, f):
    """view depths of the 3 vertices of fold face f: f % 4 of them behind z_clip (clip counts 0, 1, 2, 3 in turn)"""
    zc = c['z_clip']
    if c.get('eps_verts'):
        e = FOLD_EPS
        pool = [0.0, 0.4 * e, -0.4 * e, e * (1 + 1e-3), e * (1 - 1e-3), -e * (1 + 1e-3), -e * (1 - 1e-3)]
        z = g.uniform(0.3, 3.0, 3) * g.choice([-1., 1.], 3)
        z[f % 3] = pool[f % len(pool)]
        return z
    n_behind = f % 4
    if c.get('small_den') and n_behind in (1, 2):
        # the isolated vertex and one other 2.5e-4 z_clip on either side of the plane, the third far on the other's side
        d = zc * 2.5e-4
        if n_behind == 1:
            z = np.array([zc - d, zc + d, g.uniform(zc + 0.2, 3.0)])
        else:
            z = np.array([zc + d, zc - d, g.uniform(-1.0, zc - 0.2)])
        return g.permutation(z)
    front = g.uniform(zc + 0.01, 3.0, 3)
    behind = np.where(g.random(3) < 0.5, g.uniform(0.1, zc - 0.01, 3), g.uniform(-1.0, -0.1, 3))
    mask = np.zeros(3, bool)
    mask[g.permutation(3)[:n_behind]] = True
    return np.where(mask, behind, front)


def fold_scene(name):
    """float32 scene of one fold case (CPU): verts (V,3) world [or (B,V,3) NDC], faces, R, T, intrinsics, face map, opacities,
    cell maps.  The cameras are _cyclic_rotation's with T_z = 0.5: every view sees the same exact depths."""
    c = FOLD_BY_NAME[name]
    g = np.random.default_rng(c['seed'])
    B, F = c['B'], c['F']
    verts, faces = [], []
    hub = c.get('hub', 0)
    if hub:                                   # one vertex in front of the clip plane, shared by `hub` faces
        verts.append([g.uniform(-0.5, 0.5), 1.5, g.uniform(-0.5, 0.5)])
    tz = 0.5
    for f in range(F):
        z = _face_depths(g, c, f)
        xz = g.uniform(-0.6, 0.6, (3, 2)) * np.maximum(np.abs(z), 0.3)[:, None]
        ids = []
        for j in range(3):
            if hub and f < hub and j == 0:
                ids.append(0)
                continue
            ids.append(len(verts))
            verts.append([xz[j, 0], z[j] - tz, xz[j, 1]])
        faces.append(ids)
    verts = np.array(verts)
    verts[:, 1] = _on_grid(verts[:, 1])
    R = np.stack([_cyclic_rotation(g.uniform(0, 2 * math.pi)) for _ in range(B)])
    T = np.concatenate([g.uniform(-0.2, 0.2, (B, 2)), np.full((B, 1), tz)], 1)
    intr = (float(np.float32(g.uniform(0.8, 1.5))), float(np.float32(g.uniform(0.8, 1.5))),
            float(np.float32(g.uniform(-0.1, 0.1))), float(np.float32(g.uniform(-0.1, 0.1))))
    eps = FOLD_EPS if c.get('eps_verts') else 1e-8
    f32 = lambda a: torch.from_numpy(np.asarray(a, np.float32))
    x = dict(verts=f32(verts), faces=torch.tensor(faces, dtype=torch.int32), R=f32(R), T=f32(T), intr=intr, eps=eps,
             z_clip=c['z_clip'], persp=c['persp'], ndc=bool(c.get('ndc')), B=B, F=F)
    if x['ndc']:                              # per-view NDC input: the float64 projection, rounded once
        ndc = pt3d.world_to_ndc(x['verts'].double(), x['R'].double(), x['T'].double(), K4(torch.tensor(intr, dtype=torch.float64)), eps)
        x['verts'] = ndc.float()
    fmap = g.integers(0, N_MAPS, F)
    if c.get('killed'):
        fmap[g.permutation(np.arange(c.get('static', 0), F))[:c['killed']]] = -1
    x['face_map'] = torch.tensor(fmap, dtype=torch.int32)
    x['n_static'] = c.get('static', 0)
    x['group'] = c.get('group', 1)
    n_alpha = F // x['group']
    x['alpha_stride'] = n_alpha if c.get('alpha') == 'view' else 0
    x['faces_alpha'] = f32(g.uniform(0.3, 0.9, (B if x['alpha_stride'] else 1) * n_alpha))
    x['faces_uvs'] = f32(g.uniform(0.05, 0.95, (F, 3, 2)))
    n_cells = N_MAPS * (MAP_H // MAP_F) ** 2
    x['maps'] = f32(np.concatenate([g.uniform(0, 1, (n_cells, 3)), np.zeros((n_cells, 1))], 1))
    x['scale'] = c['scale']
    return x


def fold_depths(x):
    """float64 view depth of every (view, vertex) -- exactly the float32 one the kernels compute"""
    if x['ndc']:
        return x['verts'][..., 2].double()
    return (x['verts'].double()[None] @ x['R'].double() + x['T'].double()[:, None])[..., 2]


def slot_classes(x):
    """(B, 2F) bool masks of the slots by kind: 'exists', 'clipped' (exists and its face is clipped), 'frozen' (static or
    killed face: the forward writes nothing there)"""
    B, F = x['B'], x['F']
    z = fold_depths(x)[:, x['faces'].long()]                          # (B,F,3)
    nb = (z < x['z_clip']).sum(-1) if x['z_clip'] >= 0 else torch.zeros(B, F, dtype=torch.long)
    ntri = torch.tensor([1, 2, 1, 0])[nb]
    exists = torch.cat([ntri >= 1, ntri >= 2], 1)
    clipped = exists & torch.cat([(nb == 1) | (nb == 2)] * 2, 1)
    frozen_f = (x['face_map'] < 0).clone()
    frozen_f[:x['n_static']] = True
    frozen = torch.cat([frozen_f, frozen_f])[None].expand(B, -1)
    return dict(exists=exists, clipped=clipped, frozen=frozen, nb=nb)


def injected(name):
    """the cotangents injected into the scratch of one fold case: g_tri / g_conv (B,2F,9), g_cells (COPIES*cells,4),
    g_alpha (B*n_alpha).  Slots of static and killed faces hold 0 (the forward writes nothing there); slots that do not exist
    and g_conv of unclipped slots hold 1e3-sized garbage the fold must not read."""
    x = fold_scene(name)
    g = torch.Generator().manual_seed(1000 + FOLD_BY_NAME[name]['seed'])
    B, F = x['B'], x['F']
    k = slot_classes(x)
    live = k['exists'] & ~k['frozen']
    garbage = lambda: 1e3 * torch.randn(B, 2 * F, 9, generator=g)
    g_tri = torch.where(live[..., None], torch.randn(B, 2 * F, 9, generator=g), garbage())
    g_tri = torch.where(k['frozen'][..., None], torch.zeros(()), g_tri)
    g_conv = torch.where((k['clipped'] & ~k['frozen'])[..., None], torch.randn(B, 2 * F, 9, generator=g), garbage())
    g_conv = torch.where(k['frozen'][..., None], torch.zeros(()), g_conv)
    n_cells = x['maps'].shape[0]
    g_cells = torch.randn(COPIES * n_cells, 4, generator=g)
    g_alpha = torch.randn(B * (F // x['group']), generator=g)
    return x, dict(g_tri=g_tri.float(), g_conv=g_conv.float(), g_cells=g_cells.float(), g_alpha=g_alpha.float())


def n_alpha_out(x):
    n_alpha = x['F'] // x['group']
    return x['B'] * n_alpha if x['alpha_stride'] else n_alpha


def fold_expected(x, inj, dtype):
    """{output: unscaled gradient} of one fold case: g_verts [, g_R, g_T], g_maps (cells, xyz), g_faces_alpha"""
    out = fold_oracle(x, inj['g_tri'], inj['g_conv'], dtype)
    out['g_maps'], out['g_faces_alpha'] = fold_maps_alpha(inj['g_cells'], inj['g_alpha'], n_alpha_out(x), dtype)
    return out


# ---------------------------------------------------------------------------------------------------------- device side
def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _map_table(dev):
    from dbw_b200._lib import DbwMapDesc
    cells = (MAP_H // MAP_F) ** 2
    table = (DbwMapDesc * N_MAPS)(*[DbwMapDesc(3 * m * cells, MAP_H, MAP_H, MAP_F) for m in range(N_MAPS)])
    return torch.frombuffer(bytearray(bytes(table)), dtype=torch.int32).to(dev)


def settings_of(x, K=2, save_fragment_state=0, n_static=None, H=H_IMG, W=W_IMG):
    from dbw_b200.renderer import make_settings
    sigma = 1e-4
    V = x['verts'].shape[-2]
    return make_settings(x['B'], H, W, K, V, x['F'], N_MAPS, x['alpha_stride'], x['intr'], sigma,
                         math.log(1. / 1e-4 - 1.) * sigma, x['z_clip'], (0., 0., 0.), perspective_correct=x['persp'],
                         detach_bary=True, verts_are_ndc=x['ndc'], eps=x['eps'], n_map_floats=3 * x['maps'].shape[0],
                         maps_are_texels4=2, save_fragment_state=save_fragment_state, alpha_group=x['group'],
                         n_static_faces=x['n_static'] if n_static is None else n_static)


def _to_dev(x, dev):
    d = {k: (v.to(dev).contiguous() if torch.is_tensor(v) else v) for k, v in x.items()}
    d['table'] = _map_table(dev)
    return d


def forward_loss_grad(d, s, mask, dev):
    """runs dbw_render_forward_loss_grad; returns (workspace, scratch)"""
    from dbw_b200 import _lib
    from dbw_b200._lib import DbwLossEpilogue
    B, H, W = s.n_views, s.height, s.width
    fwd, bwd = workspace_bytes(s)
    ws = torch.empty(fwd, dtype=torch.uint8, device=dev)
    scratch = torch.full((bwd,), 0x7f, dtype=torch.uint8, device=dev)         # the call zero-fills it
    g = torch.Generator(device='cpu').manual_seed(B * 7 + H)
    env = torch.rand(B, 4, H, W, generator=g).to(dev)
    target = torch.rand(B, 3, H, W, generator=g).to(dev)
    g_env = torch.empty(B, 4, H, W, device=dev)
    partials = torch.empty(1024, device=dev)
    ep = DbwLossEpilogue()
    ep.env_rgba, ep.target, ep.g_env = env.data_ptr(), target.data_ptr(), g_env.data_ptr()
    ep.rec, ep.loss_partials, ep.n_partials, ep.inv_count, ep.env_alpha_unread = None, partials.data_ptr(), 1024, 1. / (B * 3 * H * W), 0
    _lib.check(_lib.lib().dbw_render_forward_loss_grad(
        ctypes.byref(s), _p(d['verts']), _p(d['faces']), _p(d['faces_uvs']), _p(d['face_map']), _p(d['maps']), _p(d['table']),
        None if d['ndc'] else _p(d['R']), None if d['ndc'] else _p(d['T']), _p(d['faces_alpha']), _p(ws), ws.numel(),
        ctypes.byref(ep), mask, _p(scratch), scratch.numel(), None), 'dbw_render_forward_loss_grad')
    torch.cuda.synchronize()
    return ws, scratch


def region(scratch, s, name):
    off, n = bwd_layout(s)[0][name]
    return scratch[off:off + n].view(torch.float32)


OUTPUTS = ('g_verts', 'g_faces_alpha', 'g_maps', 'g_R', 'g_T')


def prefilled_outputs(x, dev, seed, ref=None):
    """random prefills of the five outputs, of each one's expected magnitude (`ref`) when given"""
    g = torch.Generator().manual_seed(seed)
    shapes = {'g_verts': tuple(x['verts'].shape), 'g_faces_alpha': (x['faces_alpha'].numel(),), 'g_maps': tuple(x['maps'].shape),
              'g_R': tuple(x['R'].shape), 'g_T': tuple(x['T'].shape)}
    out = {}
    for k, shp in shapes.items():
        mag = 1.0 if ref is None or ref.get(k) is None else max(ref[k].abs().max().item(), 1e-30) * 0.5
        out[k] = (torch.randn(shp, generator=g) * mag).float().to(dev)
    return out


def deferred(d, s, ws, scratch, outs, scale, skip=(), dev=None):
    """dbw_render_backward_deferred into copies of `outs` (those named in `skip` passed as NULL); returns the copies"""
    from dbw_b200 import _lib
    o = {k: (None if (k in skip or (d['ndc'] and k in ('g_R', 'g_T'))) else v.clone()) for k, v in outs.items()}
    sc = torch.tensor([scale], dtype=torch.float32, device=scratch.device)
    _lib.check(_lib.lib().dbw_render_backward_deferred(
        ctypes.byref(s), _p(d['verts']), _p(d['faces']), None if d['ndc'] else _p(d['R']), None if d['ndc'] else _p(d['T']),
        _p(ws), ws.numel(), _p(sc), _p(o['g_verts']), _p(o['g_faces_alpha']), _p(o['g_maps']), _p(o['g_R']), _p(o['g_T']),
        _p(scratch), scratch.numel(), None), 'dbw_render_backward_deferred')
    torch.cuda.synchronize()
    return o


def inject(scratch, s, inj, regions=('g_tri', 'g_conv', 'g_cells', 'g_alpha')):
    """overwrites the named scratch regions with the injected cotangents (the rest of the chosen ones with 0)"""
    for name in ('g_tri', 'g_conv', 'g_cells', 'g_alpha'):
        r = region(scratch, s, name)
        r.copy_(inj[name].reshape(-1).to(r.device) if name in regions else torch.zeros_like(r))


def expected_outputs(x, pre, ref, scale):
    """prefill + scale * oracle gradient, float64, per output (g_maps: xyz of each cell, w kept)"""
    out = {}
    for k, p in pre.items():
        p = p.double().cpu()
        if k == 'g_maps':
            e = p.clone()
            e[:, :3] += scale * ref['g_maps'].double()
        elif k in ref:
            e = p + scale * ref[k].double()
        else:
            continue
        out[k] = e
    return out


def accumulated_f32(pre, scale, g32):
    """what a float32 `pre += scale * g` adds, read back as the tests read the kernels' outputs (got - pre, in float64)"""
    return (pre + torch.tensor(scale, dtype=torch.float32) * g32).double() - pre.double()


def _spread(a, b):
    return {k: rel_err(a[k], b[k]) for k in a if a[k] is not None}


def run_fold_case(name, dev):
    """(case inputs, device inputs, settings, workspace, scratch with the injection, prefills, oracle) of one fold case"""
    x, inj = injected(name)
    d = _to_dev(x, dev)
    s = settings_of(x)
    ws, scratch = forward_loss_grad(d, s, GRAD_VERTS | GRAD_MAPS | GRAD_ALPHA, dev)
    inject(scratch, s, inj)
    ref = fold_expected(x, inj, torch.float64)
    pre = prefilled_outputs(x, dev, seed=FOLD_BY_NAME[name]['seed'], ref=ref)
    return x, inj, d, s, ws, scratch, pre, ref


# ---------------------------------------------------------------------------------------------------------- projection
def projection_prefills(g64):
    """random float32 prefills of the projection gradients, half their oracle's largest magnitude"""
    gen = torch.Generator().manual_seed(7)
    return {k: (torch.randn(g64[k].shape, generator=gen, dtype=torch.float64) * 0.5 * g64[k].abs().max().item()).float()
            for k in ('g_verts', 'g_R', 'g_T', 'g_intr')}


def _project(x, dev, outs, skip=()):
    from dbw_b200 import _lib
    L = _lib.lib()
    v, R, T, intr, g_ndc = (x[k].to(dev).contiguous() for k in ('verts', 'R', 'T', 'intr', 'g_ndc'))
    B, V = R.shape[0], v.shape[0]
    ndc = torch.full((B, V, 3), float('nan'), device=dev)
    _lib.check(L.dbw_camera_project(B, V, _p(v), _p(R), _p(T), _p(intr), ctypes.c_float(x['eps']), _p(ndc), None), 'dbw_camera_project')
    o = {k: (None if k in skip else t.clone()) for k, t in outs.items()}
    _lib.check(L.dbw_camera_project_backward(B, V, _p(v), _p(R), _p(T), _p(intr), ctypes.c_float(x['eps']), _p(g_ndc),
                                             _p(o['g_verts']), _p(o['g_R']), _p(o['g_T']), _p(o['g_intr']), None),
               'dbw_camera_project_backward')
    torch.cuda.synchronize()
    return ndc, o


@pytest.mark.parametrize('name', [c['name'] for c in PROJ_CASES])
def test_projection_and_its_backward_accumulate_the_oracle(name):
    """verts_ndc, and g_verts / g_R / g_T / g_intrinsics added onto random prefills, against float64 autograd of world_to_ndc"""
    dev = _dev()
    x = proj_inputs(name)
    ndc64, g64 = proj_oracle(x, torch.float64)
    pre = {k: v.to(dev) for k, v in projection_prefills(g64).items()}
    ndc, o = _project(x, dev, pre)
    check('proj.ndc', ndc, ndc64, name)
    for k in ('g_verts', 'g_R', 'g_T', 'g_intr'):
        check(f'proj.{k}', o[k].double().cpu() - pre[k].double().cpu(), g64[k], name)     # what the call added


@pytest.mark.parametrize('name', ['B7-V33', 'B33-V3000'])
def test_projection_backward_null_outputs_leave_the_others_bit_identical(name):
    dev = _dev()
    x = proj_inputs(name)
    gen = torch.Generator().manual_seed(11)
    pre = {'g_verts': torch.randn(x['verts'].shape, generator=gen), 'g_R': torch.randn(x['R'].shape, generator=gen),
           'g_T': torch.randn(x['T'].shape, generator=gen), 'g_intr': torch.randn(x['intr'].shape, generator=gen)}
    pre = {k: v.to(dev) for k, v in pre.items()}
    _, full = _project(x, dev, pre)
    for k in pre:
        _, o = _project(x, dev, pre, skip=(k,))
        for j in pre:
            if j != k:
                assert torch.equal(o[j], full[j]), f'{j} changed when {k} was NULL'


# ---------------------------------------------------------------------------------------------------------- deferred fold
@pytest.mark.parametrize('name', [c['name'] for c in FOLD_CASES])
def test_deferred_fold_of_injected_cotangents_matches_the_oracle(name):
    """every output of dbw_render_backward_deferred, added onto random prefills, against scale * the float64 oracle; the
    garbage in slots that do not exist and in unclipped slots' g_conv is never read"""
    dev = _dev()
    x, inj, d, s, ws, scratch, pre, ref = run_fold_case(name, dev)
    k = slot_classes(x)
    if x['z_clip'] >= 0:
        counts = set(k['nb'].reshape(-1).tolist())
        assert counts == {0, 1, 2, 3} or FOLD_BY_NAME[name].get('small_den'), counts
    keep = scratch.clone()
    o1 = deferred(d, s, ws, scratch, pre, x['scale'])
    scratch.copy_(keep)
    o2 = deferred(d, s, ws, scratch, pre, x['scale'])
    spread = _spread(o1, o2)
    want = expected_outputs(x, pre, ref, x['scale'])
    for out, w in want.items():
        if o1.get(out) is None:
            continue
        bar = 'fold.g_alpha' if out == 'g_faces_alpha' else f'fold.{out}'
        got = o1[out].double().cpu()
        if out == 'g_maps':
            assert torch.equal(o1[out][:, 3], pre[out][:, 3]), 'the fold wrote a cell w'
            got, w, p = got[:, :3], w[:, :3], pre[out].double().cpu()[:, :3]
        else:
            p = pre[out].double().cpu()
        check(bar, got - p, w - p, name, floor=4 * spread[out])


@pytest.mark.parametrize('name', ['persp-B1', 'static-killed', 'ndc-B3'])
def test_each_output_null_on_its_own_leaves_the_others_bit_identical(name):
    dev = _dev()
    x, inj, d, s, ws, scratch, pre, ref = run_fold_case(name, dev)
    keep = scratch.clone()
    full = deferred(d, s, ws, scratch, pre, x['scale'])
    for skip in OUTPUTS:
        if x['ndc'] and skip in ('g_R', 'g_T'):
            continue
        scratch.copy_(keep)
        o = deferred(d, s, ws, scratch, pre, x['scale'], skip=(skip,))
        for j in OUTPUTS:
            if j != skip and full[j] is not None:
                assert torch.equal(o[j], full[j]), f'{j} changed when {skip} was NULL'


@pytest.mark.parametrize('name', ['persp-B1', 'persp-B33-group'])
def test_each_scratch_region_moves_only_its_own_output(name):
    """a cotangent in one region at a time: cell-gradient copy r -> g_maps (scale * copy r), g_alpha -> g_faces_alpha,
    g_tri / g_conv -> g_verts, g_R, g_T; every other output keeps its prefill bits"""
    dev = _dev()
    x, inj, d, s, ws, scratch, pre, _ = run_fold_case(name, dev)
    n_cells = x['maps'].shape[0]
    owners = {'g_alpha': ('g_faces_alpha',), 'geometry': ('g_verts', 'g_R', 'g_T')}
    for r in range(COPIES):
        one = dict(inj, g_cells=torch.zeros_like(inj['g_cells']))
        one['g_cells'].view(COPIES, n_cells, 4)[r] = inj['g_cells'].view(COPIES, n_cells, 4)[r]
        inject(scratch, s, one, regions=('g_cells',))
        region(scratch, s, 'g_verts_ndc').zero_()
        o = deferred(d, s, ws, scratch, pre, x['scale'])
        for j in OUTPUTS:
            if j != 'g_maps':
                assert torch.equal(o[j], pre[j]), (r, j)
        want = pre['g_maps'].double().cpu()[:, :3] + x['scale'] * inj['g_cells'].view(COPIES, n_cells, 4)[r, :, :3].double()
        check('fold.g_maps', o['g_maps'].double().cpu()[:, :3], want, f'{name} copy {r}')
    for reg, moved in (('g_alpha', owners['g_alpha']), ('geometry', owners['geometry'])):
        inject(scratch, s, inj, regions=('g_tri', 'g_conv') if reg == 'geometry' else (reg,))
        region(scratch, s, 'g_verts_ndc').zero_()
        o = deferred(d, s, ws, scratch, pre, x['scale'])
        for j in OUTPUTS:
            if j in moved:
                assert not torch.equal(o[j], pre[j]), (reg, j)
            else:
                assert torch.equal(o[j], pre[j]), (reg, j)


def test_forward_scratch_is_zero_where_the_fold_reads_without_looking():
    """the real forward's scratch: g_tri / g_conv exactly 0 in slots that do not exist (three vertices behind, the second
    slot of a face that was not split), in static and killed faces' slots, and g_conv of unclipped slots (a detach_bary pass
    writes no g_conv at all); g_tri elsewhere, clipped slots included.  And garbage in g_conv of unclipped slots leaves every output as the forward's own scratch gives it."""
    dev = _dev()
    x, _ = injected('static-killed')
    d = _to_dev(x, dev)
    s = settings_of(x)
    ws, scratch = forward_loss_grad(d, s, GRAD_VERTS | GRAD_MAPS | GRAD_ALPHA, dev)
    B, F = x['B'], x['F']
    k = slot_classes(x)
    g_tri = region(scratch, s, 'g_tri').view(B, 2 * F, 9).cpu()
    g_conv = region(scratch, s, 'g_conv').view(B, 2 * F, 9).cpu()
    assert int(k['nb'].eq(3).sum()) > 0 and int(k['frozen'].sum()) > 0
    dead = ~k['exists'] | k['frozen']
    assert (g_tri[dead] == 0).all(), 'g_tri written in a slot the fold must not see'
    assert (g_conv[dead | ~k['clipped']] == 0).all(), 'g_conv written in an unclipped or dead slot'
    live = k['exists'] & ~k['frozen']
    assert (g_tri[live] != 0).any(dim=-1).sum() > 0.25 * live.sum(), 'too few slots received a gradient: nothing was tested'
    assert (g_tri[k['clipped'] & ~k['frozen']] != 0).any(), 'no clipped slot received a gradient'
    # the fold of the forward's own scratch vs the same with garbage in g_conv of unclipped slots
    pre = prefilled_outputs(x, dev, seed=5)
    keep = scratch.clone()
    ref_o = deferred(d, s, ws, scratch, pre, 0.75)
    scratch.copy_(keep)
    gc = region(scratch, s, 'g_conv').view(B, 2 * F, 9)
    garbage = torch.randn(B, 2 * F, 9, generator=torch.Generator().manual_seed(3)).to(dev) * 1e3
    unclipped = (~k['clipped']).to(dev)
    gc.copy_(torch.where(unclipped[..., None], garbage, gc))
    o = deferred(d, s, ws, scratch, pre, 0.75)
    scratch.copy_(keep)
    o2 = deferred(d, s, ws, scratch, pre, 0.75)
    spread = _spread(ref_o, o2)
    for j in OUTPUTS:
        assert rel_err(o[j] - pre[j], ref_o[j] - pre[j]) <= 4 * spread[j], j


@pytest.mark.parametrize('mask', [GRAD_MAPS | GRAD_ALPHA, GRAD_VERTS | GRAD_ALPHA, GRAD_VERTS | GRAD_MAPS, GRAD_VERTS])
def test_gradients_outside_grad_mask_come_out_unchanged(mask):
    """a real forward without some grad_mask bits, then a deferred fold asking for everything: the outputs of the missing
    bits keep their prefill bits, the others move"""
    dev = _dev()
    x, _ = injected('persp-B33-group')
    d = _to_dev(x, dev)
    s = settings_of(x)
    ws, scratch = forward_loss_grad(d, s, mask, dev)
    pre = prefilled_outputs(x, dev, seed=9)
    o = deferred(d, s, ws, scratch, pre, 1.3)
    of = {'g_verts': GRAD_VERTS, 'g_R': GRAD_VERTS, 'g_T': GRAD_VERTS, 'g_maps': GRAD_MAPS, 'g_faces_alpha': GRAD_ALPHA}
    for j, bit in of.items():
        assert torch.equal(o[j], pre[j]) == (not mask & bit), (j, mask)


def _model_scene():
    """the bench's environment + blocks scene (10 blocks, background sphere, ground quads) as one pass, 4 of the 49 ring
    cameras, float32, with cell maps"""
    from oracle import dbw_path as D
    tpl = D.SceneTemplate(n_blocks=10, txt_size=16)
    p = D.init_params(10, 16, seed=227391)
    env = tpl.build_env(p)
    blocks, _ = tpl.build_blocks(p)
    Ve = env['verts'].shape[0]
    verts = torch.cat([env['verts'], blocks['verts']]).detach().float()
    faces = torch.cat([env['faces'], blocks['faces'] + Ve]).int()
    R, T, Km = D.ring_cameras(49)
    views = [0, 12, 24, 36]
    F = faces.shape[0]
    g = np.random.default_rng(0)
    n_cells = N_MAPS * (MAP_H // MAP_F) ** 2
    x = dict(verts=verts, faces=faces, R=R[views].contiguous(), T=T[views].contiguous(),
             intr=(float(Km[0, 0]), float(Km[1, 1]), float(Km[0, 2]), float(Km[1, 2])), eps=1e-8, z_clip=0.001, persp=True,
             ndc=False, B=len(views), F=F, face_map=torch.tensor(g.integers(0, N_MAPS, F), dtype=torch.int32), n_static=0,
             group=1, alpha_stride=0, faces_alpha=torch.from_numpy(g.uniform(0.3, 0.9, F).astype(np.float32)),
             faces_uvs=torch.from_numpy(g.uniform(0.05, 0.95, (F, 3, 2)).astype(np.float32)),
             maps=torch.from_numpy(np.concatenate([g.uniform(0, 1, (n_cells, 3)), np.zeros((n_cells, 1))], 1).astype(np.float32)))
    return x


def test_fold_of_a_real_forward_at_the_training_shape():
    """400 x 400, K = 10, the ring cameras, z-clipped ground quads: the real forward's scratch, read back through the mirror,
    folded by the library and by the oracle.  The bar is calibrated here, on the scratch the forward wrote: BAR_FACTOR x the
    float32 oracle's deviation, at most BAR_CAP (which must leave 4x that deviation), floored at 4x the spread of two runs"""
    dev = _dev()
    x = _model_scene()
    d = _to_dev(x, dev)
    s = settings_of(x, K=10, H=400, W=400)
    ws, scratch = forward_loss_grad(d, s, GRAD_VERTS | GRAD_MAPS | GRAD_ALPHA, dev)
    B, F = x['B'], x['F']
    k = slot_classes(x)
    assert int(((k['nb'] == 1) | (k['nb'] == 2)).sum()) > 0, 'no z-clipped face at these cameras'
    g_tri = region(scratch, s, 'g_tri').view(B, 2 * F, 9).cpu().clone()
    g_conv = region(scratch, s, 'g_conv').view(B, 2 * F, 9).cpu().clone()
    assert (g_tri[k['clipped']] != 0).any(), 'no clipped slot received a gradient'
    g_cells = region(scratch, s, 'g_cells').view(-1, 4).cpu().clone()
    g_alpha = region(scratch, s, 'g_alpha').cpu().clone()
    inj = dict(g_tri=g_tri, g_conv=g_conv, g_cells=g_cells, g_alpha=g_alpha)
    ref64 = fold_expected(x, inj, torch.float64)
    ref32 = fold_expected(x, inj, torch.float32)
    pre = prefilled_outputs(x, dev, seed=13, ref=ref64)
    keep = scratch.clone()
    o1 = deferred(d, s, ws, scratch, pre, 0.8125)
    scratch.copy_(keep)
    o2 = deferred(d, s, ws, scratch, pre, 0.8125)
    spread = _spread(o1, o2)
    pre32 = {k: v.cpu() for k, v in pre.items()}
    pre32['g_maps'] = pre32['g_maps'][:, :3]
    for out in ('g_verts', 'g_R', 'g_T', 'g_maps', 'g_faces_alpha'):
        dev32 = rel_err(accumulated_f32(pre32[out], 0.8125, ref32[out]), 0.8125 * ref64[out])
        bar = max(min(BAR_FACTOR * dev32, BAR_CAP), 4 * spread[out], 1e-7)
        assert 4 * dev32 <= bar <= BAR_CAP, (out, dev32, spread[out])
        got, p = o1[out].double().cpu(), pre[out].double().cpu()
        if out == 'g_maps':
            got, p = got[:, :3], p[:, :3]
        e = rel_err(got - p, 0.8125 * ref64[out])
        print(f'chain.{out}: {e:.3g} of max |oracle| (bar {bar:.3g})')
        assert e <= bar, (out, e, bar)


def test_render_backward_geometry_equals_the_deferred_fold_of_its_slot_gradients():
    """dbw_render_backward's g_verts / g_R / g_T against dbw_render_backward_deferred (scale 1) on the g_tri / g_conv that the
    render backward left in its scratch: the same geometry_backward, up to the order of the atomics"""
    from dbw_b200 import _lib
    dev = _dev()
    x, _ = injected('hub500')
    d = _to_dev(x, dev)
    s = settings_of(x, save_fragment_state=1)
    fwd, bwd = workspace_bytes(s)
    ws = torch.empty(fwd, dtype=torch.uint8, device=dev)
    B, H, W = s.n_views, s.height, s.width
    out = torch.empty(B, 4, H, W, device=dev)
    L = _lib.lib()
    _lib.check(L.dbw_render_forward(ctypes.byref(s), _p(d['verts']), _p(d['faces']), _p(d['faces_uvs']), _p(d['face_map']),
                                    _p(d['maps']), _p(d['table']), _p(d['R']), _p(d['T']), _p(d['faces_alpha']), _p(out), None,
                                    _p(ws), ws.numel(), None, None, None), 'dbw_render_forward')
    grad = torch.randn(B, 4, H, W, generator=torch.Generator().manual_seed(2)).to(dev)
    pre = prefilled_outputs(x, dev, seed=4)
    o = {k: pre[k].clone() for k in ('g_verts', 'g_R', 'g_T')}
    scratch = torch.empty(bwd, dtype=torch.uint8, device=dev)
    _lib.check(L.dbw_render_backward(ctypes.byref(s), _p(d['verts']), _p(d['faces']), _p(d['faces_uvs']), _p(d['face_map']),
                                     _p(d['maps']), _p(d['table']), _p(d['R']), _p(d['T']), _p(d['faces_alpha']), _p(ws), ws.numel(),
                                     _p(grad), None, _p(o['g_verts']), None, None, _p(o['g_R']), _p(o['g_T']), _p(scratch),
                                     scratch.numel(), None), 'dbw_render_backward')
    torch.cuda.synchronize()
    assert (region(scratch, s, 'g_tri') != 0).any()
    s0 = settings_of(x)                                       # the deferred fold's settings: no fragment records
    region(scratch, s0, 'g_verts_ndc').zero_()
    runs = []
    for _ in range(2):
        sc = scratch.clone()
        runs.append(deferred(d, s0, ws, sc, {k: pre[k] for k in OUTPUTS}, 1.0, skip=('g_maps', 'g_faces_alpha')))
    for k in ('g_verts', 'g_R', 'g_T'):
        spread = rel_err(runs[0][k] - pre[k], runs[1][k] - pre[k])
        e = rel_err(o[k] - pre[k], runs[0][k] - pre[k])
        print(f'render_backward vs deferred {k}: {e:.3g} (atomics spread {spread:.3g})')
        assert e <= max(4 * spread, 1e-6), (k, e, spread)
