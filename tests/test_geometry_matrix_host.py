"""CPU: the bars, inputs and layout of tests/test_geometry_matrix_gpu.py.

For every case of the GPU module the oracle runs once in float32 and once in float64 on the same float32 inputs and
cotangents; the float32 run's worst error (fraction of each array's largest float64 magnitude, as the GPU module measures the
kernels) is what float32 arithmetic costs there.  Each bar stays a fixed headroom above it and below BAR_CAP.  The scratch
mirror equals the library's own backward scratch size over a spread of settings, the oracle's (view, slot) mapping of
clip_faces is checked against clip_face compiled for the host, and every case's clip decisions are exact."""
import ctypes

import numpy as np
import pytest
import torch

from tests import test_geometry_matrix_gpu as M
from tests.test_device_math_host import hm  # noqa: F401  (the host-compiled dbw_math.cuh / dbw_clip.cuh)

# a bar is at least HEADROOM x the float32 oracle's deviation, and at most BAR_FACTOR * 4 x it (CPUs differ in their float32
# rounding by a factor of two or so) unless it is below 2e-6
HEADROOM = 4


def _acc(out, name, e):
    out[name] = max(out.get(name, 0.), e)


_DEV = {}


def float32_deviations():
    """{bar: worst float32-oracle deviation}: the float32 evaluation of each case, including the final float32 add onto the
    GPU module's own prefills"""
    if _DEV:
        return _DEV
    for c in M.PROJ_CASES:
        x = M.proj_inputs(c['name'])
        n64, g64 = M.proj_oracle(x, torch.float64)
        n32, g32 = M.proj_oracle(x, torch.float32)
        pre = M.projection_prefills(g64)
        _acc(_DEV, 'proj.ndc', M.rel_err(n32, n64))
        for k in g64:
            _acc(_DEV, f'proj.{k}', M.rel_err(M.accumulated_f32(pre[k], 1.0, g32[k]), g64[k]))
    for c in M.FOLD_CASES:
        x, inj = M.injected(c['name'])
        r64, r32 = M.fold_expected(x, inj, torch.float64), M.fold_expected(x, inj, torch.float32)
        pre = M.prefilled_outputs(x, 'cpu', seed=c['seed'], ref=r64)
        pre['g_maps'] = pre['g_maps'][:, :3]
        for k in r64:
            _acc(_DEV, 'fold.g_alpha' if k == 'g_faces_alpha' else f'fold.{k}',
                 M.rel_err(M.accumulated_f32(pre[k], x['scale'], r32[k]), x['scale'] * r64[k]))
    return _DEV


def test_every_bar_is_measured():
    assert set(float32_deviations()) == set(M.BARS)


@pytest.mark.parametrize('name', sorted(M.BARS))
def test_bar_sits_a_fixed_multiple_above_float32_rounding(name):
    dev, bar = float32_deviations()[name], M.BARS[name]
    print(f'{name}: float32 oracle deviates by {dev:.3g} of max; bar {bar:.3g}')
    assert HEADROOM * dev <= bar, f'{name}: float32 oracle deviates by {dev:.3g} of max; bar {bar:.3g} leaves less than {HEADROOM}x'
    assert bar <= 2e-6 or bar <= 4 * M.BAR_FACTOR * dev, f'{name}: bar {bar:.3g} is loose for a float32 deviation of {dev:.3g}'
    assert bar <= M.BAR_CAP


# ---------------------------------------------------------------------------------------------------------- scratch mirror
def _settings(B=3, F=40, V=50, K=10, H=40, W=56, n_cells=48, group=1, detach=True, texels4=2):
    from dbw_b200.renderer import make_settings
    return make_settings(B, H, W, K, V, F, 3, 0, (1., 1., 0., 0.), 1e-4, 1e-3, 0.001, (0., 0., 0.), detach_bary=detach,
                         n_map_floats=3 * n_cells, maps_are_texels4=texels4, alpha_group=group)


MIRROR_SETTINGS = [
    dict(), dict(B=1, F=1, V=3), dict(B=33, F=37, V=111), dict(F=800, V=4000, n_cells=10 * 32 * 32), dict(n_cells=1),
    dict(n_cells=7, group=4), dict(F=80, group=80), dict(K=1, detach=True), dict(K=1, detach=False),
    dict(K=1, detach=False, H=400, W=400, B=49), dict(K=1, detach=False, H=129, W=17), dict(texels4=0), dict(texels4=1),
    dict(B=7, F=1248, V=700, K=25, H=800, W=800, n_cells=5000, group=4),
]


@pytest.mark.parametrize('kw', MIRROR_SETTINGS, ids=[str(i) for i in range(len(MIRROR_SETTINGS))])
def test_scratch_mirror_matches_the_library(kw):
    """the mirror of carve_bwd (region order, 256-byte alignment, DBW_CELL_GRAD_COPIES, g_alpha of B x n_alpha) totals the
    bwd size dbw_workspace_bytes reports"""
    s = _settings(**kw)
    layout, total = M.bwd_layout(s)
    assert total == M.workspace_bytes(s)[1]
    assert list(layout) == ['g_tri', 'g_conv', 'g_verts_ndc', 'g_maps4', 'g_cells', 'bary_flags', 'g_alpha']
    assert all(off % 256 == 0 for off, _ in layout.values())


def test_every_region_changes_the_library_size_as_mirrored():
    """each region's size moves the library's total: the mirror does not match by accident of padding"""
    base = _settings(n_cells=4096, F=512, V=600, B=4)
    for kw in (dict(n_cells=4096 + 64), dict(F=512 + 64), dict(V=600 + 64), dict(B=5), dict(group=4)):
        s = _settings(**dict(dict(n_cells=4096, F=512, V=600, B=4), **kw))
        assert M.bwd_layout(s)[1] == M.workspace_bytes(s)[1] != M.workspace_bytes(base)[1], kw


# ---------------------------------------------------------------------------------------------------------- oracle mapping
@pytest.mark.parametrize('name', [c['name'] for c in M.FOLD_CASES if c['z_clip'] >= 0])
def test_oracle_slot_mapping_equals_clip_face(hm, name):  # noqa: F811
    """the fold oracle's loss equals sum over (view, face, triangle k) of <g_tri[b, k F + f], tri_k> + <g_conv, conv_k> with
    clip_face (dbw_clip.cuh, what face_setup_kernel runs) compiled for the host: slot f -> clipped face u2c[f], slot F + f ->
    u2c[f] + 1, vertex orders (p4, p5, p1) and (p4, p2, p5), (p5, p2, p3)"""
    x, inj = M.injected(name)
    B, F = x['B'], x['F']
    K = M.K4(torch.tensor(x['intr'], dtype=torch.float64))
    v = x['verts'].double()
    ndc = v if x['ndc'] else M.pt3d.world_to_ndc(v, x['R'].double(), x['T'].double(), K, x['eps'])
    fv = np.ascontiguousarray(ndc[:, x['faces'].long()].reshape(B * F, 3, 3).numpy().astype(np.float32))
    n = B * F
    ntri = np.zeros(n, np.int32)
    tri, conv = np.zeros((n, 2, 3, 3), np.float32), np.zeros((n, 2, 3, 3), np.float32)
    hm.hm_clip(fv.ctypes.data_as(ctypes.c_void_p), n, ctypes.c_float(x['z_clip']), int(x['persp']),
               ntri.ctypes.data_as(ctypes.c_void_p), tri.ctypes.data_as(ctypes.c_void_p), conv.ctypes.data_as(ctypes.c_void_p))
    k = M.slot_classes(x)
    assert (ntri.reshape(B, F) == torch.tensor([1, 2, 1, 0])[k['nb']].numpy()).all()
    gt = inj['g_tri'].double().reshape(B, 2, F, 9).transpose(0, 1).reshape(2, n, 9).numpy()
    gc = inj['g_conv'].double().reshape(B, 2, F, 9).transpose(0, 1).reshape(2, n, 9).numpy()
    clipped = ((k['nb'] == 1) | (k['nb'] == 2)).reshape(-1).numpy()
    want = size = 0.
    for kk in range(2):
        sel = ntri > kk
        want += (tri[sel, kk].reshape(-1, 9) * gt[kk][sel]).sum()
        size += np.abs(tri[sel, kk].reshape(-1, 9) * gt[kk][sel]).sum()
        sel = sel & clipped
        want += (conv[sel, kk].reshape(-1, 9) * gc[kk][sel]).sum()
        size += np.abs(conv[sel, kk].reshape(-1, 9) * gc[kk][sel]).sum()
    # the oracle's loss, rebuilt the way fold_oracle builds it
    t = torch.from_numpy(fv).double()
    cl = M.pt3d.clip_faces(t, torch.arange(B) * F, torch.full((B,), F), x['z_clip'], x['persp'])
    got = 0.
    ntri_t = torch.from_numpy(ntri).long()
    for kk in range(2):
        sel = ntri_t > kk
        got += (cl.face_verts[cl.u2c[sel] + kk].reshape(-1, 9).numpy() * gt[kk][sel.numpy()]).sum()
        sel = sel & torch.from_numpy(clipped)
        got += (cl.conversion[cl.u2c[sel] + kk].reshape(-1, 9).numpy() * gc[kk][sel.numpy()]).sum()
    assert abs(got - want) <= 1e-6 * size, (got, want, size)


# ---------------------------------------------------------------------------------------------------------- inputs
@pytest.mark.parametrize('name', [c['name'] for c in M.FOLD_CASES])
def test_fold_inputs_are_exact_and_decisive(name):
    """the float32 view depth of every (view, vertex) equals the float64 one, clear of z_clip by many ulps, and every clip
    count the case is built for occurs"""
    c = M.FOLD_BY_NAME[name]
    x, _ = M.injected(name)
    z64 = M.fold_depths(x)
    if not x['ndc']:
        v, R, T = x['verts'], x['R'], x['T']
        z32 = v[:, 0] * R[:, 0, 2, None] + v[:, 1] * R[:, 1, 2, None] + v[:, 2] * R[:, 2, 2, None] + T[:, 2, None]
        assert torch.equal(z32.double(), z64)
    if x['z_clip'] >= 0:
        gap = (z64 - x['z_clip']).abs()
        assert gap.min().item() >= 1000 * np.spacing(np.float32(x['z_clip'])), gap.min().item()
        nb = set(M.slot_classes(x)['nb'].reshape(-1).tolist())
        assert nb == {0, 1, 2, 3}, nb
    if c.get('eps_verts'):
        a = z64.abs()
        assert (a == 0).any() and ((a > 0) & (a < x['eps'])).any()
        near = a[(a > 0.5 * x['eps']) & (a < 2 * x['eps'])]
        assert ((near / x["eps"] - 1).abs() >= 5e-4).all() and (near > x['eps']).any() and (near < x['eps']).any()
    if c.get('small_den'):
        z = z64[:, x['faces'].long()]
        d = z.sort(-1).values.diff(dim=-1).min(-1).values           # the closest pair of each face's depths
        assert (d <= 1e-3 * x['z_clip']).sum() >= x['F'] // 3


@pytest.mark.parametrize('name', [c['name'] for c in M.PROJ_CASES])
def test_projection_inputs_sit_where_they_are_meant_to(name):
    """the exact-depth views hold vertices at z = 0 and at +-eps (1 +- 1e-3); every other depth is far from eps"""
    x = M.proj_inputs(name)
    z = M.proj_depths(x)
    B, V = z.shape
    a = z.abs()
    close = (a - x['eps']).abs() < 0.5 * x['eps']
    assert ((a[close] / x['eps'] - 1).abs() >= 9e-4).all()
    if B > 1:
        n_sp = min(V, len(M.SPECIAL_Z))
        assert torch.equal(z[1, :n_sp].float().double(), torch.tensor(M.SPECIAL_Z[:n_sp], dtype=torch.float32).double())
    far = ~close & (a >= x['eps'])
    assert (a[far] >= 2 * x['eps']).all() or (a[far] - x['eps']).min() > 0.1 * x['eps']
