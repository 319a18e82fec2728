"""CPU: the k-NN oracle (oracle/knn.py) against scipy's cKDTree and a sort-based brute force, the oracle's chamfer and
gradient_icp against the reference's own (tests/golden/chamfer.npz), the argument checks of the chamfer helpers, the
arithmetic of sample_points_from_meshes, the compat registration and the C-ABI checks of dbw_knn_* without a GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from tests import _chamfer_golden as CG
from oracle import knn as OK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _brute(p1, p2, l1, l2, K):
    """float32 distances in the kernel's order, then a full lexicographic (distance, index) sort per row"""
    N, P1 = p1.shape[:2]
    d_out, i_out = np.zeros((N, P1, K), np.float32), np.zeros((N, P1, K), np.int64)
    for n in range(N):
        q, t = p1[n, :l1[n]], p2[n, :l2[n]]
        dx, dy, dz = (q[:, None, c] - t[None, :, c] for c in range(3))
        d = (dx * dx + dy * dy) + dz * dz
        for r in range(len(q)):
            o = np.lexsort((np.arange(len(t)), d[r]))[:K]
            d_out[n, r, :len(o)], i_out[n, r, :len(o)] = d[r, o], o
    return d_out, i_out


@pytest.mark.parametrize('K', [1, 3, 8])
def test_f64_oracle_matches_ckdtree(K):
    g = np.random.default_rng(K)
    p1, p2 = g.uniform(-3, 3, (2, 700, 3)), g.normal(0, 1.5, (2, 900, 3))
    d, i = OK.knn_f64(p1, p2, K=K)
    for n in range(2):
        td, ti = cKDTree(p2[n]).query(p1[n], k=K)
        td, ti = td.reshape(-1, K), ti.reshape(-1, K)
        assert np.array_equal(i[n], ti)
        assert np.allclose(d[n], td ** 2, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('K', [1, 2, 5, 16])
def test_f32_oracle_on_ties_matches_a_sort(K):
    g = np.random.default_rng(10 + K)
    lattice = g.integers(-2, 3, (2, 400, 3)).astype(np.float32)                       # many exact ties
    p2 = np.concatenate([lattice, lattice[:, ::7]], 1)                                  # and exact duplicates
    p1 = np.concatenate([g.integers(-3, 4, (2, 150, 3)).astype(np.float32) * 0.5, p2[:, :50]], 1)
    l1, l2 = np.array([200, 17]), np.array([p2.shape[1], 3])                           # 3 < K: padding slots
    want = _brute(p1, p2, l1, l2, K)
    got = OK.knn_f32(p1, p2, l1, l2, K)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
    assert not got[0][1, 17:].any() and not got[1][1, 17:].any()                       # rows beyond lengths1
    if K > 3:
        assert not got[1][1, :17, 3:].any() and not got[0][1, :17, 3:].any()


def test_oracle_backward_is_the_gradient_of_the_distances():
    g = np.random.default_rng(3)
    p1, p2 = g.normal(size=(1, 40, 3)), g.normal(size=(1, 50, 3))
    gd = g.normal(size=(1, 40, 4))
    d, i = OK.knn_f64(p1, p2, K=4)
    g1, g2 = OK.knn_backward_f64(p1, p2, None, None, i, gd)
    t1, t2 = torch.tensor(p1, requires_grad=True), torch.tensor(p2, requires_grad=True)
    dd = ((t1[0, :, None] - t2[0][torch.from_numpy(i[0])]) ** 2).sum(-1)
    (dd * torch.from_numpy(gd[0])).sum().backward()
    assert np.allclose(g1, t1.grad.numpy(), atol=1e-12) and np.allclose(g2, t2.grad.numpy(), atol=1e-12)


# ------------------------------------------------------------------------------------------------ golden
def test_oracle_chamfer_reproduces_the_reference():
    gold, meta = CG.load()
    n = 0
    for case in meta['cases']:
        if 'error' in case:
            continue
        err, gerr = CG.replay(gold, case, OK.chamfer_distance)
        assert err < 1e-6, (case['name'], err)
        assert gerr is None or gerr < 1e-6, (case['name'], gerr)
        n += 1
    assert n >= 20


def test_oracle_gradient_icp_reproduces_the_reference():
    gold, meta = CG.load()
    for case in meta['icp']:
        k = f"icp_{case['name']}__"
        losses = []
        upd, (R, T, s) = OK.gradient_icp(torch.from_numpy(gold[k + 'pred']), torch.from_numpy(gold[k + 'gt']), lr=meta['lr'],
                                         n_iter=meta['n_iter'], losses=losses, **case['kwargs'])
        assert CG.rel(losses, gold[k + 'losses']) < 1e-6
        for name, v in (('R', R), ('T', T), ('s', s), ('upd', upd)):
            assert CG.rel(v.numpy(), gold[k + name]) < 1e-5, (case['name'], name)


def test_chamfer_helpers_raise_where_the_reference_raises():
    from dbw_b200 import pointcloud as PC
    gold, meta = CG.load()

    def run(args, kw):
        PC._validate_chamfer_reduction_inputs(kw.get('batch_reduction', 'mean'), kw.get('point_reduction', 'mean'))
        x, xl, xn = PC._handle_pointcloud_input(args['x'], args.get('x_lengths'), args.get('x_normals'))
        y, yl, yn = PC._handle_pointcloud_input(args['y'], args.get('y_lengths'), args.get('y_normals'))
        return OK.chamfer_distance(x, y, xl, yl, xn, yn, args.get('weights'), **kw)
    raised = 0
    for case in meta['cases']:
        args = CG.tensors(gold, case['arrays'])
        if 'error' in case:
            with pytest.raises(ValueError) as e:
                run(args, case['kwargs'])
            assert [type(e.value).__name__, str(e.value)] == case['error'], case['name']
            raised += 1
        else:
            run(args, case['kwargs'])
    assert raised == 10
    with pytest.raises(NotImplementedError):
        PC._handle_pointcloud_input(type('Pointclouds', (), {})(), None, None)


# ------------------------------------------------------------------------------------------------ sampling
def _numpy_samples(verts, faces, face, uv):
    fv = verts[faces].astype(np.float64)                                   # (F, 3, 3)
    u, v = uv.astype(np.float64)
    su = np.sqrt(u)
    w = np.stack([1 - su, su * (1 - v), su * v], -1)                       # (S, 3)
    pts = (w[:, :, None] * fv[face]).sum(1)
    n = np.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 1])
    n = n / np.linalg.norm(n, axis=1, keepdims=True)
    return pts, n[face], 0.5 * np.linalg.norm(np.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0]), axis=1)


def test_sample_points_from_meshes_arithmetic_matches_numpy():
    from dbw_b200 import geometry as G
    from dbw_b200.pointcloud import sample_points_from_meshes
    from dbw_b200.structures import Meshes
    v, f = G.ico_sphere(1)
    v = (v * torch.tensor([2.0, 1.0, 0.5])).float()
    verts = torch.stack([v, v * 3 + 1])
    degenerate = torch.zeros_like(v)                                         # zero total area: zeros, not sampled
    m = Meshes(torch.cat([verts, degenerate[None]]), f[None].expand(3, -1, -1))
    torch.manual_seed(5)
    pts, nrm = sample_points_from_meshes(m, 1000, return_normals=True)
    assert pts.shape == nrm.shape == (3, 1000, 3) and pts.dtype == torch.float32
    assert not pts[2].any() and not nrm[2].any()
    torch.manual_seed(5)                                                     # PyTorch3D's draws, in its order
    fv = verts[:, f]
    areas = 0.5 * torch.linalg.cross(fv[:, :, 1] - fv[:, :, 0], fv[:, :, 2] - fv[:, :, 0], dim=-1).norm(dim=-1)
    face = areas.multinomial(1000, replacement=True)
    uv = torch.rand(2, 2, 1000)
    for n in range(2):
        want, wn, wa = _numpy_samples(verts[n].numpy(), f.numpy(), face[n].numpy(), uv[:, n].numpy())
        assert np.allclose(areas[n].numpy(), wa, rtol=1e-5)
        assert np.abs(pts[n].numpy() - want).max() < 4e-6 * np.abs(want).max()
        assert np.abs(nrm[n].numpy() - wn).max() < 1e-5
    with pytest.raises(ValueError):
        sample_points_from_meshes(Meshes(verts, torch.zeros(2, 0, 3, dtype=torch.long)), 10)
    with pytest.raises(NotImplementedError):
        sample_points_from_meshes(m, 10, return_textures=True)
    assert sample_points_from_meshes(Meshes(verts, f[None].expand(2, -1, -1)), 7).shape == (2, 7, 3)


# ------------------------------------------------------------------------------------------------ interface
def test_knn_points_refuses_what_it_does_not_implement():
    from dbw_b200._lib import DbwError
    from dbw_b200.pointcloud import knn_points
    x = torch.zeros(1, 5, 3)
    with pytest.raises(DbwError):
        knn_points(x, x)                                                     # CPU tensors: no fallback
    with pytest.raises(NotImplementedError):
        knn_points(x, x, norm=1)
    with pytest.raises(NotImplementedError):
        knn_points(torch.zeros(1, 5, 2), torch.zeros(1, 5, 2))
    with pytest.raises(ValueError):
        knn_points(x, torch.zeros(2, 5, 3))


def test_knn_c_abi_checks_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    assert L.dbw_knn_forward(*([None] * 4), 1, 5, 5, 33, None, None, None) != 0 and b'bad sizes' in L.dbw_last_error()
    assert L.dbw_knn_forward(*([None] * 4), 1, 5, 5, 0, None, None, None) != 0
    assert L.dbw_knn_forward(*([None] * 4), 70000, 5, 5, 1, None, None, None) != 0
    assert L.dbw_knn_forward(*([None] * 4), 1, 5, 5, 4, None, None, None) != 0 and b'null pointer' in L.dbw_last_error()
    assert L.dbw_knn_backward(*([None] * 6), 1, 5, 5, 4, None, None, None) != 0 and b'null pointer' in L.dbw_last_error()
    assert L.dbw_knn_forward(*([None] * 4), 0, 5, 5, 4, None, None, None) == 0          # empty: nothing to do
    assert L.dbw_knn_backward(*([None] * 6), 1, 0, 5, 4, None, None, None) == 0


def test_compat_registers_the_point_cloud_ops():
    """in a subprocess (the stand-ins must not leak): the reference's chamfer imports resolve to dbw_b200.pointcloud,
    the SVD ICP and Pointclouds stay placeholders"""
    code = r'''
import sys; sys.path.insert(0, %r)
import dbw_b200, dbw_b200.compat as compat
from dbw_b200 import pointcloud as PC
if 'pytorch3d' in compat.install():
    from pytorch3d.ops.knn import knn_gather, knn_points
    from pytorch3d.ops import sample_points_from_meshes, knn_points as k2, iterative_closest_point
    from pytorch3d.loss import chamfer_distance
    from pytorch3d.loss.chamfer import _validate_chamfer_reduction_inputs, _handle_pointcloud_input, chamfer_distance as c2
    from pytorch3d.structures import Pointclouds
    assert knn_points is k2 is PC.knn_points and knn_gather is PC.knn_gather
    assert sample_points_from_meshes is PC.sample_points_from_meshes and chamfer_distance is c2 is PC.chamfer_distance
    assert _validate_chamfer_reduction_inputs is PC._validate_chamfer_reduction_inputs
    assert _handle_pointcloud_input is PC._handle_pointcloud_input
    for P in (iterative_closest_point, Pointclouds):
        try:
            P()
            raise SystemExit('placeholder did not raise')
        except NotImplementedError:
            pass
print('OK')
''' % ROOT
    res = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and 'OK' in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
