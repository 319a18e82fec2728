"""GPU: the reference's chamfer calls and gradient_icp (tests/golden/chamfer.npz, frozen from its own code) run through
compat.install() -> pytorch3d.ops.knn.knn_points on the sm_90a kernels, and sample_points_from_meshes on CUDA tensors."""
import sys

import numpy as np
import pytest
import torch

from oracle import knn as OK
from tests import _chamfer_golden as CG

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')


@pytest.fixture
def compat_knn():
    """pytorch3d.ops.knn.knn_points as compat.install() registers it; the stand-in modules are removed afterwards"""
    import dbw_b200.compat as compat
    saved = set(sys.modules)
    try:
        compat.install()
        from pytorch3d.ops.knn import knn_points
        yield knn_points
    finally:
        for k in set(sys.modules) - saved:
            if getattr(sys.modules[k], '__dbw_compat__', False):
                del sys.modules[k]


def test_golden_chamfer_calls_through_compat(compat_knn):
    from dbw_b200.pointcloud import knn_points
    assert compat_knn is knn_points
    gold, meta = CG.load()
    n = 0
    for case in meta['cases']:
        if 'error' in case:
            continue
        err, gerr = CG.replay(gold, case, lambda **k: OK.chamfer_distance(**k, knn_points=compat_knn), device=DEV)
        assert err < 1e-5, (case['name'], err)
        assert gerr is None or gerr < 1e-5, (case['name'], gerr)
        n += 1
    assert n >= 20


def test_pytorch3d_chamfer_distance_on_the_golden_calls():
    """PyTorch3D's own chamfer_distance is the reference's with direction_reduction='sum' and return_L1=False (point means
    differ only for empty clouds, which these calls do not divide by)"""
    from dbw_b200.pointcloud import chamfer_distance
    gold, meta = CG.load()
    n = 0
    for case in meta['cases']:
        kw = dict(case['kwargs'])
        if 'error' in case or kw.pop('return_L1', False) or kw.pop('direction_reduction', 'sum') != 'sum':
            continue
        err, gerr = CG.replay(gold, dict(case, kwargs=kw), chamfer_distance, device=DEV)
        assert err < 1e-5 and (gerr is None or gerr < 1e-5), (case['name'], err, gerr)
        n += 1
    assert n >= 5


def test_golden_gradient_icp_through_compat(compat_knn):
    gold, meta = CG.load()
    for case in meta['icp']:
        k = f"icp_{case['name']}__"
        losses = []
        upd, (R, T, s) = OK.gradient_icp(torch.from_numpy(gold[k + 'pred']).to(DEV), torch.from_numpy(gold[k + 'gt']).to(DEV),
                                         lr=meta['lr'], n_iter=meta['n_iter'], knn_points=compat_knn, losses=losses,
                                         **case['kwargs'])
        assert CG.rel(losses, gold[k + 'losses']) < 1e-5, case['name']
        for name, v in (('R', R), ('T', T), ('s', s), ('upd', upd)):
            assert CG.rel(v.cpu().numpy(), gold[k + name]) < 1e-4, (case['name'], name)


def test_sample_points_from_meshes_on_the_gpu():
    from dbw_b200 import geometry as G
    from dbw_b200.pointcloud import sample_points_from_meshes
    from dbw_b200.structures import Meshes
    v, f = G.ico_sphere(2)
    verts = torch.stack([v * torch.tensor([2.0, 1.0, 0.5]), v * 3 + 1]).float()
    m = Meshes(verts.to(DEV), f[None].expand(2, -1, -1).to(DEV))
    torch.manual_seed(3)
    pts, nrm = sample_points_from_meshes(m, 20000, return_normals=True)
    # the same draws, replayed: areas -> multinomial -> rand(2, N, S), then the same torch ops on CPU tensors
    torch.manual_seed(3)
    fv = verts[:, f].to(DEV)
    areas = 0.5 * torch.linalg.cross(fv[:, :, 1] - fv[:, :, 0], fv[:, :, 2] - fv[:, :, 0], dim=-1).norm(dim=-1)
    face = areas.multinomial(20000, replacement=True).cpu()
    u, w = torch.rand(2, 2, 20000, device=DEV).cpu()
    fvc = verts[:, f]
    pick = lambda a: a.gather(1, face[..., None].expand(-1, -1, 3))
    su = u.sqrt()
    want = (1 - su)[..., None] * pick(fvc[:, :, 0]) + (su * (1 - w))[..., None] * pick(fvc[:, :, 1]) \
        + (su * w)[..., None] * pick(fvc[:, :, 2])
    got = pts.cpu()
    assert (got - want).abs().max() <= 4 * torch.finfo(torch.float32).eps * want.abs().max()
    # every sample lies on its face: in its plane and inside its edges
    a, b, c = pick(fvc[:, :, 0]).double(), pick(fvc[:, :, 1]).double(), pick(fvc[:, :, 2]).double()
    nn = torch.linalg.cross(b - a, c - a, dim=-1)
    p = got.double()
    assert (((p - a) * nn).sum(-1) / nn.norm(dim=-1)).abs().max() < 1e-5 * p.abs().max()
    for e0, e1 in ((a, b), (b, c), (c, a)):
        assert (torch.linalg.cross(e1 - e0, p - e0, dim=-1) * nn).sum(-1).min() > -1e-5 * nn.norm(dim=-1).max() ** 2
    nc = nrm.cpu().double()
    assert torch.allclose(nc.norm(dim=-1), torch.ones(2, 20000, dtype=torch.float64), atol=1e-6)
    assert ((nc * nn).sum(-1) / nn.norm(dim=-1)).min() > 1 - 1e-5
