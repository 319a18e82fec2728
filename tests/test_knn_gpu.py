"""GPU: the k-NN kernels (csrc/dbw_knn.cu) through dbw_b200.pointcloud.knn_points -- dists and idx bit for bit against
the float32 oracle (oracle/knn.py) over a covering set of shapes, K buckets, lengths and ties; indices against scipy's
cKDTree at the EMS/MBF size; gradients against the float64 closed form."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import knn as OK

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')


def _run(p1, p2, l1, l2, K):
    from dbw_b200.pointcloud import knn_points
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    r = knn_points(t(p1), t(p2), None if l1 is None else t(l1), None if l2 is None else t(l2), K=K)
    return r.dists.cpu().numpy(), r.idx.cpu().numpy()


def _check(p1, p2, l1, l2, K):
    got = _run(p1, p2, l1, l2, K)
    want = OK.knn_f32(p1, p2, l1, l2, K)
    assert got[0].tobytes() == want[0].tobytes(), 'dists differ'
    assert np.array_equal(got[1], want[1]), 'idx differ'


def _clouds(seed, N, P1, P2):
    g = np.random.default_rng(seed)
    return g.normal(0, 1, (N, P1, 3)).astype(np.float32), g.normal(0, 1.2, (N, P2, 3)).astype(np.float32)


# (N, P1, P2): single points, sizes around the 512-point tile and the 128 / 256-query CTAs, and the long extremes
SHAPES = [(1, 1, 1), (3, 1, 7), (1, 257, 511), (3, 777, 1537), (1, 129, 513), (3, 300, 10), (1, 70000, 513),
          (1, 1000, 70000)]


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('K', [1, 2, 3, 4, 8, 13, 16, 32])
def test_bit_identical_to_the_f32_oracle(shape, K):
    N, P1, P2 = shape
    if P1 * P2 > 1e7 and K not in (1, 8, 32):
        pytest.skip('long shapes: one K per bucket family')
    p1, p2 = _clouds(K, N, P1, P2)
    _check(p1, p2, None, None, K)


@pytest.mark.parametrize('K', [1, 4, 32])
def test_lengths_zero_one_and_full(K):
    p1, p2 = _clouds(5, 3, 600, 900)
    for l1, l2 in (([0, 1, 600], [900, 0, 1]), ([600, 599, 1], [1, 900, 513]), ([1, 0, 600], [0, 1, 900])):
        _check(p1, p2, np.array(l1), np.array(l2), K)


@pytest.mark.parametrize('K', [1, 5, 16])
def test_duplicates_and_exact_ties(K):
    g = np.random.default_rng(40 + K)
    lat = g.integers(-3, 4, (3, 3000, 3)).astype(np.float32)                 # integer lattice: ties everywhere
    p2 = np.concatenate([lat, lat[:, ::5], lat[:, :600]], 1)                 # exact duplicates, across tiles
    p1 = np.concatenate([g.integers(-4, 5, (3, 1100, 3)).astype(np.float32) * 0.5, p2[:, 100:400]], 1)
    _check(p1, p2, None, np.array([p2.shape[1], 1000, 7]), K)


def test_indices_equal_ckdtree_at_the_ems_size():
    g = np.random.default_rng(7)
    n = 500_000
    p1 = g.normal(0, 1, (1, n, 3)).astype(np.float32)
    p2 = (g.normal(0, 1, (1, n, 3)) * [1.2, 0.9, 1.0]).astype(np.float32)
    d, i = _run(p1, p2, None, None, 1)
    td, ti = cKDTree(p2[0].astype(np.float64)).query(p1[0].astype(np.float64), k=2, workers=-1)
    untied = td[:, 1] ** 2 - td[:, 0] ** 2 > 1e-6 * td[:, 1] ** 2
    assert untied.mean() > 0.99
    assert np.array_equal(i[0, untied, 0], ti[untied, 0])
    assert np.allclose(d[0, :, 0], td[:, 0] ** 2, rtol=1e-5, atol=1e-10)


@pytest.mark.parametrize('K', [1, 4, 32])
def test_gradients_match_the_f64_closed_form(K):
    from dbw_b200.pointcloud import knn_points
    p1, p2 = _clouds(9, 2, 3000, 2500)
    l1, l2 = np.array([3000, 1777]), np.array([2000, 2500])
    g = np.random.default_rng(10).normal(size=(2, 3000, K)).astype(np.float32)
    t1 = torch.from_numpy(p1).to(DEV).requires_grad_(True)
    t2 = torch.from_numpy(p2).to(DEV).requires_grad_(True)
    r = knn_points(t1, t2, torch.from_numpy(l1).to(DEV), torch.from_numpy(l2).to(DEV), K=K)
    (r.dists * torch.from_numpy(g).to(DEV)).sum().backward()
    w1, w2 = OK.knn_backward_f64(p1, p2, l1, l2, r.idx.cpu().numpy(), g)
    for got, want in ((t1.grad, w1), (t2.grad, w2)):
        got = got.cpu().numpy().astype(np.float64)
        assert np.linalg.norm(got - want) / np.linalg.norm(want) < 1e-5
    assert not t1.grad[1, 1777:].any()


def test_return_nn_and_knn_gather():
    from dbw_b200.pointcloud import knn_points
    p1, p2 = _clouds(11, 2, 100, 6)
    l2 = torch.tensor([6, 3], device=DEV)
    r = knn_points(torch.from_numpy(p1).to(DEV), torch.from_numpy(p2).to(DEV), lengths2=l2, K=4, return_nn=True)
    want = torch.from_numpy(p2).to(DEV)[torch.arange(2, device=DEV)[:, None, None], r.idx]
    want[1, :, 3:] = 0
    assert torch.equal(r.knn, want)
    with pytest.raises(Exception):
        knn_points(torch.zeros(1, 4, 3, device=DEV), torch.zeros(1, 4, 3, device=DEV), K=33)
    with pytest.raises(Exception):
        knn_points(torch.zeros(1, 4, 3, device=DEV, dtype=torch.float64), torch.zeros(1, 4, 3, device=DEV, dtype=torch.float64))
