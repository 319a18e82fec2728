"""GPU: the RANSAC kernels (csrc/dbw_ransac.cu) against the float64 oracle (oracle/baselines.py) and the reference's own
Ransac (tests/golden/baselines.npz), from 10^3 to 3 10^6 points; the preprocessing against the reference's outputs; and the
EMS / MBF evaluators against a torch composition of the same stages."""
import json
import types

import numpy as np
import pytest
import torch

from oracle import baselines as O
from oracle import knn as OK
from tests.golden.make_baselines_golden import PREPROCESS_SEED, RANSAC_CASES, cloud, scan
from tests.test_baselines_host import GOLDEN, THRESH, _within_boundary
from tests.test_dtu_eval_gpu import _dtu_dir

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
LARGE_CASES = [(1000, 21), (250000, 4), (3000000, 8)]


def _fit(pc_np, seed):
    from dbw_b200 import baselines as B
    pc = torch.from_numpy(pc_np).to(DEV)
    torch.manual_seed(seed)
    fit = B._ransac(pc, 3, 100, 10, THRESH)
    torch.cuda.synchronize()
    return pc, fit


def _check_against_oracle(pc_np, fit):
    idx = fit['idx'].cpu().numpy().reshape(-1, 3)
    params64, _ = O.solve(pc_np, idx)
    params = fit['params'].cpu().numpy()
    assert params.tobytes() == params64.astype(np.float32).tobytes()
    counts = fit['counts'].cpu().numpy()
    for h in range(len(idx)):
        assert _within_boundary(pc_np, params64[h], counts[h], 1.0), h
    best, best_n, improvements = O.select(counts, 10)
    assert (fit['hypothesis'], fit['n_inliers'], fit['n_models']) == (best, best_n, improvements)
    assert np.array_equal(np.asarray(fit['model'], np.float32), params[best])
    return idx, params64, counts


@pytest.mark.parametrize('n,seed', RANSAC_CASES)
def test_ransac_reproduces_the_reference(n, seed):
    from dbw_b200.baselines import ransac_filter, ransac_ground_mask
    k = f'ransac_{n}_{seed}__'
    pc_np = cloud(n, seed)
    pc, fit = _fit(pc_np, seed)
    idx, params64, counts = _check_against_oracle(pc_np, fit)
    assert np.array_equal(idx, GOLDEN[k + 'draws'])                              # the reference's draws
    assert fit['hypothesis'] == O.select(GOLDEN[k + 'counts'], 10)[0]
    assert (fit['n_inliers'], fit['n_models']) == (GOLDEN[k + 'best_n'], GOLDEN[k + 'n_models'])
    np.testing.assert_allclose(fit['model'], GOLDEN[k + 'model'], rtol=1e-5, atol=1e-6)
    keep = np.unpackbits(GOLDEN[k + 'keep'])[:n].astype(bool)
    assert len(O.boundary(pc_np, params64[fit['hypothesis']], THRESH)) == 0
    torch.manual_seed(seed)
    mask, model, n_in = ransac_ground_mask(pc)
    assert np.array_equal(~mask.cpu().numpy(), keep) and model == fit['model'] and n_in == fit['n_inliers']
    torch.manual_seed(seed)
    kept, model, n_in = ransac_filter(pc)
    assert kept.cpu().numpy().tobytes() == pc_np[keep].tobytes()                   # the reference's cloud, in order


@pytest.mark.parametrize('n,seed', LARGE_CASES)
def test_ransac_counts_and_filter_against_the_oracle(n, seed):
    from dbw_b200 import baselines as B
    pc_np = cloud(n, seed)
    pc, fit = _fit(pc_np, seed)
    _, params64, _ = _check_against_oracle(pc_np, fit)
    best = fit['hypothesis']
    inlier = torch.empty(n, dtype=torch.uint8, device=DEV)
    kept = torch.full((n, 3), float('nan'), device=DEV)
    n_kept = B._filter(pc, fit, THRESH, kept=kept, inlier=inlier)
    ref = O.inliers(pc_np, params64[best], THRESH)
    got = inlier.bool().cpu().numpy()
    differ = np.nonzero(got != ref)[0]
    assert np.isin(differ, O.boundary(pc_np, params64[best], THRESH)).all()
    assert int(n_kept.item()) == n - fit['n_inliers'] == int((~got).sum())
    assert kept[:n - fit['n_inliers']].cpu().numpy().tobytes() == pc_np[~got].tobytes()
    assert torch.isnan(kept[n - fit['n_inliers']:]).all()                           # nothing written past the kept points


def test_two_calls_give_identical_bits():
    from dbw_b200.baselines import ransac_filter
    pc_np = cloud(1000000, 13)
    a, b = _fit(pc_np, 13)[1], _fit(pc_np, 13)[1]
    for key in ('idx', 'params', 'counts', 'result'):
        assert torch.equal(a[key], b[key]), key
    pc = torch.from_numpy(pc_np).to(DEV)
    torch.manual_seed(13)
    k1 = ransac_filter(pc)[0]
    torch.manual_seed(13)
    k2 = ransac_filter(pc)[0]
    assert k1.cpu().numpy().tobytes() == k2.cpu().numpy().tobytes()


def test_non_finite_points_are_never_inliers():
    from dbw_b200.baselines import ransac_filter
    pc_np = cloud(5000, 2)
    pc_np[::7, 2] = np.nan
    pc_np[3::11, 0] = np.inf
    pc = torch.from_numpy(pc_np).to(DEV)
    torch.manual_seed(2)
    kept, model, n_in = ransac_filter(pc)
    bad = ~np.isfinite(pc_np).all(1)
    k = kept.cpu().numpy()
    assert (~np.isfinite(k).all(1)).sum() == bad.sum()                               # every non-finite point is kept


@pytest.mark.parametrize('name', ['ems', 'mbf'])
@pytest.mark.parametrize('filter_ground', [False, True])
def test_preprocess_writes_the_reference_files(tmp_path, name, filter_ground):
    from dbw_b200.baselines import DTU3DPreprocess
    from dbw_b200.dtu_eval import read_ply
    pc_gt, scale_mat = scan()
    ds = types.SimpleNamespace(pc_gt=torch.from_numpy(pc_gt), scale_mat=torch.from_numpy(scale_mat))
    DTU3DPreprocess(tmp_path, name, filter_ground=filter_ground, device=DEV).run({'scan7': ds}, seed=PREPROCESS_SEED)
    k = f'preprocess_{name}_{int(filter_ground)}__'
    # the device's matmul and mean round differently from the CPU's in the last bits
    np.testing.assert_allclose(np.load(tmp_path / 'scan7_scale.npy'), GOLDEN[k + 'scale'], rtol=1e-6)
    ply = read_ply(tmp_path / 'scan7.ply')
    assert ply.shape == GOLDEN[k + 'ply'].shape
    np.testing.assert_allclose(ply, GOLDEN[k + 'ply'], rtol=0, atol=2e-5)


# ------------------------------------------------------------------------------------------------ evaluators
SCALE_MAT = np.array([[212.5, 0, 0, -11.25], [0, 212.5, 0, 37.5], [0, 0, 212.5, 640.0], [0, 0, 0, 1]], np.float32)


def _scene_fixture(tmp_path, verts_world):
    """a synthetic scan: pc_gt (standardised space) near the baseline's surface, an STL cloud, ObsMask and Plane"""
    g = np.random.default_rng(1)
    v = verts_world.reshape(-1, 3)
    stl = (v[g.integers(0, len(v), 6000)] + g.normal(0, 0.5, (6000, 3))).astype(np.float32).astype(np.float64)
    lo, hi = v.min(0) - 5, v.max(0) + 5
    res = 2.0
    obs = np.ones(tuple(int(x) for x in np.ceil((hi - lo) / res) + 1), bool)
    plane = np.array([[0.], [0.], [1.], [-(lo[2] + 3)]])
    _dtu_dir(tmp_path / 'DTU', 7, stl, obs, np.stack([lo, hi]), np.array([[res]]), plane)
    inv = np.linalg.inv(SCALE_MAT.astype(np.float64))
    gt = (stl[:4000] + g.normal(0, 0.3, (4000, 3))) @ inv[:3, :3] + inv[:3, 3]
    return types.SimpleNamespace(pc_gt=torch.from_numpy(gt.astype(np.float32)), scale_mat=torch.from_numpy(SCALE_MAT)), \
        dict(stl=stl, obs=obs, bb=np.stack([lo, hi]), res=np.array([[res]]), plane=plane)


def _composition(ds, scene_cpu, seed, dtu, dtu_seed):
    """the evaluation's stages composed from torch and the oracle's chamfer (the reference's chamfer_distance)"""
    from dbw_b200.baselines import N_POINTS_EVAL
    from dbw_b200.dtu_eval import evaluate_arrays
    from dbw_b200.pointcloud import knn_points, sample_points_from_meshes
    torch.manual_seed(seed)
    gt = ds.pc_gt[torch.randperm(len(ds.pc_gt))][:N_POINTS_EVAL]
    points = sample_points_from_meshes(scene_cpu, num_samples=N_POINTS_EVAL).to(DEV)
    inv = ds.scale_mat.inverse().to(DEV)
    points = points @ inv[:3, :3] + inv[:3, 3]
    acc, comp = OK.chamfer_distance(points, gt[None].to(DEV), return_L1=True, direction_reduction='none',
                                    knn_points=knn_points)[0]
    v, f = scene_cpu.get_mesh_verts_faces(0)
    r = evaluate_arrays(v, f, dtu['stl'], dtu['obs'], dtu['bb'], dtu['res'], dtu['plane'], seed=dtu_seed, device=DEV)
    return 10 * acc.item(), 10 * comp.item(), r['acc'], r['comp']


def _check_scores(tmp_path, got, want):
    s = got['scan7']
    np.testing.assert_allclose([s['chL1_acc'], s['chL1_comp'], s['acc'], s['comp']], want, rtol=1e-6, atol=0)
    lines = (tmp_path / 'run' / 'scan7_scores.tsv').read_text().splitlines()
    assert lines[0] == 'n_blocks\tchL1_acc\tchL1_comp'
    assert lines[1] == '\t'.join('{:.5f}'.format(x) for x in (s['n_blocks'], s['chL1_acc'], s['chL1_comp']))
    assert (tmp_path / 'run' / 'dtu_scores_scan7.tsv').read_text().startswith('acc\tcomp\tavg\n')


def test_ems_evaluator_equals_the_composition(tmp_path):
    from scipy.spatial.transform import Rotation
    from dbw_b200.baselines import EMSEvaluator
    from dbw_b200.geometry import ico_sphere, signed_pow
    from dbw_b200.structures import Meshes, join_meshes_as_scene
    g = np.random.default_rng(5)
    N = 4
    spq = np.c_[g.uniform(0.2, 1.5, (N, 2)), g.uniform(0.5, 1.5, (N, 3)), g.uniform(-np.pi, np.pi, (N, 3)),
                g.uniform(-4, 4, (N, 3))]
    mean, scale = np.array([-2.0, 35.0, 660.0], np.float32), np.float32(0.05)
    (tmp_path / 'ems').mkdir()
    np.save(tmp_path / 'ems' / 'scan7_spq.npy', spq)
    np.save(tmp_path / 'ems' / 'scan7_scale.npy', np.r_[mean, scale].astype(np.float32))
    # the scene, restated: parametric superquadrics on the level-1 icosphere, rotated ZYX, translated, mapped back
    p = torch.from_numpy(spq).float()
    v, f = ico_sphere(1)
    eta, omega = torch.asin(v[:, 1])[None].expand(N, -1), torch.atan2(v[:, 0], v[:, 2])[None].expand(N, -1)
    e1, e2 = p[:, 0:1], p[:, 1:2]
    ce, se, co, so = signed_pow(torch.cos(eta), e1), signed_pow(torch.sin(eta), e1), signed_pow(torch.cos(omega), e2), \
        signed_pow(torch.sin(omega), e2)
    verts = torch.stack([ce * so, se, ce * co], -1) * p[:, None, 2:5]
    R = torch.from_numpy(Rotation.from_euler('ZYX', spq[:, 5:8]).as_matrix()).float()
    verts = (R @ verts.permute(0, 2, 1) + p[:, 8:11, None]).permute(0, 2, 1) / torch.from_numpy(np.r_[scale]) \
        + torch.from_numpy(mean)
    scene = join_meshes_as_scene(Meshes(verts, f[None].expand(N, -1, -1)))
    ds, dtu = _scene_fixture(tmp_path, verts.numpy())
    want = _composition(ds, scene, 3, dtu, 11)
    got = EMSEvaluator(tmp_path / 'run', tmp_path / 'ems', device=DEV).run({'scan7': ds}, tmp_path / 'DTU', seed=3, dtu_seed=11)
    assert got['scan7']['n_blocks'] == N
    _check_scores(tmp_path, got, want)


def test_mbf_evaluator_equals_the_composition(tmp_path):
    from dbw_b200.baselines import MBFEvaluator, box_hull_faces
    from dbw_b200.geometry import random_rotations
    from dbw_b200.structures import Meshes, join_meshes_as_scene
    g = np.random.default_rng(6)
    N = 5
    unit = np.array([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)], np.float64)
    R = random_rotations(N, generator=torch.Generator().manual_seed(6)).numpy().astype(np.float64)
    bbox = np.stack([(unit * g.uniform(0.3, 1.2, 3)) @ R[i].T + g.uniform(-3, 3, 3) for i in range(N)])
    mean, scale = np.array([-2.0, 35.0, 660.0], np.float32), np.float32(0.025)
    (tmp_path / 'mbf' / 'scan7').mkdir(parents=True)
    np.save(tmp_path / 'mbf' / 'scan7_scale.npy', np.r_[mean, scale].astype(np.float32))
    (tmp_path / 'mbf' / 'scan7' / 'UH.json').write_text(json.dumps({'bbox': bbox.tolist()}))
    verts = torch.Tensor(bbox.tolist()).float() / torch.from_numpy(np.r_[scale]) + torch.from_numpy(mean)
    faces = torch.stack([torch.from_numpy(box_hull_faces(v.numpy())) for v in verts])
    scene = join_meshes_as_scene(Meshes(verts, faces))
    ds, dtu = _scene_fixture(tmp_path, verts.numpy())
    want = _composition(ds, scene, 4, dtu, 12)
    got = MBFEvaluator(tmp_path / 'run', tmp_path / 'mbf', device=DEV).run({'scan7': ds}, tmp_path / 'DTU', seed=4, dtu_seed=12)
    assert got['scan7']['n_blocks'] == N
    _check_scores(tmp_path, got, want)
