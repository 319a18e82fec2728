"""GPU: the DTU chamfer evaluation kernels (csrc/dbw_eval.cu) against the CPU restatement (oracle/mesh_eval.py), and
dbw_b200.dtu_eval.evaluate_mesh against tests/golden/dtu_eval.npz (the reference's own evaluate_mesh on a synthetic
scene), including the trainer's call sequence on a model."""
import os
from copy import deepcopy

import numpy as np
import pytest
import torch
from scipy.io import savemat
from scipy.spatial import cKDTree

from oracle import mesh_eval as M

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device('cuda:0')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(HERE, 'golden', 'dtu_eval.npz')))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _dtu_dir(root, scan, stl, obs_mask, bb, res, plane):
    from dbw_b200.dtu_eval import write_ply
    os.makedirs(os.path.join(root, 'ObsMask'), exist_ok=True)
    os.makedirs(os.path.join(root, 'Points', 'stl'), exist_ok=True)
    savemat(os.path.join(root, 'ObsMask', f'ObsMask{scan}_10.mat'), {'ObsMask': obs_mask, 'BB': bb, 'Res': res})
    savemat(os.path.join(root, 'ObsMask', f'Plane{scan}.mat'), {'P': plane})
    write_ply(os.path.join(root, 'Points', 'stl', f'stl{scan:03}_total.ply'), stl)


# ------------------------------------------------------------------------------------------------ sampling
def test_sampling_is_bit_identical_to_the_oracle(gold):
    from dbw_b200.dtu_eval import sample_mesh_points
    V = gold['verts'].astype(np.float64)
    v, f = M.remove_unreferenced(V, gold['faces'])
    got = sample_mesh_points(_cuda(v), _cuda(f)).cpu().numpy()
    assert got.tobytes() == M.sample_mesh(v, f).tobytes()
    # random, thin, huge triangles (one with ~1e5 samples: its rows are split over warps)
    g = np.random.default_rng(8)
    tv = g.normal(0, 4, (300, 3, 3)) + g.uniform(-200, 200, (300, 1, 3))
    tv[::9, 2] = tv[::9, 0] + (tv[::9, 1] - tv[::9, 0]) * 0.37 + 1e-4
    tv[5] = [[-50, -40, 3], [60, -35, 9], [-8, 70, -2]]
    tv[17, 2] = tv[17, 1]
    tv = tv.astype(np.float32).astype(np.float64).reshape(-1, 3)
    f = np.arange(len(tv)).reshape(-1, 3)
    want = M.sample_mesh(tv, f)
    assert len(want) > 100000
    assert sample_mesh_points(_cuda(tv), _cuda(f)).cpu().numpy().tobytes() == want.tobytes()
    assert sample_mesh_points(_cuda(tv), _cuda(f[:0])).shape == (0, 3)


# ------------------------------------------------------------------------------------------------ downsample
def test_radius_downsample_equals_the_greedy_loop_with_duplicates():
    from dbw_b200.dtu_eval import radius_downsample
    g = np.random.default_rng(1)
    pts = g.uniform(0, 12, (70000, 3))
    pts = np.concatenate([pts, pts[g.integers(0, len(pts), 30000)]])            # exact duplicates
    pts = pts[g.permutation(len(pts))]
    keep, rounds = radius_downsample(_cuda(pts))
    want = M.greedy_downsample(pts)
    assert np.array_equal(keep.cpu().numpy(), want)
    assert 1 <= rounds < 200
    print(f'downsample of {len(pts)} points: {rounds} rounds, {want.sum()} kept')


def test_radius_downsample_equals_the_greedy_loop_on_a_clustered_cloud():
    """a chain in chain order (each decision waits for the previous one: many rounds) plus dense clusters"""
    from dbw_b200._lib import DbwError
    from dbw_b200.dtu_eval import radius_downsample
    g = np.random.default_rng(2)
    chain = np.stack([np.arange(1500) * 0.15, np.zeros(1500), np.zeros(1500)], 1) + g.normal(0, 1e-4, (1500, 3))
    blobs = np.concatenate([g.normal(c, 0.25, (4000, 3)) for c in g.uniform(-30, -5, (10, 3))])
    blobs = blobs[g.permutation(len(blobs))]
    pts = np.concatenate([chain, blobs])
    keep, rounds = radius_downsample(_cuda(pts))
    assert np.array_equal(keep.cpu().numpy(), M.greedy_downsample(pts))
    assert rounds > 20
    print(f'clustered cloud: {rounds} rounds')
    with pytest.raises(DbwError, match='max_rounds'):
        radius_downsample(_cuda(chain), max_rounds=3)
    k0, r0 = radius_downsample(_cuda(pts[:0]))
    assert k0.shape == (0,) and r0 == 0


# ------------------------------------------------------------------------------------------------ nearest neighbour
def _check_nn(q, t, got):
    want = M.nn_distance(q, t)
    got = got.cpu().numpy()
    assert np.array_equal(np.isinf(got), np.isinf(want))
    fin = np.isfinite(want)
    np.testing.assert_allclose(got[fin], want[fin], rtol=1e-12, atol=0)
    return fin


def test_nearest_distances_match_ckdtree():
    from dbw_b200.dtu_eval import nearest_distances
    g = np.random.default_rng(5)
    # a surface-like target cloud (sphere shells), queries near it, inside it and far from it
    d = g.normal(size=(200000, 3))
    t = d / np.linalg.norm(d, axis=1, keepdims=True) * g.choice([40., 90.], (200000, 1)) + g.normal(0, 0.3, (200000, 3))
    q = np.concatenate([t[:50000] + g.normal(0, 2, (50000, 3)), g.uniform(-150, 150, (50000, 3)),
                        g.normal(0, 1, (2000, 3)) + [300, 0, 0]])
    fin = _check_nn(q, t, nearest_distances(_cuda(q), _cuda(t)))
    assert 0 < fin.sum() < len(q)
    # duplicates among the targets, and queries exactly on targets
    t2 = np.concatenate([t[:1000], t[:1000]])
    _check_nn(t2[:500], t2, nearest_distances(_cuda(t2[:500]), _cuda(t2)))


def test_nearest_distances_edge_cases():
    from dbw_b200.dtu_eval import nearest_distances
    g = np.random.default_rng(6)
    t = g.normal(0, 5, (1000, 3))
    far = g.normal(0, 1, (300, 3)) + [0, 0, 80]                              # every query farther than 20
    out = nearest_distances(_cuda(far), _cuda(t))
    assert torch.isinf(out).all()
    assert nearest_distances(_cuda(far[:0]), _cuda(t)).shape == (0,)
    assert torch.isinf(nearest_distances(_cuda(far), _cuda(t[:0]))).all()
    one = t[:1]                                                               # a single target
    _check_nn(t, one, nearest_distances(_cuda(t), _cuda(one)))
    flat = t.copy()                                                           # a flat target set (zero extent in z)
    flat[:, 2] = 1.5
    _check_nn(t, flat, nearest_distances(_cuda(t), _cuda(flat)))


def test_point_functions_refuse_cpu_tensors():
    from dbw_b200._lib import DbwError
    from dbw_b200.dtu_eval import nearest_distances, radius_downsample
    with pytest.raises(DbwError):
        radius_downsample(torch.zeros(4, 3, dtype=torch.float64))
    with pytest.raises(DbwError):
        nearest_distances(torch.zeros(4, 3, dtype=torch.float64, device=DEV), torch.zeros(4, 3, dtype=torch.float64))


# ------------------------------------------------------------------------------------------------ evaluate_mesh
def test_evaluate_mesh_reproduces_the_reference_golden(gold, tmp_path, capsys):
    from dbw_b200 import Meshes
    from dbw_b200.dtu_eval import evaluate_arrays, evaluate_mesh, read_ply
    _dtu_dir(tmp_path / 'DTU', 7, gold['stl'], gold['obs_mask'], gold['bb'], gold['res'], gold['plane'])
    out = tmp_path / 'run'
    out.mkdir()
    mesh = Meshes(torch.from_numpy(gold['verts'])[None].to(DEV), torch.from_numpy(gold['faces'])[None].to(DEV))
    s = evaluate_mesh(mesh, 7, tmp_path / 'DTU', out, order=gold['order'])
    np.testing.assert_allclose([s['acc'], s['comp'], s['avg']], gold['scores'], rtol=1e-12, atol=0)
    tsv, want = (out / 'dtu_scores.tsv').read_text(), str(gold['tsv'])
    assert tsv.split('\n')[0] == want.split('\n')[0] and not tsv.endswith('\n') and tsv.count('\t') == want.count('\t')
    np.testing.assert_allclose([float(x) for x in tsv.split('\n')[1].split('\t')],
                               [float(x) for x in want.split('\n')[1].split('\t')], rtol=1e-12, atol=0)
    print('TSV identical to the reference text:', tsv == want)
    assert 'dtu_scores: acc=' in capsys.readouterr().out
    # the intermediate clouds, exactly
    r = evaluate_arrays(gold['verts'], gold['faces'], gold['stl'], gold['obs_mask'], gold['bb'], gold['res'], gold['plane'],
                        order=gold['order'])
    assert r['shuffled'].cpu().numpy().tobytes() == gold['shuffled'].tobytes()
    assert r['data_in'].cpu().numpy().tobytes() == gold['data_in'].tobytes()
    assert r['data_in_obs'].cpu().numpy().tobytes() == gold['data_in'][gold['data_in_obs_mask']].tobytes()
    assert r['stl_above'].cpu().numpy().tobytes() == gold['stl'][gold['stl_above_mask']].tobytes()
    # the visualisation clouds: data_down / stl, coloured as the reference colours them
    d2s_ply, s2d_ply = out / 'vis_007_d2s.ply', out / 'vis_007_s2d.ply'
    assert read_ply(d2s_ply).tobytes() == r['data_down'].cpu().numpy().tobytes()
    assert read_ply(s2d_ply).tobytes() == gold['stl'].tobytes()
    n = len(r['data_down'])
    raw = d2s_ply.read_bytes()
    cols = np.frombuffer(raw[raw.index(b'end_header\n') + 11:], [('p', '<f8', 3), ('c', 'u1', 3)], count=n)['c']
    d2s = np.full(n, -1.0)
    idx = torch.nonzero(r['inbound']).reshape(-1)[r['grid_inbound']][r['in_obs']].cpu().numpy()
    d2s[idx] = r['d2s'].cpu().numpy()
    assert np.all(cols[d2s < 0] == [0, 0, 255]) and np.all(cols[d2s >= 20] == [0, 255, 0])
    near = (d2s >= 0) & (d2s < 20)
    a = np.clip(d2s[near], None, 1)
    assert np.all(cols[near][:, 0] == 255) and np.all(np.abs(cols[near][:, 1].astype(float) - 255 * (1 - a)) <= 0.5 + 1e-9)
    # the path form, and a run without visualisation under a random order
    from dbw_b200 import geometry
    assert hasattr(geometry, 'load_obj')
    obj = tmp_path / 'mesh.obj'
    obj.write_text(''.join(f'v {x!r} {y!r} {z!r}\n' for x, y, z in gold['verts'].astype(np.float64).tolist())
                   + ''.join(f'f {a + 1} {b + 1} {c + 1}\n' for a, b, c in gold['faces'].tolist()))
    s2 = evaluate_mesh(str(obj), 7, str(tmp_path / 'DTU'), str(out), suffix='_obj', save_viz=False, order=gold['order'])
    assert s2 == s and (out / 'dtu_scores_obj.tsv').exists() and not (out / 'vis_007_d2s_obj.ply').exists()
    s3 = evaluate_mesh(mesh, 7, tmp_path / 'DTU', out, suffix='_rand', save_viz=False)
    assert abs(s3['avg'] - s['avg']) < 0.05 * s['avg']


def test_trainer_call_sequence_on_a_model(tmp_path):
    """Trainer.evaluate() on a DTU run: build_blocks(filter_transparent=True, as_scene=True), scale to millimetres with
    the dataset's scale_mat, Meshes, evaluate_mesh(scene, scan_id, DATASETS_PATH / 'DTU', run_dir, save_viz=False)"""
    from dbw_b200 import Meshes
    from dbw_b200.dbw import create_model
    from dbw_b200.dtu_eval import evaluate_arrays, evaluate_mesh
    from tests.test_host_logic import DTU_DEFAULT_MODEL
    torch.manual_seed(0)
    cfg = {'model': deepcopy(DTU_DEFAULT_MODEL)}
    cfg['model']['mesh']['txt_size'] = 32
    model = create_model(cfg, (64, 64)).to(DEV)
    model.eval()
    with torch.no_grad():
        model.alpha_logit.fill_(3.0)
    scale = torch.tensor([[60., 0, 0, -12.], [0, 60., 0, 7.], [0, 0, 60., 480.], [0, 0, 0, 1]], device=DEV)
    scene = model.build_blocks(filter_transparent=True, as_scene=True)
    verts, faces = scene.get_mesh_verts_faces(0)
    scene = Meshes((verts @ scale[:3, :3] + scale[:3, 3])[None], faces[None])
    v = scene.get_mesh_verts_faces(0)[0].detach().cpu().numpy()
    g = np.random.default_rng(0)
    stl = (v[g.integers(0, len(v), 4000)] + g.normal(0, 0.5, (4000, 3))).astype(np.float32).astype(np.float64)
    lo, hi = v.min(0) - 5, v.max(0) + 5
    res = 2.0
    obs = np.ones(tuple(int(x) for x in np.ceil((hi - lo) / res) + 1), bool)
    plane = np.array([[0.], [0.], [1.], [-(lo[2] + 10)]])
    _dtu_dir(tmp_path / 'DTU', 24, stl, obs, np.stack([lo, hi]), np.array([[res]]), plane)
    run = tmp_path / 'run'
    run.mkdir()
    s = evaluate_mesh(scene, 24, tmp_path / 'DTU', run, save_viz=False)
    assert (run / 'dtu_scores.tsv').read_text().startswith('acc\tcomp\tavg\n')
    assert all(np.isfinite(x) and x > 0 for x in s.values())
    # under an explicit order the numbers are the CPU restatement's
    vv, ff = (t.detach().cpu().numpy() for t in scene.get_mesh_verts_faces(0))
    n = len(M.data_pcd(vv, ff))
    order = g.permutation(n)
    r = evaluate_arrays(vv, ff, stl, obs, np.stack([lo, hi]), np.array([[res]]), plane, order=order)
    o = M.evaluate(vv, ff, order, obs, np.stack([lo, hi]), np.array([[res]]), plane, stl)
    assert r['data_in'].cpu().numpy().tobytes() == o['data_in'].tobytes()
    np.testing.assert_allclose([r['acc'], r['comp'], r['avg']], [o['acc'], o['comp'], o['avg']], rtol=1e-12, atol=0)
    print(f'trainer sequence: {n} sampled points, acc={s["acc"]:.4f} comp={s["comp"]:.4f}, {r["rounds"]} downsample rounds')
