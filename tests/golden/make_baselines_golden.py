"""Generates tests/golden/baselines.npz: the reference's OWN baseline preprocessing code of a checkout of
monniert/differentiable-blocksworld named by DBW_REFERENCE, extracted with `ast` by tests/_refextract.py and run on the CPU:
  - Ransac.fit with LSLinearRegressor (src/utils/ransac.py) on synthetic clouds (a tilted ground plane plus objects, 10^3 to
    10^5 points, several seeds): every round's draws, every hypothesis's parameters and count (the reference's own predict
    and predicate), the chosen model and the cloud the preprocessing keeps (dtu_3d_process.py:36-41), as a packed mask;
  - LSLinearRegressor.fit on degenerate samples (collinear points, a repeated index, one point three times);
  - create_sq_meshes (src/utils/superquadric.py) on the vertices of dbw_b200.geometry.ico_sphere(1);
  - DTU3DPreprocess.run (src/dtu_3d_process.py) on a synthetic scan, EMS and MBF, with and without the ground filter: the
    saved {tag}_scale.npy and the cloud handed to save_ply.
The clouds themselves are not stored: `cloud(n, seed)` regenerates them (numpy's PCG64 stream is fixed); their bytes are
pinned by a digest.  Only data is stored.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_baselines_golden.py
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

RANSAC_CASES = [(1000, 3), (1000, 11), (10000, 0), (10000, 5), (100000, 1), (100000, 2)]      # (points, seed)
PREPROCESS_POINTS, PREPROCESS_SEED = 6000, 1234
SQ_SEED = 9


def cloud(n, seed):
    """(n, 3) float32: 60% of the points on the plane z = 0.05 + 0.1 x - 0.2 y (noise 0.004), the rest on three boxes and a
    sphere standing on it, in the unit-sphere range of a standardised DTU scan"""
    g = np.random.default_rng(seed)
    n_ground = int(0.6 * n)
    xy = g.uniform(-0.9, 0.9, (n_ground, 2))
    ground = np.c_[xy, 0.05 + 0.1 * xy[:, 0] - 0.2 * xy[:, 1] + g.normal(0, 0.004, n_ground)]
    parts = [ground]
    rest = n - n_ground
    for k, (cx, cy, s) in enumerate([(-0.4, -0.3, 0.2), (0.3, 0.2, 0.15), (0.0, 0.5, 0.1)]):
        m = rest // 4
        u = g.uniform(-1, 1, (m, 3))
        face = g.integers(0, 3, m)
        u[np.arange(m), face] = np.sign(u[np.arange(m), face])        # on the box's surface
        base = 0.05 + 0.1 * cx - 0.2 * cy
        parts.append(np.c_[cx + s * u[:, 0], cy + s * u[:, 1], base + s * (1 + u[:, 2])])
    m = n - sum(len(p) for p in parts)
    v = g.normal(0, 1, (m, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    parts.append(np.c_[0.5 + 0.15 * v[:, 0], -0.5 + 0.15 * v[:, 1], 0.3 + 0.15 * v[:, 2]])
    pc = np.concatenate(parts).astype(np.float32)
    return pc[g.permutation(n)]


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()[:8], np.int64)[0]


def scan(seed=PREPROCESS_SEED, n=PREPROCESS_POINTS):
    """a synthetic DTU scan: pc_gt in the standardised space and a float32 scale matrix (scale and offset, as cameras.npz)"""
    scale_mat = np.eye(4, dtype=np.float32)
    scale_mat[:3, :3] *= 212.5
    scale_mat[:3, 3] = [-11.25, 37.5, 640.0]
    return cloud(n, seed), scale_mat


def degenerate_samples(pc):
    """(name, (3,) indices) of samples whose X^T X is singular or nearly: collinear xy, a repeated index, one point thrice"""
    a, b = pc[0], pc[1]
    d = b[:2] - a[:2]
    # the point of the cloud closest to the line through a and b in xy (not a or b)
    dist = np.abs((pc[:, 0] - a[0]) * d[1] - (pc[:, 1] - a[1]) * d[0])
    dist[:2] = np.inf
    c = int(np.argmin(dist))
    return [('collinear', [0, 1, c]), ('repeated', [0, 0, 1]), ('repeated_last', [5, 7, 7]), ('one_point', [3, 3, 3])]


class _TorchRecorder(types.ModuleType):
    """torch, with every torch.randint call recorded"""
    def __init__(self):
        super().__init__('torch')
        self.draws = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def randint(self, *a, **k):
        r = torch.randint(*a, **k)
        self.draws.append(r.clone())
        return r


def main():
    from _refextract import extract, extract_method, have_reference
    if not have_reference():
        sys.exit('set DBW_REFERENCE to a checkout of monniert/differentiable-blocksworld')
    from dbw_b200 import geometry as G
    from dbw_b200.structures import Meshes

    import random
    util = extract('src/utils/__init__.py', ['use_seed'], dict(
        wraps=__import__('functools').wraps, rand_get_state=random.getstate, rand_set_state=random.setstate, rand_seed=random.seed, np_get_state=np.random.get_state,
        np_set_state=np.random.set_state, np_seed=np.random.seed, torch_get_state=torch.get_rng_state,
        torch_set_state=torch.set_rng_state, torch_seed=torch.manual_seed))
    rec = _TorchRecorder()
    rs = extract('src/utils/ransac.py', ['LSLinearRegressor', 'Ransac'],
                 {'torch': rec, 'use_seed': util['use_seed'], 'print_log': lambda *a, **k: None})
    Ransac, LS = rs['Ransac'], rs['LSLinearRegressor']
    out = {}

    for n, seed in RANSAC_CASES:
        k = f'ransac_{n}_{seed}__'
        pc_np = cloud(n, seed)
        pc = torch.from_numpy(pc_np)
        rec.draws = []
        ransac = Ransac()
        X, y = pc[:, :2], pc[:, 2:3]
        ransac.fit(X, y, seed=seed)
        B, P = ransac.batch_size, ransac.n_points
        params, counts = [], []
        for idxs in rec.draws:                   # replay each round's fit and count with the reference's own code
            m = LS().fit(X[idxs].view(B, P, -1), y[idxs].view(B, P, -1))
            diff = (y[None].expand(B, -1, -1) - m.predict(X[None].expand(B, -1, -1))).flatten(1)
            counts.append((diff.pow(2) < ransac.thresh).sum(1))
            params.append(m.params[..., 0])
        model = ransac.best_models[-1]
        is_inlier = (model.predict(pc[:, :2]) - pc[:, 2:]).pow(2) < ransac.thresh
        keep = ~is_inlier[:, 0]
        out[k + 'digest'] = digest(pc_np)
        out[k + 'draws'] = torch.stack(rec.draws).numpy().reshape(-1, P)
        out[k + 'params'] = torch.cat(params).numpy()
        out[k + 'counts'] = torch.cat(counts).numpy().astype(np.int64)
        out[k + 'best_n'] = np.int64(ransac.best_n)
        out[k + 'n_models'] = np.int64(len(ransac.best_models))
        out[k + 'model'] = model.params[:, 0].numpy()
        out[k + 'keep'] = np.packbits(keep.numpy())
        print(n, seed, 'best_n', ransac.best_n, 'models', len(ransac.best_models), 'kept', int(keep.sum()))

    pc = torch.from_numpy(cloud(RANSAC_CASES[0][0], RANSAC_CASES[0][1]))
    for name, idx in degenerate_samples(pc.numpy()):
        k = f'degenerate_{name}__'
        out[k + 'idx'] = np.array(idx, np.int64)
        i = torch.tensor(idx)
        try:
            m = LS().fit(pc[i, :2][None], pc[i, 2:3][None])
            diff = (pc[None, :, 2:3] - m.predict(pc[None, :, :2])).flatten(1)
            out[k + 'params'] = m.params[0, :, 0].numpy()
            out[k + 'count'] = np.int64((diff.pow(2) < 0.001).sum())
        except RuntimeError as e:                # torch.linalg's error for an exactly singular float32 matrix
            out[k + 'raised'] = np.array(str(e).splitlines()[0])
        print(name, {kk[len(k):]: v for kk, v in out.items() if kk.startswith(k)})

    # create_sq_meshes on PyTorch3D's level-1 icosphere (dbw_b200.geometry.ico_sphere restates it)
    mesh_ns = {'get_icosphere': lambda level=3: Meshes(*(t[None] for t in G.ico_sphere(level))), 'Meshes': Meshes}
    sq = extract('src/utils/pytorch.py', ['signed_pow'])
    sq = extract('src/utils/superquadric.py', ['parametric_sq', 'create_sq_meshes'], dict(mesh_ns, signed_pow=sq['signed_pow']))
    g = np.random.default_rng(SQ_SEED)
    eps = torch.from_numpy(g.uniform(0.1, 1.9, (7, 2)).astype(np.float32))
    eps[0] = torch.tensor([1.0, 1.0])
    eps[1] = torch.tensor([0.1, 1.9])
    S = torch.from_numpy(g.uniform(0.05, 2.0, (7, 3)).astype(np.float32))
    m = sq['create_sq_meshes'](eps[:, 0:1], eps[:, 1:2], S, level=3)
    out['sq__eps'], out['sq__S'] = eps.numpy(), S.numpy()
    out['sq__verts'], out['sq__faces'] = m.verts_padded().numpy(), m.faces_padded().numpy()

    # DTU3DPreprocess.run on one synthetic scan
    pc_gt, scale_mat = scan()
    saved = {}

    class Dataset:
        def __init__(self, **kw):
            self.pc_gt, self.scale_mat = torch.from_numpy(pc_gt), torch.from_numpy(scale_mat)

    npns = types.SimpleNamespace(save=lambda path, a: saved.__setitem__(('scale', os.path.basename(str(path))), a))
    pp = extract('src/dtu_3d_process.py', ['N_POINTS_EMS_FIT', 'N_POINTS_MBF_FIT'])
    run = extract_method('src/dtu_3d_process.py', 'DTU3DPreprocess', 'run', dict(
        np=npns, torch=torch, EVAL_SCAN_IDS=['scan7'], get_dataset=lambda name: Dataset, Ransac=rs['Ransac'],
        print_log=lambda *a, **k: None, N_POINTS_EMS_FIT=pp['N_POINTS_EMS_FIT'], N_POINTS_MBF_FIT=pp['N_POINTS_MBF_FIT'],
        save_ply=lambda path, verts: saved.__setitem__(('ply', os.path.basename(str(path))), verts.numpy())))
    out['preprocess__pc_gt_digest'] = digest(pc_gt)
    out['preprocess__scale_mat'] = scale_mat
    for name in ('ems', 'mbf'):
        for fg in (False, True):
            saved.clear()
            torch.manual_seed(PREPROCESS_SEED)                      # run(seed=...) through the reference's use_seed
            run(_Self(name, fg))
            k = f'preprocess_{name}_{int(fg)}__'
            out[k + 'scale'] = saved[('scale', 'scan7_scale.npy')]
            out[k + 'ply'] = saved[('ply', 'scan7.ply')]
            print(name, fg, out[k + 'scale'], out[k + 'ply'].shape)
    np.savez_compressed(os.path.join(HERE, 'baselines.npz'), **out)
    print('wrote', os.path.join(HERE, 'baselines.npz'))


class _Self:
    """the DTU3DPreprocess instance run() reads: run_dir / name, model_name, filter_ground, device"""
    def __init__(self, name, fg):
        self.run_dir, self.model_name, self.filter_ground, self.device = _Dir(), name, fg, torch.device('cpu')


class _Dir:
    def __truediv__(self, name):
        return name


if __name__ == '__main__':
    main()
