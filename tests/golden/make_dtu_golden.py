"""Generates tests/golden/dtu_eval.npz: the reference's OWN evaluate_mesh (src/utils/dtu_eval.py of a checkout of
monniert/differentiable-blocksworld named by DBW_REFERENCE, extracted with `ast` by tests/_refextract.py) run on a small
synthetic DTU scene.  Open3D, multiprocessing, tqdm and print_log are replaced by serial stand-ins, np.random.default_rng
by a seeded generator that records the permutation it applies, and scikit-learn's NearestNeighbors by a recorder: its
fit / kneighbors calls receive exactly the arrays the evaluation computes (the shuffled data_pcd, data_in in order,
data_in_obs, stl_above).  Only data is stored.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_dtu_golden.py
"""
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch
from scipy.io import loadmat, savemat
from scipy.spatial import cKDTree

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from _refextract import extract, have_reference  # noqa: E402

SEED = 2024


def _ico(level=1):
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7],
         [9, 8, 1]]
    v = list(v / np.linalg.norm(v, axis=1, keepdims=True))
    for _ in range(level):
        mid, nf = {}, []
        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.asarray(v), np.asarray(f, np.int64)


def dtu_case(seed=SEED):
    """(verts float32, faces int64, stl fp64, ObsMask, BB, Res, P) of a small synthetic scene in millimetres"""
    g = np.random.default_rng(seed)
    iv, iff = _ico(1)
    verts, faces = [], []

    def add(v, f):
        faces.append(f + sum(len(x) for x in verts))
        verts.append(v)
    for c, r in [((0.3, -1.7, 2.2), 4.1), ((31.7, 8.9, -3.3), 2.6), ((88.4, 4.1, 1.7), 3.3), ((260.0, 3.0, 0.0), 2.3)]:
        Q = np.linalg.qr(g.normal(size=(3, 3)))[0]
        add(iv @ Q * r + np.asarray(c), iff)
    # one large triangle, a zero-area triangle (repeated vertex), a triangle with n1 = 0 (0.05 mm edge against 6 mm),
    # and an unreferenced vertex
    add(np.array([[-12.1, -9.3, -6.2], [14.7, -7.9, -5.1], [-3.3, 17.2, -7.4]]), np.array([[0, 1, 2]]))
    add(np.array([[5.1, 5.2, 5.3], [6.4, 4.9, 5.5]]), np.array([[0, 1, 0]]))
    add(np.array([[-8.0, 9.0, 3.0], [-7.961, 9.031, 3.0], [-8.0 + 3.6, 9.0 - 4.8, 3.0]]), np.array([[0, 1, 2]]))
    verts.append(np.array([[1.0, 2.0, 3.0]]))
    V = np.concatenate(verts).astype(np.float32)
    F = np.concatenate(faces).astype(np.int64)
    # STL: noisy samples around the first sphere and the big triangle, a cluster > 20 mm from every data point, and a
    # cluster below the plane z = -15
    s1 = g.normal(size=(1500, 3))
    s1 = s1 / np.linalg.norm(s1, axis=1, keepdims=True) * (4.1 + g.normal(0, 0.15, (1500, 1))) + np.array([0.3, -1.7, 2.2])
    a, b = g.uniform(size=(1200, 1)), g.uniform(size=(1200, 1))
    a, b = np.where(a + b > 1, 1 - a, a), np.where(a + b > 1, 1 - b, b)
    tv = V[F[4 * 80]].astype(np.float64)          # the large triangle
    s2 = tv[0] + a * (tv[1] - tv[0]) + b * (tv[2] - tv[0]) + g.normal(0, 0.2, (1200, 3))
    s3 = g.normal(0, 1.5, (300, 3)) + np.array([0.0, 60.0, 5.0])
    s4 = g.normal(0, 1.5, (300, 3)) + np.array([2.0, 0.0, -22.0])
    stl = np.concatenate([s1, s2, s3, s4]).astype(np.float32).astype(np.float64)
    BB = np.array([[-25.31, -20.77, -18.13], [45.23, 30.91, 22.47]])
    Res = np.array([[4.0]])
    shape = tuple(int(x) for x in np.ceil((BB[1] - BB[0]) / 4.0) + 1)
    ObsMask = g.uniform(size=shape) < 0.85
    P = np.array([[0.05], [-0.03], [1.0], [15.0]])
    return V, F, stl, ObsMask, BB, Res, P


class _Recorder:
    """NearestNeighbors stand-in: the real scikit-learn estimator, recording what it is given"""
    log = []

    def __init__(self, *a, **k):
        import sklearn.neighbors as skln
        self.nn = skln.NearestNeighbors(*a, **k)

    def fit(self, X):
        _Recorder.log.append(('fit', np.array(X)))
        self.nn.fit(X)
        return self

    def radius_neighbors(self, X, **k):
        return self.nn.radius_neighbors(X, **k)

    def kneighbors(self, X, **k):
        d, i = self.nn.kneighbors(X, **k)
        _Recorder.log.append(('kneighbors', np.array(X), d[:, 0].copy()))
        return d, i


class _TriangleMesh:
    def __init__(self, verts, faces):
        self.vertices, self.triangles = np.asarray(verts, np.float64), np.asarray(faces, np.int64)

    def remove_unreferenced_vertices(self):              # survivors keep their order
        used = np.zeros(len(self.vertices), bool)
        used[self.triangles.reshape(-1)] = True
        remap = np.cumsum(used) - 1
        self.vertices, self.triangles = self.vertices[used], remap[self.triangles]


class _Pool:
    def __enter__(self): return self
    def __exit__(self, *a): return False
    def map(self, fn, it, chunksize=None): return [fn(x) for x in it]


def _subsequence_mask(full, sub):
    m, k = np.zeros(len(full), bool), 0
    for i in range(len(full)):
        if k < len(sub) and np.array_equal(full[i], sub[k]):
            m[i], k = True, k + 1
    assert k == len(sub) and np.array_equal(full[m], sub)
    return m


def ref_dtu_eval():
    assert have_reference()
    from dbw_b200.structures import Meshes
    V, F, stl, ObsMask, BB, Res, P = dtu_case()
    perms = []

    class _Rng:
        def __init__(self, *a):
            self.g = np.random.Generator(np.random.PCG64(SEED))

        def shuffle(self, x, axis=0):
            assert axis == 0
            p = self.g.permutation(len(x))
            perms.append(p)
            x[...] = x[p]
    o3d = SimpleNamespace(
        geometry=SimpleNamespace(TriangleMesh=_TriangleMesh),
        utility=SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64), Vector3iVector=lambda a: np.asarray(a, np.int64)),
        io=SimpleNamespace(read_point_cloud=lambda path: SimpleNamespace(points=stl)))
    tqdm = lambda total=None: SimpleNamespace(set_description=lambda s: None, update=lambda n: None, close=lambda: None)
    class _Random:
        default_rng = _Rng

        def __getattr__(self, k): return getattr(np.random, k)

    class _Np:                                          # numpy, with np.random.default_rng seeded (for this function only)
        random = _Random()

        def __getattr__(self, k): return getattr(np, k)
    ns = extract('src/utils/dtu_eval.py', ['MAX_DIST', 'PATCH', 'DOWNSAMPLE_DENSITY', 'sample_single_tri', 'evaluate_mesh'],
                 {'np': _Np(), 'o3d': o3d, 'mp': SimpleNamespace(freeze_support=lambda: None, Pool=_Pool), 'tqdm': tqdm,
                  'P3DMeshes': Meshes, 'loadmat': loadmat, 'skln': SimpleNamespace(NearestNeighbors=_Recorder),
                  'print_log': lambda s: print(s), 'Path': __import__('pathlib').Path})
    _Recorder.log = []
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, 'ObsMask'))
        savemat(os.path.join(d, 'ObsMask', 'ObsMask7_10.mat'), {'ObsMask': ObsMask, 'BB': BB, 'Res': Res})
        savemat(os.path.join(d, 'ObsMask', 'Plane7.mat'), {'P': P})
        ns['evaluate_mesh'](Meshes(torch.from_numpy(V)[None], torch.from_numpy(F)[None]), 7, d, d, save_viz=False)
        tsv = open(os.path.join(d, 'dtu_scores.tsv')).read()
    log = _Recorder.log
    assert [e[0] for e in log] == ['fit', 'fit', 'kneighbors', 'fit', 'kneighbors'], [e[0] for e in log]
    shuffled, data_in, data_in_obs, stl_above = log[0][1], log[3][1], log[2][1], log[4][1]
    d2s, s2d = log[2][2], log[4][2]
    # no decision may hinge on the last bits: no pair within 1e-9 of the downsample radius, no NN distance within 1e-9
    # of the cutoff
    t = cKDTree(shuffled)
    assert len(t.query_pairs(0.2 + 1e-9)) == len(t.query_pairs(0.2 - 1e-9))
    assert not np.any(np.abs(d2s - 20) < 1e-9) and not np.any(np.abs(s2d - 20) < 1e-9)
    assert np.any(d2s >= 20) and np.any(s2d >= 20) and len(stl_above) < len(stl)
    acc, comp, avg = (float(x) for x in tsv.split('\n')[1].split('\t'))
    # data_in_obs and stl_above are stored as masks over data_in and stl (subsequences: half the bytes)
    in_obs, above = _subsequence_mask(data_in, data_in_obs), _subsequence_mask(stl, stl_above)
    return dict(verts=V, faces=F, stl=stl, obs_mask=ObsMask, bb=BB, res=Res, plane=P, order=perms[0].astype(np.int64),
                shuffled=shuffled, data_in=data_in, data_in_obs_mask=in_obs, stl_above_mask=above,
                scores=np.array([acc, comp, avg]), tsv=np.array(tsv))


if __name__ == '__main__':
    if not have_reference():
        sys.exit('DBW_REFERENCE names no reference checkout')
    out = ref_dtu_eval()
    np.savez_compressed(os.path.join(HERE, 'dtu_eval.npz'), **out)
    print('wrote dtu_eval.npz', {k: getattr(v, 'shape', None) for k, v in out.items()}, os.path.getsize(os.path.join(HERE, 'dtu_eval.npz')))
