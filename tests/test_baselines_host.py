"""CPU: the baseline tooling without a GPU.  The float64 oracle (oracle/baselines.py) against what the reference's own
Ransac wrote (tests/golden/baselines.npz, made by tests/golden/make_baselines_golden.py); the RANSAC math of
csrc/dbw_ransac_math.cuh compiled for the host (tests/host_math/dbw_ransac_host.cpp, g++ -ffp-contract=off) against the
oracle, degenerate samples included; the superquadric meshes, the box hulls and the EMS / MBF standardisation against the
reference; and the C-ABI's refusals, which fail before anything reaches a device.  The kernels are tested in
tests/test_baselines_gpu.py."""
import ctypes
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from oracle import baselines as O
from tests.golden.make_baselines_golden import (PREPROCESS_SEED, RANSAC_CASES, cloud, degenerate_samples, digest, scan)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = np.load(os.path.join(HERE, 'golden', 'baselines.npz'))
THRESH = 1e-3


@pytest.fixture(scope='module')
def hm():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_ransac_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_ransac_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    L.hm_solve.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp]
    L.hm_solve.restype = None
    L.hm_count.argtypes = [ctypes.c_int64, vp, ctypes.c_int, vp, ctypes.c_float, vp, ctypes.c_int, vp]
    L.hm_count.restype = None
    L.hm_select.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _solve(hm, pc, idx):
    idx = np.ascontiguousarray(idx, np.int64)
    out = np.empty((len(idx), 3), np.float32)
    hm.hm_solve(_p(pc), len(idx), idx.shape[1], _p(idx), _p(out))
    return out


def _count(hm, pc, params, flag_h=-1):
    params = np.ascontiguousarray(params, np.float32)
    counts = np.empty(len(params), np.int64)
    inlier = np.zeros(len(pc), np.uint8)
    hm.hm_count(len(pc), _p(pc), len(params), _p(params), THRESH, _p(counts), flag_h, _p(inlier))
    return counts, inlier.astype(bool)


def _case(n, seed):
    k = f'ransac_{n}_{seed}__'
    return k, cloud(n, seed)


def _within_boundary(pc, abc, count, kappa):
    """count lies between the float64 inliers off the boundary and those plus every boundary point"""
    b = O.boundary(pc, abc, THRESH, kappa)
    inl = O.inliers(pc, abc, THRESH)
    inl[b] = False
    return int(inl.sum()) <= count <= int(inl.sum()) + len(b)


@pytest.mark.parametrize('n,seed', RANSAC_CASES)
def test_oracle_reproduces_the_reference_ransac(n, seed):
    k, pc = _case(n, seed)
    assert digest(pc) == GOLDEN[k + 'digest']                       # the regenerated cloud is the one the golden saw
    idx = GOLDEN[k + 'draws']
    r = O.ransac(pc, idx)
    assert r['best'] >= 0 and r['best_n'] == GOLDEN[k + 'best_n'] and r['improvements'] == GOLDEN[k + 'n_models']
    np.testing.assert_allclose(r['params'][r['best']], GOLDEN[k + 'model'], rtol=1e-5, atol=1e-6)
    # every hypothesis's count, up to the points on the threshold (the reference solves in float32: kappa widens the band)
    kappa = O.condition(pc, idx)
    for h in range(len(idx)):
        assert _within_boundary(pc, r['params'][h], GOLDEN[k + 'counts'][h], kappa[h]), h
    keep = np.unpackbits(GOLDEN[k + 'keep'])[:n].astype(bool)
    assert np.array_equal(r['keep'], keep)


@pytest.mark.parametrize('n,seed', RANSAC_CASES)
def test_host_math_solve_and_count_against_the_oracle(hm, n, seed):
    k, pc = _case(n, seed)
    idx = GOLDEN[k + 'draws']
    params64, _ = O.solve(pc, idx)
    params = _solve(hm, pc, idx)
    assert params.tobytes() == params64.astype(np.float32).tobytes()        # same operations in the same order
    counts, _ = _count(hm, pc, params)
    for h in range(len(idx)):
        assert _within_boundary(pc, params64[h], counts[h], 1.0), h
    best_n, improvements = ctypes.c_int64(), ctypes.c_int()
    best = hm.hm_select(_p(counts), len(counts), 10, ctypes.byref(best_n), ctypes.byref(improvements))
    assert (best, best_n.value, improvements.value) == O.select(counts, 10)
    assert best == O.select(GOLDEN[k + 'counts'], 10)[0]
    _, inlier = _count(hm, pc, params[best:best + 1], 0)
    assert np.array_equal(~inlier, np.unpackbits(GOLDEN[k + 'keep'])[:n].astype(bool))


def test_select_keeps_the_first_maximum_and_strict_improvements(hm):
    g = np.random.default_rng(4)
    cases = [np.array([3, 5, 5, 1, 5, 6, 6, 0, 0, 6], np.int64), np.zeros(20, np.int64),
             np.array([0, 0, 2, 2, 2, 1, 2, 2, 3, 3, 3, 3], np.int64)]
    cases += [g.integers(0, 6, 40).astype(np.int64) for _ in range(50)]
    for c in cases:
        for batch in (1, 2, 4):
            if len(c) % batch:
                continue
            best_n, improvements = ctypes.c_int64(), ctypes.c_int()
            best = hm.hm_select(_p(c), len(c), batch, ctypes.byref(best_n), ctypes.byref(improvements))
            assert (best, best_n.value, improvements.value) == O.select(c, batch)
    best_n, improvements = ctypes.c_int64(), ctypes.c_int()
    c = cases[0]
    assert hm.hm_select(_p(c), 10, 5, ctypes.byref(best_n), ctypes.byref(improvements)) == 5   # the first of round 2's 6s
    assert (best_n.value, improvements.value) == (6, 2)                                          # replaces round 1's first 5


def test_degenerate_samples(hm):
    """Singular or near-singular X^T X.  The reference's float32 inverse returns a rounding-noise plane (a few dozen inliers
    out of 1000, against 705 for the chosen plane); the float64 adjugate here gives another rounding-noise plane, or NaN when
    the determinant is exactly 0 (one point thrice), which counts no inlier.  Either way such a sample is far from winning a
    round, so the choice is unaffected."""
    n, seed = RANSAC_CASES[0]
    pc = cloud(n, seed)
    best_n = int(GOLDEN[f'ransac_{n}_{seed}__best_n'])
    for name, idx in degenerate_samples(pc):
        k = f'degenerate_{name}__'
        assert list(GOLDEN[k + 'idx']) == idx
        params64, det = O.solve(pc, np.array([idx]))
        params = _solve(hm, pc, [idx])
        assert params.tobytes() == params64.astype(np.float32).tobytes(), name
        counts, _ = _count(hm, pc, params)
        assert _within_boundary(pc, params64[0], counts[0], 1.0), name
        assert counts[0] < best_n // 10 and GOLDEN[k + 'count'] < best_n // 10, name
        if name == 'one_point':
            assert det[0] == 0 and np.isnan(params).all() and counts[0] == 0
        else:
            assert abs(det[0]) < 1e-6 * 3, name                     # near-singular: the 3x3 determinant of a unit cloud is O(1e-2)


def test_create_sq_meshes_equals_the_reference():
    from dbw_b200.baselines import create_sq_meshes
    eps = torch.from_numpy(GOLDEN['sq__eps'])
    m = create_sq_meshes(eps[:, 0:1], eps[:, 1:2], torch.from_numpy(GOLDEN['sq__S']))
    assert m.faces_padded().numpy().tolist() == GOLDEN['sq__faces'].tolist()
    assert m.verts_padded().numpy().tobytes() == GOLDEN['sq__verts'].tobytes()
    assert m.verts_padded().shape == (7, 42, 3)


def test_box_hull_faces_are_the_twelve_outward_triangles():
    from dbw_b200.baselines import box_hull_faces
    from dbw_b200.geometry import random_rotations
    g = torch.Generator().manual_seed(3)
    R = random_rotations(20, generator=g).numpy().astype(np.float64)
    rng = np.random.default_rng(3)
    unit = np.array([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)], np.float64)
    for r in R:
        half = rng.uniform(0.05, 2.0, 3)
        corners = (unit * half) @ r.T + rng.normal(0, 5, 3)
        corners = corners[rng.permutation(8)]
        f = box_hull_faces(corners)
        assert f.shape == (12, 3) and sorted(set(f.ravel())) == list(range(8))
        a, b, c = corners[f[:, 0]], corners[f[:, 1]], corners[f[:, 2]]
        n = np.cross(b - a, c - a)
        area = 0.5 * np.linalg.norm(n, axis=1).sum()
        assert abs(area - 8 * (half[0] * half[1] + half[1] * half[2] + half[0] * half[2])) < 1e-6 * area
        assert ((n * ((a + b + c) / 3 - corners.mean(0))).sum(1) > 0).all()
        # each edge of the closed surface is used once in each direction
        edges = {(int(f[t, i]), int(f[t, (i + 1) % 3])) for t in range(12) for i in range(3)}
        assert len(edges) == 36 and all((j, i) in edges for i, j in edges)


@pytest.mark.parametrize('name', ['ems', 'mbf'])
def test_preprocess_standardisation_equals_the_reference_on_the_cpu(tmp_path, name):
    """without the ground filter every stage is a torch op, so a CPU run is the reference's bit for bit"""
    from dbw_b200.baselines import DTU3DPreprocess
    from dbw_b200.dtu_eval import read_ply
    pc_gt, scale_mat = scan()
    assert digest(pc_gt) == GOLDEN['preprocess__pc_gt_digest']

    scan7 = types.SimpleNamespace(pc_gt=torch.from_numpy(pc_gt), scale_mat=torch.from_numpy(scale_mat))
    DTU3DPreprocess(tmp_path, name, device='cpu').run({'scan7': scan7}, seed=PREPROCESS_SEED)
    k = f'preprocess_{name}_0__'
    assert np.load(tmp_path / 'scan7_scale.npy').tobytes() == GOLDEN[k + 'scale'].tobytes()
    ply = read_ply(tmp_path / 'scan7.ply')
    assert ply.dtype == np.float64 and np.array_equal(ply, GOLDEN[k + 'ply'].astype(np.float64))


def test_seeded_runs_restore_the_global_rng(tmp_path):
    from dbw_b200.baselines import DTU3DPreprocess
    pc_gt, scale_mat = scan(n=500)

    scan1 = types.SimpleNamespace(pc_gt=torch.from_numpy(pc_gt), scale_mat=torch.from_numpy(scale_mat))
    torch.manual_seed(0)
    before = torch.get_rng_state()
    DTU3DPreprocess(tmp_path, 'ems', device='cpu').run({'scan1': scan1}, seed=5)
    assert torch.equal(torch.get_rng_state(), before)


def test_c_abi_refusals_and_result_layout(tmp_path):
    from dbw_b200 import _lib
    from dbw_b200.baselines import ransac_ground_mask, DTU3DPreprocess
    L = _lib.lib()
    nbytes = ctypes.c_size_t(0)
    assert L.dbw_ransac_workspace_bytes(2500000, 100, ctypes.byref(nbytes)) == 0
    tiles = (2500000 + 1023) // 1024
    assert nbytes.value == 256 + 100 * tiles * 4
    assert L.dbw_ransac_workspace_bytes(1, 1, ctypes.byref(nbytes)) == 0 and nbytes.value == 256 + 16
    for n, h in ((0, 100), (2 ** 31, 100), (10, 0), (10, _lib.RANSAC_MAX_HYPOTHESES + 1)):
        assert L.dbw_ransac_workspace_bytes(n, h, ctypes.byref(nbytes)) != 0
    fake = ctypes.c_void_p(256)                                            # never dereferenced: the checks fail first
    assert L.dbw_ransac_fit(10, fake, 10, 2, fake, fake, None) != 0
    assert b'out of range' in L.dbw_last_error()
    assert L.dbw_ransac_fit(10, fake, 10, _lib.RANSAC_MAX_SAMPLE + 1, fake, fake, None) != 0
    assert L.dbw_ransac_count(10, fake, 10, fake, 1e-3, fake, fake, 0, None) != 0
    assert b'workspace too small' in L.dbw_last_error()
    assert L.dbw_ransac_select(100, 7, fake, fake, fake, None) != 0
    assert L.dbw_ransac_filter(10, fake, None, 1e-3, None, None, fake, fake, 1 << 20, None) != 0
    assert L.dbw_ransac_filter(10, fake, fake, 1e-3, None, None, fake, fake, 16, None) != 0
    # the ctypes mirror has the layout gcc gives the header
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "dbw_render.h"\nint main(void) { printf("%zu %zu %zu %zu %d %d\\n", '
                   'sizeof(DbwRansacResult), offsetof(DbwRansacResult, hypothesis), offsetof(DbwRansacResult, n_inliers), '
                   'offsetof(DbwRansacResult, n_improvements), DBW_RANSAC_MAX_HYPOTHESES, DBW_RANSAC_MAX_SAMPLE); return 0; }\n')
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else 'gcc'
    subprocess.run([gcc, '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(tmp_path / 'layout')], check=True)
    got = subprocess.run([str(tmp_path / 'layout')], check=True, capture_output=True, text=True).stdout.split()
    R = _lib.DbwRansacResult
    assert [int(v) for v in got] == [ctypes.sizeof(R), R.hypothesis.offset, R.n_inliers.offset, R.n_improvements.offset,
                                     _lib.RANSAC_MAX_HYPOTHESES, _lib.RANSAC_MAX_SAMPLE]
    with pytest.raises(_lib.DbwError, match='CUDA tensor'):
        ransac_ground_mask(torch.zeros(10, 3))
    with pytest.raises(NotImplementedError):
        DTU3DPreprocess(tmp_path, 'cuboids')
