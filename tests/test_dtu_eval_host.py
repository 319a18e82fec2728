"""CPU: the DTU chamfer evaluation without a GPU.
  - the numpy + cKDTree restatement (oracle/mesh_eval.py) against tests/golden/dtu_eval.npz, the output of the
    reference's own evaluate_mesh (tests/golden/make_dtu_golden.py): data_pcd and data_in bit for bit and in order, the
    observation and plane masks exactly, the scores to 1e-12;
  - the sampling math of the kernels (csrc/dbw_eval_math.cuh compiled for the host) bit for bit against the reference's
    numpy formulation, over random, thin, huge and degenerate triangles;
  - the PLY reader / writer of dbw_b200.dtu_eval, and the C layout of DbwEvalGrid."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import mesh_eval as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, 'golden', 'dtu_eval.npz')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def test_oracle_reproduces_the_reference_evaluation(gold):
    r = M.evaluate(gold['verts'], gold['faces'], gold['order'], gold['obs_mask'], gold['bb'], gold['res'], gold['plane'], gold['stl'])
    assert r['shuffled'].tobytes() == gold['shuffled'].tobytes()
    # before the shuffle data_pcd is [vertices; samples]: the referenced vertices lead
    n_ref = len(np.unique(gold['faces']))
    assert len(gold['verts']) == n_ref + 1                     # the scene has one unreferenced vertex
    assert r['data_in'].tobytes() == gold['data_in'].tobytes()
    assert r['data_in_obs'].tobytes() == gold['data_in'][gold['data_in_obs_mask']].tobytes()
    assert r['stl_above'].tobytes() == gold['stl'][gold['stl_above_mask']].tobytes()
    np.testing.assert_allclose([r['acc'], r['comp'], r['avg']], gold['scores'], rtol=1e-12, atol=0)
    tsv = str(gold['tsv'])
    assert tsv.startswith('acc\tcomp\tavg\n') and not tsv.endswith('\n')
    np.testing.assert_allclose([float(x) for x in M.scores_tsv(r['acc'], r['comp'], r['avg']).split('\n')[1].split('\t')],
                               [float(x) for x in tsv.split('\n')[1].split('\t')], rtol=1e-12, atol=0)


def test_golden_scene_covers_the_edge_cases(gold):
    V, F = gold['verts'].astype(np.float64), gold['faces']
    v1, v2, n1, n2, ok = M.triangle_lattice(V[F])
    assert (~ok).sum() >= 1                                    # a zero-area triangle
    assert np.any(ok & (n1 == 0))                              # a triangle with n1 = 0
    assert (n1 * n2)[ok].max() > 5000                          # one large triangle
    r = M.evaluate(gold['verts'], gold['faces'], gold['order'], gold['obs_mask'], gold['bb'], gold['res'], gold['plane'], gold['stl'])
    assert len(r['data_in']) < len(r['data_down'])             # points outside BB +- PATCH
    assert len(r['data_in_obs']) < len(r['data_in'])           # outside the mask grid / unobserved
    assert len(r['stl_above']) < len(gold['stl'])              # STL points below the plane
    assert np.isinf(r['d2s']).any() and np.isinf(r['s2d']).any()   # nothing within 20 mm


# ------------------------------------------------------------------------------------------------ host-compiled sampling math
@pytest.fixture(scope='module')
def he():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_eval_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_eval_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.he_sample.restype = ctypes.c_int64
    L.he_sample.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    return L


def _numpy_reference_samples(tri_vert):
    """the reference's formulation (np.linalg.norm, np.cross, np.mgrid), for comparison"""
    v1 = tri_vert[:, 1] - tri_vert[:, 0]
    v2 = tri_vert[:, 2] - tri_vert[:, 0]
    l1 = np.linalg.norm(v1, axis=-1, keepdims=True)
    l2 = np.linalg.norm(v2, axis=-1, keepdims=True)
    area2 = np.linalg.norm(np.cross(v1, v2), axis=-1, keepdims=True)
    nz = (area2 > 0)[:, 0]
    l1, l2, area2, v1, v2, tri_vert = [a[nz] for a in [l1, l2, area2, v1, v2, tri_vert]]
    thr = 0.2 * np.sqrt(l1 * l2 / area2)
    n1, n2 = np.floor(l1 / thr), np.floor(l2 / thr)
    out = []
    for i in range(len(n1)):
        c = np.mgrid[:n1[i, 0] + 1, :n2[i, 0] + 1]
        c += 0.5
        c[0] /= max(n1[i, 0], 1e-7)
        c[1] /= max(n2[i, 0], 1e-7)
        c = np.transpose(c, (1, 2, 0))
        k = c[c.sum(axis=-1) < 1]
        out.append(v1[i:i + 1] * k[:, :1] + v2[i:i + 1] * k[:, 1:] + tri_vert[i:i + 1, 0])
    return np.concatenate(out) if out else np.zeros((0, 3)), n1[:, 0], n2[:, 0], nz


def _random_triangles(seed):
    g = np.random.default_rng(seed)
    tris = []
    for k in range(60):
        c = g.uniform(-300, 300, 3)
        s = [0.05, 0.6, 3.0, 12.0][k % 4]
        t = c + g.normal(0, s, (3, 3))
        if k % 7 == 3:                                        # thin: third vertex almost on the first edge
            t[2] = t[0] + (t[1] - t[0]) * g.uniform(0.2, 0.8) + g.normal(0, 1e-3, 3)
        if k % 11 == 5:                                       # degenerate: repeated vertex
            t[2] = t[0]
        tris.append(t)
    tris.append(np.array([[0., 0., 0.], [0.05, 0.01, 0.], [0.3, 6.0, 0.]]))           # n1 = 0
    tris.append(np.array([[-40., -30., 5.], [45., -20., 9.], [-5., 50., -3.]]))       # huge: ~8e4 samples
    return np.asarray(tris, np.float32).astype(np.float64)   # float32 mesh vertices, as the evaluation receives them


@pytest.mark.parametrize('seed', [0, 1])
def test_host_compiled_sampling_matches_numpy_bit_for_bit(he, seed):
    tv = np.ascontiguousarray(_random_triangles(seed))
    F = len(tv)
    ref, n1, n2, nz = _numpy_reference_samples(tv.copy())
    rec, rows = np.zeros((F, 12)), np.zeros(F, np.int64)
    out = np.zeros((len(ref) + 16, 3))
    n = he.he_sample(tv.ctypes.data, F, rec.ctypes.data, rows.ctypes.data, out.ctypes.data, len(out))
    assert n == len(ref) and len(ref) > 80000
    assert out[:n].tobytes() == ref.tobytes()
    assert rec[nz, 9].tobytes() == n1.tobytes() and rec[nz, 10].tobytes() == n2.tobytes()
    assert np.all(rows[~nz] == 0)
    # and the oracle's restatement agrees
    assert M.sample_mesh(tv.reshape(-1, 3), np.arange(3 * F).reshape(F, 3)).tobytes() == ref.tobytes()


# ------------------------------------------------------------------------------------------------ PLY, C layout
@pytest.mark.parametrize('binary', [True, False])
def test_ply_round_trip(tmp_path, binary):
    from dbw_b200.dtu_eval import read_ply, write_ply
    g = np.random.default_rng(3)
    pts = g.normal(0, 100, (257, 3))
    col = g.uniform(0, 1, (257, 3))
    p = tmp_path / 'a.ply'
    write_ply(p, pts, col, binary=binary)
    got = read_ply(p)
    assert got.dtype == np.float64 and got.tobytes() == pts.tobytes()
    head = open(p, 'rb').read(300)
    assert b'property uchar red' in head and (b'binary_little_endian' in head) == binary


def test_ply_reader_skips_other_properties_and_reads_float(tmp_path):
    from dbw_b200.dtu_eval import read_ply
    pts = np.random.default_rng(4).normal(0, 10, (9, 3)).astype(np.float32)
    arr = np.zeros(9, [('nx', '<f4'), ('x', '<f4'), ('y', '<f4'), ('z', '<f4'), ('quality', 'u1')])
    arr['x'], arr['y'], arr['z'] = pts.T
    hdr = ('ply\nformat binary_little_endian 1.0\ncomment made by a test\nelement vertex 9\nproperty float nx\nproperty float x\n'
           'property float y\nproperty float z\nproperty uchar quality\nelement face 0\nproperty list uchar int vertex_indices\n'
           'end_header\n')
    p = tmp_path / 'b.ply'
    p.write_bytes(hdr.encode() + arr.tobytes())
    assert read_ply(p).tobytes() == pts.astype(np.float64).tobytes()
    q = tmp_path / 'c.ply'
    q.write_text('ply\nformat ascii 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\n'
                 'property uchar red\nend_header\n1 2 3 255\n4.5 -5 6e2 0\n')
    assert read_ply(q).tolist() == [[1, 2, 3], [4.5, -5, 600]]


def test_eval_grid_layout_and_argument_checks_without_a_gpu(tmp_path):
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is not None:
        cls = _lib.DbwEvalGrid
        lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
                 '  printf("size %zu\\n", sizeof(DbwEvalGrid));']
        lines += [f'  printf("{f} %zu\\n", offsetof(DbwEvalGrid, {f}));' for f, _ in cls._fields_]
        lines += ['  return 0;', '}']
        (tmp_path / 'l.c').write_text('\n'.join(lines))
        subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'l.c'), '-o',
                        str(tmp_path / 'l')], check=True)
        got = dict(l.split() for l in subprocess.run([str(tmp_path / 'l')], capture_output=True, text=True, check=True).stdout.splitlines())
        assert int(got['size']) == ctypes.sizeof(cls) == 64
        for f, _ in cls._fields_:
            assert int(got[f]) == getattr(cls, f).offset, f
    L = _lib.lib()
    g = _lib.DbwEvalGrid()
    g.cell, g.block = 1.0, 3
    g.dims[:] = [4, 4, 4]
    assert L.dbw_eval_nn_distance(None, 5, None, None, ctypes.byref(g), 20.0, None, None) != 0
    assert b'bad grid' in L.dbw_last_error()
    assert L.dbw_eval_sample_setup(None, None, 3, None, None, None) != 0 and b'null pointer' in L.dbw_last_error()
    rounds = ctypes.c_int32(0)
    assert L.dbw_eval_radius_downsample(*([None] * 5), 10, 0.2, 0, None, ctypes.byref(rounds), None, 0, None) != 0
    # empty inputs are no-ops
    assert L.dbw_eval_sample_setup(None, None, 0, None, None, None) == 0
    assert L.dbw_eval_nn_distance(None, 0, None, None, ctypes.byref(g), 20.0, None, None) == 0
