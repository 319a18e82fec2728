"""CPU: the DEVICE math of the regulariser kernels (differentiable-blocksworld_b200/csrc/dbw_reg_math.cuh) compiled for the
host (tests/host_math/dbw_reg_host.cpp, g++ -ffp-contract=off) and checked against float64 torch autograd of the oracle's
statement of the reference: the as_sdf=2 superquadric implicit and its gradients with respect to the point and both
exponents -- inside, outside, at and beyond the +-5 clamp, with coordinates below the safe_pow clamp -- the TV norms and
their derivatives, at zero differences too, and the parsimony square root.  The kernels' orchestration (sampling, sums,
chain rule to the leaves) is covered by tests/test_regularisers_gpu.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import dbw_path as D

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'host_math', 'dbw_reg_host.cpp')
TV_CODES = {'l2': 0, 'l1': 1, 'l2sq': 2}
TV_NORMS = {'l1': lambda t: t.abs().sum(-1), 'l2': lambda t: D.safe_pow(t.pow(2).sum(-1), 0.5), 'l2sq': lambda t: t.pow(2).sum(-1)}


@pytest.fixture(scope='module')
def hr():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_reg_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', SRC, '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _points():
    """block-frame points: well inside, near the surface, outside, on and beyond the +-5 clamp, and with coordinates whose
    square is below the safe_pow clamp (|x| < 1e-3)"""
    g = np.random.default_rng(3)
    inside = g.uniform(-0.6, 0.6, (40, 3))
    shell = g.normal(size=(40, 3))
    shell = shell / np.linalg.norm(shell, axis=1, keepdims=True) * g.uniform(0.9, 1.1, (40, 1))
    outside = g.uniform(-4.5, 4.5, (40, 3))
    clamp = g.uniform(-1.5, 1.5, (24, 3))
    clamp[np.arange(24), np.arange(24) % 3] = np.where(np.arange(24) % 2 == 0, 1, -1) * np.where(np.arange(24) < 12, 5.0, 6.5)
    tiny = g.uniform(-0.8, 0.8, (24, 3))
    tiny[np.arange(24), np.arange(24) % 3] = g.uniform(-9e-4, 9e-4, 24)
    tiny[:6, :] = g.uniform(-5e-4, 5e-4, (6, 3))            # every coordinate below the clamp: res hits its own clamp too
    return np.concatenate([inside, shell, outside, clamp, tiny]).astype(np.float32)


@pytest.mark.parametrize('e1,e2', [(1.0, 1.0), (0.3, 1.6), (1.9, 0.25), (0.12, 0.12)])
def test_superquadric_implicit_and_its_gradients_match_torch(hr, e1, e2):
    pts = _points()
    n = len(pts)
    e = np.tile(np.float32([e1, e2]), (n, 1))
    g = np.random.default_rng(5).uniform(-1, 1, n).astype(np.float32)
    sdf, sdf_b = np.zeros(n, np.float32), np.zeros(n, np.float32)
    gl, ge = np.zeros((n, 3), np.float32), np.zeros((n, 2), np.float32)
    hr.hr_sq_implicit(n, _p(pts), _p(e), _p(g), _p(sdf), _p(sdf_b), _p(gl), _p(ge))
    assert np.array_equal(sdf, sdf_b)

    P = torch.from_numpy(pts).double().requires_grad_(True)
    E1 = torch.full((n,), float(np.float32(e1)), dtype=torch.float64, requires_grad=True)
    E2 = torch.full((n,), float(np.float32(e2)), dtype=torch.float64, requires_grad=True)
    ref = D.implicit_sq(P, E1, E2)
    ref.backward(torch.from_numpy(g).double())
    # sdf: powf with exponents up to 1/0.12 in float32 against float64
    ok = np.isfinite(ref.detach().numpy())
    np.testing.assert_allclose(sdf[ok], ref.detach().numpy()[ok], rtol=5e-5, atol=1e-5)
    assert np.array_equal(np.isfinite(sdf), ok)
    # point gradient: exactly zero beyond the +-5 clamp and for coordinates below the safe_pow clamp, like torch
    gref = P.grad.numpy()
    assert (gl[gref == 0] == 0).all()
    assert (np.abs(gref[(gl == 0) & (gref != 0)]) < 1e-20).all()        # elsewhere only float32 underflow gives a zero
    fin = np.isfinite(gref).all(1) & np.isfinite(gl).all(1)
    scale = np.abs(gref[fin]).max(1, keepdims=True) + 1e-6
    np.testing.assert_allclose(gl[fin] / scale, gref[fin] / scale, atol=2e-4)
    # exponent gradients, per point
    for k, ref_e in enumerate((E1.grad.numpy(), E2.grad.numpy())):
        fin = np.isfinite(ref_e)
        np.testing.assert_allclose(ge[fin, k], ref_e[fin], rtol=2e-3, atol=2e-4 * max(1.0, np.abs(ref_e[fin]).max()))


@pytest.mark.parametrize('tv_type', ['l1', 'l2', 'l2sq'])
def test_tv_norms_and_derivatives_match_torch_at_and_away_from_zero(hr, tv_type):
    g = np.random.default_rng(7)
    d = g.normal(scale=0.05, size=(64, 3)).astype(np.float32)
    d[:8] = 0.0                                              # zero differences: sign(0) = 0, safe_pow below its clamp
    d[8:16, 1] = 0.0                                         # one zero channel
    d[16:20] = 2e-4                                          # |d|^2 below 1e-6: l2 passes no gradient there
    n = len(d)
    gu = g.uniform(0.5, 2.0, n).astype(np.float32)
    out, gd = np.zeros(n, np.float32), np.zeros((n, 3), np.float32)
    hr.hr_tv_norm(TV_CODES[tv_type], n, _p(d), _p(gu), _p(out), _p(gd))
    t = torch.from_numpy(d).double().requires_grad_(True)
    ref = TV_NORMS[tv_type](t)
    ref.backward(torch.from_numpy(gu).double())
    np.testing.assert_allclose(out, ref.detach().numpy(), rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(gd, t.grad.numpy(), rtol=1e-5, atol=1e-7)
    assert np.array_equal(gd == 0, t.grad.numpy() == 0)
    if tv_type != 'l2sq':
        assert (gd[:8] == 0).all()


def test_parsimony_root_and_derivative_match_torch(hr):
    a = np.float32([0.0, 1e-7, 1e-6, 2e-6, 0.0025, 0.3, 0.5, 0.99, 1.0])
    out, grad = np.zeros_like(a), np.zeros_like(a)
    hr.hr_parsimony(len(a), _p(a), _p(out), _p(grad))
    # float32 torch: the clamp's bound is the float 1e-6 (a = 1e-6f passes its gradient), as on the product's tensors
    t = torch.from_numpy(a).requires_grad_(True)
    D.safe_pow(t, 0.5).sum().backward()
    np.testing.assert_allclose(out, D.safe_pow(t.detach(), 0.5).numpy(), rtol=1e-6)
    np.testing.assert_allclose(grad, t.grad.numpy(), rtol=1e-6)
    assert grad[2] > 0 and grad[1] == 0


def test_ctypes_mirror_has_the_layout_the_c_compiler_gives_the_header(tmp_path):
    """DbwRegularisers: size and field offsets as gcc lays the header out == the ctypes mirror in _lib.py"""
    import shutil
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    cls = _lib.DbwRegularisers
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(DbwRegularisers));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DbwRegularisers, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(exe)],
                   check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
