"""CPU: the gradient of the camera poses.

1. The projection backward of csrc/dbw_camera.cuh -- the one Jacobian project_verts_backward_kernel (vertex gradient) and
   camera_grad_kernel (pose gradient) both inline -- compiled for the host (tests/host_math/dbw_camera_host.cpp) and driven
   per (view, vertex) as the kernels drive it, against torch autograd of oracle.pt3d.world_to_ndc in float64: random poses,
   plus a signed-permutation view whose depths are exact and include 0, the |z| < eps clamp and negative z.
2. The float64 oracle's own d/dR and d/dT (autograd through world_to_ndc and the rasterizer) against central differences,
   so that the GPU tests can take it as the reference."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import dbw_path as D
from oracle import pt3d

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'host_math', 'dbw_camera_host.cpp')
EPS32 = float(np.float32(1e-8))          # proj_eps as the kernels see it (a float)


@pytest.fixture(scope='module')
def hc():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_camera_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', SRC, '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rotation(g):
    q, r = np.linalg.qr(g.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))[None]
    return q if np.linalg.det(q) > 0 else -q


def _inputs(seed):
    """verts (V,3), R (B,3,3), T (B,3), g_ndc (B,V,3) float32.  Views 0-2: random rotations, the points 2.5-5.5 in front.
    View 3: R a signed permutation with T = 0, so view z = -Z exactly; the first vertices get Z = 0, +-5e-9 (inside the
    clamp), +-2e-8, +-1e-4 and +-0.3, the rest lie on both sides of the camera plane."""
    g = np.random.default_rng(seed)
    V = 48
    verts = g.uniform(-1.5, 1.5, (V, 3))
    special = [0.0, 5e-9, -5e-9, 2e-8, -2e-8, 1e-4, -1e-4, 0.3, -0.3]
    verts[:len(special), 2] = special
    R = [_rotation(g) for _ in range(3)] + [np.array([[0., 1., 0.], [1., 0., 0.], [0., 0., -1.]])]
    T = [g.uniform(-0.3, 0.3, 3) + np.array([0., 0., 4.]) for _ in range(3)] + [np.zeros(3)]
    g_ndc = g.normal(size=(4, V, 3))
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    return f32(verts), f32(R), f32(T), f32(g_ndc)


@pytest.mark.parametrize('intr', [(1.7, 2.1, 0.0, 0.0), (1.2, 0.9, 0.15, -0.25)])
@pytest.mark.parametrize('seed', [0, 1])
def test_projection_backward_matches_autograd(hc, seed, intr):
    verts, R, T, g_ndc = _inputs(seed)
    B, V = R.shape[0], verts.shape[0]
    fx, fy, px, py = intr
    gv, gR, gT = np.zeros((V, 3), np.float32), np.zeros((B, 3, 3), np.float32), np.zeros((B, 3), np.float32)
    hc.hc_project_backward(B, V, _p(verts), _p(R), _p(T), ctypes.c_float(fx), ctypes.c_float(fy), ctypes.c_float(px),
                           ctypes.c_float(py), ctypes.c_float(EPS32), _p(g_ndc), _p(gv), _p(gR), _p(gT))

    K = torch.zeros(4, 4, dtype=torch.float64)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[2, 3], K[3, 2] = (float(np.float32(x)) for x in (fx, fy, px, py, 1.0, 1.0))
    v64, R64, T64 = (torch.from_numpy(a).double().requires_grad_(True) for a in (verts, R, T))
    ndc = pt3d.world_to_ndc(v64, R64, T64, K, eps=EPS32)
    z = ndc[3, :9, 2].detach()
    assert (z == 0).any() and ((z.abs() < EPS32) & (z != 0)).any() and (z < 0).any(), 'the special depths are missing'
    ref_v, ref_R, ref_T = torch.autograd.grad((ndc * torch.from_numpy(g_ndc).double()).sum(), [v64, R64, T64])
    for b in range(B):
        for name, got, ref in (('g_R', gR[b], ref_R[b]), ('g_T', gT[b], ref_T[b])):
            ref = ref.numpy()
            err = np.abs(got - ref).max() / np.abs(ref).max()
            assert err < 2e-5, f'view {b} {name}: {err:.3e}'
    err = np.abs(gv - ref_v.numpy()).max(1) / np.abs(ref_v.numpy()).max(1)
    assert err.max() < 2e-5, f'g_verts: {err.max():.3e}'


def test_camera_gradients_of_an_ndc_render_fail_loudly():
    """R and T are not part of a render from NDC vertices: asking for their gradient is an error (raised before any device
    work, so this runs without a GPU)"""
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    L = _lib.lib()
    s = make_settings(1, 8, 8, 1, 3, 1, 1, 0, (1, 1, 0, 0), 0., 0., None, (0, 0, 0), n_map_floats=12, verts_are_ndc=True,
                      save_fragment_state=True)
    fake = ctypes.c_void_p(16)          # never dereferenced: the call fails on its arguments
    args = [ctypes.byref(s)] + [fake] * 9 + [fake, 1 << 20, fake, None, fake, None, None]
    assert L.dbw_render_backward(*args, fake, None, fake, 1 << 20, None) != 0
    assert b'verts_are_ndc' in L.dbw_last_error()
    assert L.dbw_render_backward(*args, None, None, None, 1 << 20, None) != 0      # no scratch: the null check
    assert b'null pointer' in L.dbw_last_error()


def test_oracle_camera_gradients_match_finite_differences():
    """soft blocks render (sigma > 0, K = 10), constant textures so that detaching the barycentrics does not matter"""
    tpl = D.SceneTemplate(n_blocks=3, txt_size=16)
    p = D.init_params(3, 16, seed=2, dtype=torch.float64)
    p['textures'] = torch.randn(3, 1, 1, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(1)).expand(3, 16, 16, 3).clone()
    R, T, K = D.ring_cameras(2, dtype=torch.float64)
    blocks, alpha = tpl.build_blocks(p)
    fa = alpha.detach().repeat_interleave(tpl.BNF)
    imgs = torch.rand(2, 3, 32, 40, generator=torch.Generator().manual_seed(0), dtype=torch.float64)

    def loss_fn(R_, T_):
        out = D.render(blocks, R_, T_, K, (32, 40), sigma=1e-3, faces_per_pixel=10, z_clip=0.001, detach_bary=True, faces_alpha=fa)
        return D.mse_loss(imgs, out[:, :3]) + out[:, 3].mean()

    Rg, Tg = R.clone().requires_grad_(True), T.clone().requires_grad_(True)
    gR, gT = torch.autograd.grad(loss_fn(Rg, Tg), [Rg, Tg])
    assert gR.abs().max() > 0 and gT.abs().max() > 0
    h = 1e-6
    for name, idx in [('R', (0, 0, 2)), ('R', (1, 2, 1)), ('R', (1, 0, 0)), ('T', (0, 2)), ('T', (1, 0)), ('T', (0, 1))]:
        pr, pt = R.clone(), T.clone()
        (pr if name == 'R' else pt)[idx] += h
        lp = loss_fn(pr, pt).item()
        (pr if name == 'R' else pt)[idx] -= 2 * h
        lm = loss_fn(pr, pt).item()
        fd, ag = (lp - lm) / (2 * h), (gR if name == 'R' else gT)[idx].item()
        assert abs(fd - ag) <= 1e-4 * max(abs(fd), abs(ag)) + 1e-9, (name, idx, fd, ag)
