"""CPU: per-view intrinsics (dbw_camera_project / dbw_camera_project_backward, renderer.project_verts).

1. The projection and its backward -- camera_project_kernel's arithmetic and the csrc/dbw_camera.cuh functions the backward
   kernels inline, dbw_intrinsics_accumulate among them -- compiled for the host (tests/host_math/dbw_intrinsics_host.cpp)
   and driven per (view, vertex) as the kernels drive them, against torch autograd of oracle.pt3d.world_to_ndc in float64,
   one K per view: random poses and intrinsics, plus a signed-permutation view whose depths are exact and include 0, the
   |z| < eps clamp and negative z.  The float64 oracle's d/dK against central differences.
2. The C-ABI: both entry points exported; argument validation.
3. The data-parallel step with intrinsics gradients (ViewParallel(max_pose_views=N, intrinsics=True)) over two gloo ranks:
   the gradient reaching the caller's K equals the single-process gradient, bit-identical on both ranks; the bucket layout."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import pt3d
from tests.test_camera_grad_host import EPS32, _inputs
from tests.test_host_logic import _GlooBucket

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'host_math', 'dbw_intrinsics_host.cpp')


@pytest.fixture(scope='module')
def hi():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_intrinsics_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', SRC, '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _intrinsics(B, seed):
    """(B,4) float32: focal lengths +-5 % around 1.7 / 2.1, principal points shifted per view"""
    g = np.random.default_rng(100 + seed)
    f = np.array([1.7, 2.1]) * g.uniform(0.95, 1.05, (B, 2))
    return np.ascontiguousarray(np.concatenate([f, g.uniform(-0.25, 0.25, (B, 2))], 1).astype(np.float32))


def _K64(intr):
    """(B,4,4) float64 K of the reference's layout (src/dataset/dtu.py:102-106) holding the given (fx, fy, px, py)"""
    K = torch.zeros(len(intr), 4, 4, dtype=torch.float64)
    i = torch.from_numpy(intr).double()
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 3], K[:, 3, 2] = i[:, 0], i[:, 1], i[:, 2], i[:, 3], 1., 1.
    return K


def _oracle_ndc(v, R, T, K):
    """per-view float64 projection: oracle.pt3d.world_to_ndc takes one K, so each view is projected with its own"""
    return torch.cat([pt3d.world_to_ndc(v, R[b:b + 1], T[b:b + 1], K[b], eps=EPS32) for b in range(R.shape[0])])


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_projection_forward_and_backward_match_autograd(hi, seed):
    verts, R, T, g_ndc = _inputs(seed)
    B, V = R.shape[0], verts.shape[0]
    intr = _intrinsics(B, seed)
    ndc = np.zeros((B, V, 3), np.float32)
    hi.hi_project(B, V, _p(verts), _p(R), _p(T), _p(intr), ctypes.c_float(EPS32), _p(ndc))
    gv, gR, gT, gI = (np.zeros(s, np.float32) for s in ((V, 3), (B, 3, 3), (B, 3), (B, 4)))
    hi.hi_project_backward(B, V, _p(verts), _p(R), _p(T), _p(intr), ctypes.c_float(EPS32), _p(g_ndc), _p(gv), _p(gR), _p(gT), _p(gI))

    K = _K64(intr).requires_grad_(True)
    v64, R64, T64 = (torch.from_numpy(a).double().requires_grad_(True) for a in (verts, R, T))
    ref = _oracle_ndc(v64, R64, T64, K)
    z = ref[3, :9, 2].detach()
    assert (z == 0).any() and ((z.abs() < EPS32) & (z != 0)).any() and (z < 0).any(), 'the special depths are missing'
    # forward: float32 arithmetic against float64, relative to each coordinate's magnitude (the clamp makes some huge)
    err = np.abs(ndc - ref.detach().numpy()) / np.maximum(np.abs(ref.detach().numpy()), 1.0)
    assert err.max() < 2e-6, err.max()
    ref_v, ref_R, ref_T, ref_K = torch.autograd.grad((ref * torch.from_numpy(g_ndc).double()).sum(), [v64, R64, T64, K])
    ref_I = torch.stack([ref_K[:, 0, 0], ref_K[:, 1, 1], ref_K[:, 0, 2], ref_K[:, 1, 2]], -1)
    for b in range(B):
        for name, got, want in (('g_R', gR[b], ref_R[b]), ('g_T', gT[b], ref_T[b]), ('g_K', gI[b], ref_I[b])):
            want = want.numpy()
            scale = max(np.abs(want).max(), 1e-30)
            assert np.abs(got - want).max() <= 2e-5 * scale, (name, b, np.abs(got - want).max(), scale)
    assert np.abs(gv - ref_v.numpy()).max() <= 2e-5 * np.abs(ref_v.numpy()).max()


def test_oracle_intrinsics_gradient_matches_central_differences():
    """float64 d/d(fx, fy, px, py) of a weighted sum of the per-view projection, away from the clamp, against central
    differences: the reference the GPU tests take"""
    verts, R, T, g_ndc = _inputs(5)
    B = 3                                                        # the random views (view 3 holds the clamp's depths)
    intr = _intrinsics(B, 5)
    v64, R64, T64 = (torch.from_numpy(a).double() for a in (verts, R[:B], T[:B]))
    w = torch.from_numpy(g_ndc[:B]).double()
    K = _K64(intr).requires_grad_(True)
    (g,) = torch.autograd.grad((_oracle_ndc(v64, R64, T64, K) * w).sum(), [K])
    h = 1e-6
    for b in range(B):
        for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)):
            Kp, Km = K.detach().clone(), K.detach().clone()
            Kp[b, i, j] += h
            Km[b, i, j] -= h
            fd = ((_oracle_ndc(v64, R64, T64, Kp) * w).sum() - (_oracle_ndc(v64, R64, T64, Km) * w).sum()) / (2 * h)
            assert abs(fd.item() - g[b, i, j].item()) <= 1e-7 * max(1.0, abs(fd.item())), (b, i, j, fd.item(), g[b, i, j].item())


def test_c_abi_entry_points_validate_their_arguments():
    from dbw_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(8)                 # never dereferenced: every call below fails before any launch
    f = ctypes.c_float
    cases = [
        (L.dbw_camera_project, (0, 4, one, one, one, one, f(1e-8), one, None), 'n_views and n_verts must be positive'),
        (L.dbw_camera_project, (2, 0, one, one, one, one, f(1e-8), one, None), 'n_views and n_verts must be positive'),
        (L.dbw_camera_project, (2, 4, one, one, one, None, f(1e-8), one, None), 'intrinsics are required'),
        (L.dbw_camera_project, (2, 4, one, one, one, one, f(0.0), one, None), 'eps must be positive'),
        (L.dbw_camera_project, (2, 4, one, one, one, one, f(1e-8), None, None), 'verts_ndc is required'),
        (L.dbw_camera_project, (1 << 16, 1 << 15, one, one, one, one, f(1e-8), one, None), '32-bit indexing'),
        (L.dbw_camera_project_backward, (0, 4, one, one, one, one, f(1e-8), one, one, one, one, one, None), 'must be positive'),
        (L.dbw_camera_project_backward, (2, 4, None, one, one, one, f(1e-8), one, one, one, one, one, None), 'are required'),
        (L.dbw_camera_project_backward, (2, 4, one, one, one, one, f(1e-8), None, one, one, one, one, None), 'g_ndc is required'),
    ]
    for fn, args, msg in cases:
        assert fn(*args) != 0, (fn, args)
        assert msg in L.dbw_last_error().decode(), L.dbw_last_error()


def test_project_verts_reads_four_entries_of_each_K():
    from dbw_b200.renderer import intrinsics_of
    K = torch.arange(3 * 16, dtype=torch.float64).view(3, 4, 4).requires_grad_(True)
    i = intrinsics_of(K)
    assert torch.equal(i.detach(), torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], -1).detach())
    i.sum().backward()
    assert K.grad.sum() == 12 and torch.equal(K.grad[:, 0, 0], torch.ones(3)) and torch.equal(K.grad[:, 1, 2], torch.ones(3))


# ------------------------------------------------------------------------------------------------ data-parallel step
B, H, W = 5, 48, 5
MAX_POSE_VIEWS = 8
CONFIGS = [(row_bands, reduce_at) for row_bands in (False, True) for reduce_at in ('leaf', 'scene')]


class _ToyIntrinsics(torch.nn.Module):
    """the ViewParallel contract with per-pixel 'renders' of each view's (fx, fy, px, py), routed through the gradient-sum
    point as DifferentiableBlocksWorld routes them; honours inp['rows'] the way the kernels do"""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.linspace(0.1, 0.9, W))
        self.textures = torch.nn.Parameter(torch.linspace(-1, 1, 6))
        self.n_total_views, self.noise_generator, self.grad_sum_point = None, None, None

    def _fused_loss_ok(self, imgs):
        return True

    def can_sum_gradients_at_scene_tensors(self, imgs):
        return True

    def grad_sum_floats(self):
        return W + 3

    def forward(self, inp, labels=None):
        from dbw_b200.renderer import intrinsics_of
        verts, cells = self.w.exp(), torch.sigmoid(self.textures).view(3, 2).mean(1)
        R, T, K = inp['R'], inp['T'], inp.get('K')
        if self.grad_sum_point is not None:
            verts, cells = self.grad_sum_point(verts, cells)
            R, T = self.grad_sum_point.cameras(inp)
            K = self.grad_sum_point.intrinsics(K)
        k = intrinsics_of(K)
        imgs = inp['imgs']
        y = torch.arange(H, dtype=imgs.dtype)[None, :, None] / H
        cam = ((R * torch.linspace(-1, 1, 9).view(3, 3)).sum((1, 2)) + (k * torch.tensor([0.3, -0.2, 0.5, 0.7])).sum(1))[:, None, None]
        cam = cam + (T * cells).sum(1)[:, None, None] * y + k[:, :1, None] * cells[0] * y
        err = (imgs * verts[None, None] + torch.sin(cam) * cells.sum() - 0.5) ** 2
        if inp.get('rows') is not None:
            yi = torch.arange(H)[None, :, None]
            err = err * ((yi >= inp['rows'][:, 0, None, None]) & (yi < inp['rows'][:, 1, None, None]))
        rgb = err.sum() / (self.n_total_views * H * W)
        reg = self.textures.pow(2).sum() + self.w.sum()
        return {'rgb': rgb, 'tv': reg, 'total': rgb + reg}


def _data():
    g = torch.Generator().manual_seed(1)
    imgs, R0, T0 = torch.rand(B, H, W, generator=g), torch.rand(B, 3, 3, generator=g), torch.rand(B, 3, generator=g)
    K0 = torch.zeros(B, 4, 4)
    K0[:, 0, 0], K0[:, 1, 1] = 1.7 + 0.1 * torch.rand(B, generator=g), 2.1 + 0.1 * torch.rand(B, generator=g)
    K0[:, 0, 2], K0[:, 1, 2], K0[:, 2, 3], K0[:, 3, 2] = 0.1 * torch.randn(B, generator=g), 0.1 * torch.randn(B, generator=g), 1, 1
    scale = (1 + 0.05 * torch.randn(B, generator=g)).requires_grad_(True)          # a focal-scale refinement leaf
    dT = (0.1 * torch.randn(B, 3, generator=g)).requires_grad_(True)
    return imgs, R0, T0, K0, scale, dT


def _with_scale(K0, scale):
    """K0 with fx, fy scaled per view (the principal point untouched)"""
    f = torch.stack([scale, scale, torch.ones_like(scale), torch.ones_like(scale)], -1)
    return K0 * torch.diag_embed(f) + K0 * (1 - torch.eye(4))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from dbw_b200.parallel import ViewParallel
    for row_bands, reduce_at in CONFIGS:
        torch.manual_seed(0)
        model = _ToyIntrinsics()
        vp = ViewParallel(model, seed=123, row_bands=row_bands, reduce_at=reduce_at, max_pose_views=MAX_POSE_VIEWS, intrinsics=True,
                          peer_factory=_GlooBucket if reduce_at == 'scene' else None)
        imgs, R0, T0, K0, scale, dT = _data()
        vp.forward_backward({'imgs': imgs, 'R': R0, 'T': T0 + dT, 'K': _with_scale(K0, scale)})
        sizes = list(vp.bucket.peer.sizes) if vp.bucket.peer is not None else None
        out[(rank, row_bands, reduce_at)] = (scale.grad.clone(), dT.grad.clone(), vp.bucket.grads_flat().clone(), sizes)
    dist.destroy_process_group()


def _reference():
    torch.manual_seed(0)
    model = _ToyIntrinsics()
    model.n_total_views = B
    imgs, R0, T0, K0, scale, dT = _data()
    total = model({'imgs': imgs, 'R': R0, 'T': T0 + dT, 'K': _with_scale(K0, scale)})['total']
    *g, gs, gT = torch.autograd.grad(total, list(model.parameters()) + [scale, dT])
    return gs, gT, torch.cat([x.reshape(-1) for x in g])


def test_intrinsics_gradients_summed_over_two_gloo_ranks_equal_single_process():
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(2, 37000 + os.getpid() % 2000, out), nprocs=2, join=True)
    gs, gT, gp = _reference()
    assert gs.abs().min() > 0 and gT.abs().max() > 0
    for row_bands, reduce_at in CONFIGS:
        r0, r1 = out[(0, row_bands, reduce_at)], out[(1, row_bands, reduce_at)]
        for i in range(3):
            assert torch.equal(r0[i], r1[i]), (row_bands, reduce_at, i)
        what = f'row_bands={row_bands} reduce_at={reduce_at}'
        assert torch.allclose(r0[0], gs, rtol=1e-5, atol=1e-7), what
        assert torch.allclose(r0[1], gT, rtol=1e-5, atol=1e-7), what
        assert torch.allclose(r0[2], gp, rtol=1e-5, atol=1e-7), what
        if reduce_at == 'scene':                  # one exchange per step: the scene tensors, then 9 + 3 + 4 floats per view
            assert r0[3] == [W + 3 + 16 * B], (what, r0[3])


def test_one_process_bucket_layout_with_intrinsics():
    """world size 1, leaf bucket gathered: g_R (B x 9), g_T (B x 3), then g_intrinsics (B x 4) after the parameter gradients;
    the arena reserves 16 floats per pose view, and 12 without the option (the layout of a pose-only step)"""
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.renderer import intrinsics_of
    torch.manual_seed(0)
    vp = ViewParallel(_ToyIntrinsics(), seed=123, max_pose_views=MAX_POSE_VIEWS, intrinsics=True, gather_grads=True)
    imgs, R0, T0, K0, scale, dT = _data()
    K0 = K0.requires_grad_(True)
    vp.forward_backward({'imgs': imgs, 'R': R0, 'T': T0 + dT, 'K': K0})
    n_pad = vp.bucket.flat.numel()
    assert vp.bucket._all.numel() == n_pad + 16 * MAX_POSE_VIEWS
    region = vp.bucket._all[n_pad + 12 * B:n_pad + 16 * B]
    assert torch.equal(region.view(B, 4), intrinsics_of(K0.grad))
    assert torch.equal(vp.bucket._all[n_pad + 9 * B:n_pad + 12 * B].view(B, 3), dT.grad)
    plain = ViewParallel(_ToyIntrinsics(), seed=123, max_pose_views=MAX_POSE_VIEWS, gather_grads=True)
    assert plain.bucket._all.numel() == n_pad + 12 * MAX_POSE_VIEWS


def test_steps_refuse_intrinsics_gradients_they_cannot_carry():
    from dbw_b200.parallel import ViewParallel
    imgs, R0, T0, K0, scale, dT = _data()
    inp = {'imgs': imgs, 'R': R0, 'T': T0, 'K': _with_scale(K0, scale)}
    with pytest.raises(RuntimeError, match=r"inp\['K'\] requires grad"):
        ViewParallel(_ToyIntrinsics(), seed=1).forward_backward(inp)
    with pytest.raises(RuntimeError, match='intrinsics=True'):
        ViewParallel(_ToyIntrinsics(), seed=1, max_pose_views=8).forward_backward(inp)
    with pytest.raises(ValueError, match='max_pose_views > 0'):
        ViewParallel(_ToyIntrinsics(), seed=1, intrinsics=True)
    with pytest.raises(ValueError, match='full batch'):
        ViewParallel(_ToyIntrinsics(), seed=1, max_pose_views=8, intrinsics=True).forward_backward(dict(inp, K=inp['K'][:3]))
    assert scale.grad is None
