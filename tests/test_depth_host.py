"""CPU: the depth outputs of the raster kernels.

1. The per-fragment depth and its derivative (csrc/dbw_depth_math.cuh) compiled for the host
   (tests/host_math/dbw_depth_host.cpp), against float64 torch autograd of PyTorch3D's zbuf: pz = bc . (z0, z1, z2) with
   the barycentrics perspective-corrected and clipped as the render's, differentiated with respect to the triangle's 9
   coordinates -- perspective correction on and off, barycentric clipping on and off, pixels inside and outside (halo
   fragments, where the clip is active), z-clipped triangles after the clip conversion (oracle clip_faces), and the guarded
   cases (a pixel on a vertex, where clipping renormalises to exactly one barycentric).
2. The C-ABI: both depth entry points are exported and refuse, with a message and without a device, what they do not cover.
3. The SASS of every kernel the depth outputs did not add is the parent build's (tests/golden/render_sass_sm90a.json holds
   SHA-256 digests of each kernel's instructions, as cuobjdump prints them without addresses)."""
import ctypes
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import pt3d

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'host_math', 'dbw_depth_host.cpp')


@pytest.fixture(scope='module')
def hd():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_depth_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', '-Wno-unknown-pragmas', SRC, '-o', so], check=True)
    lib = ctypes.CDLL(so)
    lib.hd_depth.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p,
                             ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _host(hd, tri, p, persp, clipb, g):
    tri = np.ascontiguousarray(tri, dtype=np.float32).reshape(9)
    p = np.ascontiguousarray(p, dtype=np.float32)
    pz, inside, gv = np.zeros(1, np.float32), np.zeros(1, np.int32), np.zeros(9, np.float32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    hd.hd_depth(P(tri), P(p), int(persp), int(clipb), float(g), P(pz), P(inside), P(gv))
    return float(pz[0]), bool(inside[0]), gv


def _oracle(tri, p, persp, clipb):
    """float64 zbuf of one (pixel, triangle) pair: PyTorch3D's BarycentricCoordinatesForward, perspective correction and
    clipping, then pz = bary . z; and its gradient with respect to the triangle's 9 coordinates"""
    t = torch.tensor(np.asarray(tri, dtype=np.float64).reshape(3, 3), requires_grad=True)
    px, py = (float(c) for c in p)
    v0, v1, v2 = t[0], t[1], t[2]
    edge = lambda qx, qy, a, b: (qx - a[0]) * (b[1] - a[1]) - (qy - a[1]) * (b[0] - a[0])
    area = edge(v2[0], v2[1], v0, v1) + 1e-8
    b = torch.stack([edge(px, py, v1, v2), edge(px, py, v2, v0), edge(px, py, v0, v1)]) / area
    if persp:
        z0, z1, z2 = t[0, 2], t[1, 2], t[2, 2]
        tt = torch.stack([b[0] * z1 * z2, z0 * b[1] * z2, z0 * z1 * b[2]])
        b = tt / tt.sum().clamp(min=1e-8)
    if clipb:
        w = b.clamp(min=0)
        b = w / w.sum().clamp(min=1e-5)
    pz = (b * t[:, 2]).sum()
    g, = torch.autograd.grad(pz, t)
    return pz.item(), g.reshape(9).numpy()


def _check(hd, tri, p, persp, clipb, what):
    # the oracle sees the float32 inputs the kernels see: a thin clipped triangle's gradient is ill-conditioned in its inputs
    tri, p = np.asarray(tri, dtype=np.float32), np.asarray(p, dtype=np.float32)
    pz, _, gv = _host(hd, tri, p, persp, clipb, 1.0)
    rz, rg = _oracle(tri, p, persp, clipb)
    zs = max(abs(v) for v in np.asarray(tri).reshape(3, 3)[:, 2])
    assert abs(pz - rz) <= 1e-4 * zs, f'{what}: pz {pz} vs {rz}'        # the GPU bar: 1e-4 of the depth range
    # the project's gradient bars (tests/test_raster_matrix_gpu.py): 1e-3 relative L2, 2e-3 of the largest magnitude per element
    scale = np.abs(rg).max() + 1e-12
    err = np.abs(gv - rg).max()
    rel = np.linalg.norm(gv - rg) / (np.linalg.norm(rg) + 1e-30)
    assert rel <= 1e-3 and err <= 2e-3 * scale, f'{what}: grad rel {rel:.3e}, max err {err:.3e} vs max |ref| {scale:.3e}\n{gv}\n{rg}'


def _random_tris(seed, n):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        xy = g.uniform(-0.9, 0.9, (3, 2))
        z = g.uniform(0.5, 6.0, 3)
        out.append(np.concatenate([xy, z[:, None]], 1))
    return out


@pytest.mark.parametrize('persp', [True, False])
@pytest.mark.parametrize('clipb', [True, False])
def test_depth_and_gradient_inside(hd, persp, clipb):
    g = np.random.default_rng(1)
    for i, tri in enumerate(_random_tris(2, 40)):
        w = g.dirichlet([2, 2, 2])
        p = (w[:, None] * tri[:, :2]).sum(0)
        pz, inside, _ = _host(hd, tri, p, persp, clipb, 1.0)
        assert inside, i
        _check(hd, tri, p, persp, clipb, f'tri {i}')


@pytest.mark.parametrize('persp', [True, False])
def test_depth_and_gradient_of_halo_fragments(hd, persp):
    """pixels outside the triangle (a soft render keeps them within the blur radius): the clip of the barycentrics is active"""
    g = np.random.default_rng(3)
    n = 0
    for i, tri in enumerate(_random_tris(4, 200)):
        w = g.dirichlet([2, 2, 2]) * 1.4 - 0.2 * g.permutation([1.0, 0.0, 0.0])
        w = w / w.sum()
        if (w > 0).all():
            continue
        p = (w[:, None] * tri[:, :2]).sum(0)
        _, inside, _ = _host(hd, tri, p, persp, True, 1.0)
        if inside:
            continue
        _check(hd, tri, p, persp, True, f'halo tri {i}')
        n += 1
    assert n >= 20


@pytest.mark.parametrize('persp', [True, False])
def test_z_clipped_triangles_after_the_clip_conversion(hd, persp):
    """a face straddling z_clip = 0.001 is rasterized as its clipped triangle(s): zbuf is the z interpolated on those"""
    g = np.random.default_rng(5)
    n = 0
    for _ in range(40):
        fv = np.concatenate([g.uniform(-0.8, 0.8, (3, 2)), np.array([[g.uniform(-0.5, -0.05)], [g.uniform(0.5, 3)], [g.uniform(0.5, 3)]])], 1)
        fv = torch.tensor(fv[None], dtype=torch.float64)
        cl = pt3d.clip_faces(fv, torch.tensor([0]), torch.tensor([1]), 0.001, persp)
        for tri in cl.face_verts.numpy():
            if abs(np.cross(tri[1, :2] - tri[0, :2], tri[2, :2] - tri[0, :2])) < 2e-2:
                continue                # slivers: their float32 barycentrics are ill-conditioned, whatever the math
            assert tri[:, 2].min() >= 0.001 - 1e-9
            # pixels on screen inside the clipped triangle (a vertex on the clip plane projects to NDC coordinates in the
            # hundreds, where no pixel is and float32 edge functions cancel)
            for p in g.uniform(-1, 1, (40, 2)):
                if _host(hd, tri, p, persp, True, 1.0)[1]:
                    _check(hd, tri, p, persp, True, 'clipped')
                    n += 1
    assert n >= 20


@pytest.mark.parametrize('persp', [True, False])
def test_guarded_cases(hd, persp):
    """a pixel exactly on a vertex: two barycentrics vanish and clipping renormalises the third to exactly 1, so zbuf is that
    vertex's z; a pixel beyond a vertex (two barycentrics negative) gives the same"""
    tri = np.array([[0.5, -0.25, 2.0], [-0.5, -0.25, 3.0], [0.0, 0.5, 4.0]], dtype=np.float32)
    for p, z in (((0.5, -0.25), 2.0), ((0.0, 0.75), 4.0)):
        pz, _, gv = _host(hd, tri, p, persp, True, 1.0)
        assert pz == z
        _check(hd, tri, p, persp, True, f'vertex {p}')
    pz, _, gv = _host(hd, tri, (0.1, 0.0), persp, True, 0.0)
    assert not gv.any(), 'a zero depth gradient gives zero'


# ------------------------------------------------------------------------------------------------ C-ABI
def test_depth_entry_points_are_exported_and_refuse_what_they_do_not_cover():
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    L = _lib.lib()
    assert {'dbw_render_forward_depth', 'dbw_render_backward_depth'} <= set(_lib.EXPORTS)
    s = make_settings(2, 16, 16, 4, 8, 4, 1, 0, (1., 1., 0., 0.), 1e-4, 9e-4, -1.0, (0, 0, 0), n_map_floats=3 * 16)
    rows = torch.zeros(2, 2, dtype=torch.int32)
    s.view_rows = rows.data_ptr()                  # host memory: never read, the call refuses first
    one = ctypes.c_void_p(8)
    assert L.dbw_render_forward_depth(ctypes.byref(s), *[one] * 9, one, None, one, 1 << 20, None, None, one, one, None) != 0
    assert b'row bands' in L.dbw_last_error()
    assert L.dbw_render_backward_depth(ctypes.byref(s), *[one] * 10, 1 << 20, one, None, one, one, one, None, None, None,
                                       None, one, 1 << 20, None) != 0
    assert b'row bands' in L.dbw_last_error()
    s.view_rows = None
    assert L.dbw_render_forward_depth(ctypes.byref(s), *[one] * 9, one, None, one, 1 << 20, one, None, one, one, None) != 0
    assert b'face_shade' in L.dbw_last_error()
    s.faces_per_pixel = 0
    assert L.dbw_render_forward_depth(ctypes.byref(s), *[one] * 9, one, None, one, 1 << 20, None, None, one, one, None) != 0
    assert b'faces_per_pixel' in L.dbw_last_error()


# ------------------------------------------------------------------------------------------------ SASS
def _sass_digests(cubin):
    out, cur = {}, None
    dump = subprocess.run([os.path.join(os.path.dirname(shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'), 'cuobjdump'),
                           '-sass', cubin], check=True, capture_output=True, text=True).stdout
    for line in dump.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        if cur:
            ins = re.sub(r'/\*[0-9a-f]{4,}\*/', '', line).strip()
            if ins:
                out[cur].append(ins)
    return {k: hashlib.sha256('\n'.join(v).encode()).hexdigest() for k, v in out.items()}


def test_kernels_without_depth_keep_their_sass(tmp_path):
    nvcc = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
    if nvcc is None:
        pytest.skip('nvcc is not installed')
    csrc = os.path.join(ROOT, 'differentiable-blocksworld_b200', 'csrc')
    cubin = str(tmp_path / 'dbw_render.cubin')
    subprocess.run([nvcc, '-O3', '-std=c++17', '-lineinfo', '-prec-div=false', '-gencode', 'arch=compute_90a,code=sm_90a', '-cubin',
                    os.path.join(csrc, 'dbw_render.cu'), '-o', cubin], check=True)
    got = _sass_digests(cubin)
    want = json.load(open(os.path.join(HERE, 'golden', 'render_sass_sm90a.json')))
    changed = sorted(k for k in want if got.get(k) != want[k])
    assert not changed, f'SASS changed: {changed}'
    added = sorted(k for k in got if k not in want)
    assert added and all('depth' in k for k in added), added
