"""CPU checks of the view-rendering layer (dbw_b200/views.py) and of the resolving hard render's arithmetic:
PyTorch3D's look-at cameras, the reference's circle trajectory, the box filter / composite / uint8 conversion of
csrc/dbw_viz_math.cuh compiled for the host against numpy, the mp4 and GIF writers, the new C-ABI symbols and their
refusals, and the registers and shared memory of every kernel that existed before the resolving kernel."""
import ctypes
import json
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from dbw_b200 import views as V

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------ cameras
def test_look_at_view_transform_known_values():
    for d in (0.5, 1.0, 2.732):
        R, T = V.look_at_view_transform(dist=d, elev=0, azim=0)
        assert torch.allclose(R, torch.diag(torch.tensor([-1., 1., -1.]))[None], atol=1e-7)
        assert torch.allclose(T, torch.tensor([[0., 0., d]]), atol=1e-7)


def test_look_at_view_transform_random_cameras():
    g = torch.Generator().manual_seed(0)
    N = 64
    dist = torch.rand(N, generator=g) * 5 + 0.5
    elev = torch.rand(N, generator=g) * 170 - 85
    azim = torch.rand(N, generator=g) * 720 - 360
    at = torch.randn(N, 3, generator=g)
    R, T = V.look_at_view_transform(dist, elev, azim, at=at)
    assert R.shape == (N, 3, 3) and T.shape == (N, 3)
    assert torch.allclose(R @ R.transpose(1, 2), torch.eye(3).expand(N, -1, -1), atol=1e-5)
    assert torch.allclose(torch.linalg.det(R), torch.ones(N), atol=1e-5)
    e, a = torch.deg2rad(elev.double()), torch.deg2rad(azim.double())
    C_ref = dist.double()[:, None] * torch.stack([e.cos() * a.sin(), e.sin(), e.cos() * a.cos()], 1) + at.double()
    C = -(T[:, None] @ R.transpose(1, 2))[:, 0]                 # camera centre: X_cam = X R + T = 0
    assert torch.allclose(C.double(), C_ref, atol=1e-4)
    at_cam = (at[:, None] @ R)[:, 0] + T                         # `at` lies on the optical axis at depth dist
    assert torch.allclose(at_cam, torch.stack([torch.zeros(N), torch.zeros(N), dist], 1), atol=1e-4)
    up_cam = (torch.tensor([[0., 1., 0.]]) @ R)                  # world up points up in the image
    assert (up_cam[:, 0, 1] > 0).all()


def test_look_at_broadcasting_and_degrees():
    R1, T1 = V.look_at_view_transform(2.0, 30.0, torch.tensor([0., 90., 180.]))
    R2, T2 = V.look_at_view_transform(torch.tensor([2.0] * 3), math.radians(30), torch.deg2rad(torch.tensor([0., 90., 180.])),
                                      degrees=False)
    assert R1.shape == (3, 3, 3) and torch.allclose(R1, R2, atol=1e-6) and torch.allclose(T1, T2, atol=1e-6)
    R3, T3 = V.look_at_view_transform(eye=((0., 0., 2.),))
    assert torch.allclose(R3, V.look_at_view_transform(2.0)[0], atol=1e-7) and torch.allclose(T3, torch.tensor([[0., 0., 2.]]))
    with pytest.raises(ValueError):
        V.look_at_view_transform(torch.ones(2), torch.zeros(3))


def test_compat_registers_the_look_at_functions():
    import sys
    import dbw_b200.compat as compat
    saved = {k: v for k, v in sys.modules.items() if k == 'pytorch3d' or k.startswith('pytorch3d.')}
    try:
        for k in saved:
            del sys.modules[k]
        compat._pytorch3d()
        from pytorch3d.renderer import look_at_view_transform, look_at_rotation
        assert look_at_view_transform is V.look_at_view_transform and look_at_rotation is V.look_at_rotation
    finally:
        for k in [k for k in sys.modules if k == 'pytorch3d' or k.startswith('pytorch3d.')]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_circle_trajectory_closed_form():
    for N in (1, 7, 240):
        R, T = V.get_circle_traj(N_views=N)
        t = torch.linspace(0, 2, N + 1, dtype=torch.float64)[:-1] * math.pi
        a, e = torch.deg2rad(t.cos() * 15 - 180), torch.deg2rad(t.sin() * 15)
        C = torch.stack([e.cos() * a.sin(), e.sin(), e.cos() * a.cos()], 1)        # dist 1 around the origin
        z = -C
        x = torch.nn.functional.normalize(torch.cross(torch.tensor([[0., 1., 0.]], dtype=torch.float64).expand(N, -1), z, dim=1), dim=1)
        y = torch.cross(z, x, dim=1)
        R_ref = torch.stack([x, y, z], 2)
        assert torch.allclose(R.double(), R_ref, atol=1e-6)
        assert torch.allclose(T.double(), torch.tensor([[0., 0., 1.]], dtype=torch.float64).expand(N, -1), atol=1e-6)


# ------------------------------------------------------------------ the resolve arithmetic, compiled for the host
@pytest.fixture(scope='module')
def hv():
    src = os.path.join(HERE, 'host_math', 'dbw_viz_host.cpp')
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_viz_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', src, '-o', so], check=True)
    L = ctypes.CDLL(so)
    for f in (L.hv_box, L.hv_composite, L.hv_u8):
        f.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _samples(g, n):
    """float32 samples in the ranges a render produces, plus exact zeros / ones, tiny and large values"""
    x = g.random((n, 16), dtype=np.float32)
    x[: n // 8] = np.float32(1.0)
    x[n // 8: n // 4] = 0.0
    x[n // 4: n // 4 + 16] = np.float32(1e-40)                       # subnormal sums: the 1/16 scaling must stay exact
    x[n // 3: n // 3 + 32] *= np.float32(3e4)
    return x


def test_box_filter_equals_numpy_row_major_mean(hv):
    g = np.random.default_rng(0)
    n = 1 << 16
    x = _samples(g, n)
    out = np.empty(n, np.float32)
    hv.hv_box(n, _p(x), _p(out))
    acc = np.zeros(n, np.float32)
    for k in range(16):                                             # avg_pool2d's order: rows, then columns, from 0
        acc = acc + x[:, k]
    ref = acc / np.float32(16)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    # and torch's avg_pool2d on the CPU gives the same bits for frames laid out as 4x4 blocks
    img = torch.from_numpy(x[:1024].reshape(32, 32, 4, 4).transpose(0, 2, 1, 3).reshape(1, 1, 128, 128).copy())
    pooled = torch.nn.functional.avg_pool2d(img, 4).reshape(-1).numpy()
    assert np.array_equal(pooled.view(np.uint32), out[:1024].view(np.uint32))


def test_composite_and_uint8_equal_numpy(hv):
    g = np.random.default_rng(1)
    n = 1 << 16
    rec = g.random(n, dtype=np.float32) * np.float32(1.2) - np.float32(0.1)
    a = g.random(n, dtype=np.float32)
    a[:1000] = 0.0
    a[1000:2000] = 1.0
    bkg = g.random(n, dtype=np.float32)
    out = np.empty(n, np.float32)
    hv.hv_composite(n, _p(rec), _p(a), _p(bkg), _p(out))
    ref = rec * a + (np.float32(1) - a) * bkg
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    x = np.concatenate([g.random(n, dtype=np.float32) * np.float32(1.4) - np.float32(0.2),
                        np.array([0, 1, -0.0, 1 / 255, 254.5 / 255, 255.5 / 255, np.nextafter(1, 0)], np.float32)])
    u8 = np.empty(len(x), np.uint8)
    hv.hv_u8(len(x), _p(x), _p(u8))
    ref8 = np.clip(x * np.float32(255), 0, 255).astype(np.uint8)
    assert np.array_equal(u8, ref8)
    t8 = (torch.from_numpy(x) * 255).clamp(0, 255).to(torch.uint8).numpy()
    assert np.array_equal(u8, t8)


# ------------------------------------------------------------------ writers
def _read_mp4(path):
    import cv2
    cap = cv2.VideoCapture(str(path))
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f[..., ::-1])
    cap.release()
    return np.stack(frames)


@pytest.mark.parametrize('size', [(48, 64), (37, 53), (20, 15)])
def test_save_video_reads_back(tmp_path, size):
    H, W = size
    g = torch.Generator().manual_seed(2)
    n = 13
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing='ij')
    imgs = torch.stack([torch.stack([xx, yy, (xx + yy) / 2]) * (k + 1) / n for k in range(n)])
    imgs = (imgs + 0.02 * torch.rand(imgs.shape, generator=g)).clamp(0, 1)
    out = tmp_path / 'v.mp4'
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        V.save_video(imgs, 'v.mp4')
    finally:
        os.chdir(cwd)
    frames = _read_mp4(out)
    # mp4v codes 4:2:0 chroma: an odd height or width gains one edge-replicated row / column
    assert frames.shape == (n, H + H % 2, W + W % 2, 3)
    ref = (imgs * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8).numpy().astype(np.float64)
    mse = ((frames[:, :H, :W].astype(np.float64) - ref) ** 2).mean()
    assert 10 * np.log10(255 ** 2 / mse) > 30                       # lossy, but the same pictures


def test_video_writer_streams_chunks(tmp_path):
    frames = np.random.default_rng(3).integers(0, 256, (10, 16, 24, 3), dtype=np.uint8)
    with V.VideoWriter(tmp_path / 's.mp4') as vw:
        vw.write(frames[:3])
        vw.write(torch.from_numpy(frames[3:]))
    assert vw.count == 10 and _read_mp4(tmp_path / 's.mp4').shape == (10, 16, 24, 3)


def test_save_gif_frames_duration_and_size_cap(tmp_path):
    from PIL import Image
    imgs = torch.rand(30, 3, 40, 300, generator=torch.Generator().manual_seed(4))
    V.save_gif(imgs, tmp_path / 'a.gif')
    im = Image.open(tmp_path / 'a.gif')
    assert im.n_frames == 30 and im.size == (256, round(40 * 256 / 300))           # fitted inside 256 x 256
    assert im.info['duration'] == int(10 * 1000 / 30) // 10 * 10                  # GIF delays are in 10 ms units
    V.save_gif(torch.rand(600, 3, 8, 8), tmp_path / 'b.gif', size=None)           # autodecimate: every other frame
    assert Image.open(tmp_path / 'b.gif').n_frames == 300


# ------------------------------------------------------------------ C-ABI and kernels
def test_viz_symbols_exported_and_refusals():
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    L = _lib.lib()
    assert {'dbw_viz_workspace_bytes', 'dbw_render_forward_viz'} <= set(_lib.EXPORTS)
    assert L.dbw_abi_version() == 8
    sz = ctypes.c_size_t(0)

    def settings(**kw):
        args = dict(B=2, H=64, W=48, K=1, sigma=0.0, blur=0.0)
        args.update(kw)
        return make_settings(args['B'], args['H'], args['W'], args['K'], 10, 8, 1, 0, (1., 1., 0., 0.), args['sigma'],
                             args['blur'], None, (0., 0., 0.), n_map_floats=48)
    assert L.dbw_viz_workspace_bytes(ctypes.byref(settings()), 4, ctypes.byref(sz)) == 0 and sz.value > 0
    two = ctypes.c_size_t(0)
    L.dbw_viz_workspace_bytes(ctypes.byref(settings(B=4)), 4, ctypes.byref(two))
    assert two.value > sz.value
    bad = [(settings(), 2, 'factor'), (settings(K=2), 4, 'hard'), (settings(sigma=1e-4), 4, 'hard'), (settings(H=62), 4, 'multiples')]
    for s, factor, why in bad:
        assert L.dbw_viz_workspace_bytes(ctypes.byref(s), factor, ctypes.byref(sz)) != 0
        assert why in L.dbw_last_error().decode()
        # the render refuses before it touches a pointer
        rc = L.dbw_render_forward_viz(ctypes.byref(s), *([None] * 10), factor, None, 0, None, None, None, 0, None)
        assert rc != 0 and why in L.dbw_last_error().decode()
    s = settings()
    rc = L.dbw_render_forward_viz(ctypes.byref(s), *([None] * 10), 4, None, 0, None, None, None, 0, None)
    assert rc != 0 and 'both NULL' in L.dbw_last_error().decode()
    rc = L.dbw_render_forward_viz(ctypes.byref(s), *([None] * 10), 4, ctypes.c_void_p(16), 3, ctypes.c_void_p(16), None, None, 0, None)
    assert rc != 0 and 'bkg_views' in L.dbw_last_error().decode()
    s = settings()
    s.save_fragment_state = 1
    assert L.dbw_viz_workspace_bytes(ctypes.byref(s), 4, ctypes.byref(sz)) != 0


def test_eye_light_is_refused():
    with pytest.raises(NotImplementedError):
        V.render_views(None, torch.eye(3)[None], torch.zeros(1, 3), eye_light=True)
    with pytest.raises(NotImplementedError):
        V.render_rotated_views(None, eye_light=True)


def stable_kernel_name(name):
    """a mangled kernel name without the build-dependent part: nvcc names a file's anonymous namespace
    `_GLOBAL__N__<hash>_<n>_<file>_cu_<hash>` with hashes that change with the build (the source's path among them);
    the namespace, given by its length prefix, becomes `<anon:file_cu>`"""
    out, pos = [], 0
    for m in re.finditer(r'(\d+)_GLOBAL__N__', name):
        if m.start() < pos:
            continue
        n = int(m.group(1))
        ident = name[m.end(1):m.end(1) + n]
        file = re.match(r'_GLOBAL__N__[0-9a-f]+_\d+_(\w+?_cu)_[0-9a-f]+$', ident)
        out.append(name[pos:m.start()] + f'<anon:{file.group(1) if file else "?"}>')
        pos = m.end(1) + n
    return ''.join(out) + name[pos:]


def test_stable_kernel_name_drops_the_build_hashes():
    a = '_ZN45_GLOBAL__N__703f8c05_12_dbw_lpips_cu_5239b50717lpips_pool_kernelILb0EEEvPK6float4PS1_liiiPKi'
    b = '_ZN45_GLOBAL__N__1a2b3c4d_12_dbw_lpips_cu_9f8e7d6c17lpips_pool_kernelILb0EEEvPK6float4PS1_liiiPKi'
    assert stable_kernel_name(a) == stable_kernel_name(b) == '_ZN<anon:dbw_lpips_cu>17lpips_pool_kernelILb0EEEvPK6float4PS1_liiiPKi'
    assert stable_kernel_name('_Z26raster_hard_forward_kernel12RasterParams') == '_Z26raster_hard_forward_kernel12RasterParams'


def test_existing_kernels_keep_their_registers_and_shared_memory():
    """the resolving kernel is a separate instantiation: every kernel of the library before it keeps its resources"""
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump is not installed')
    lib = os.path.join(ROOT, 'differentiable-blocksworld_b200', 'libdbw_render.so')
    text = subprocess.run([cuobjdump, '-res-usage', lib], check=True, capture_output=True, text=True).stdout
    now = {}
    for name, reg, shared in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)', text):
        now[stable_kernel_name(name)] = {'REG': int(reg), 'SHARED': int(shared)}
    with open(os.path.join(HERE, 'golden', 'kernel_resources_sm90a.json')) as fh:
        before = json.load(fh)
    assert '_Z23resolve_hard_viz_kernel12RasterParams6VizOut' in now
    changed = {k: (v, now.get(k)) for k, v in before.items() if now.get(k) != v}
    assert not changed, changed
