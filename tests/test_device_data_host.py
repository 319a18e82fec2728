"""CPU: the training-view loader without a GPU.  The resampler's math (differentiable-blocksworld_b200/csrc/dbw_data_math.cuh,
compiled for the host with the host-side coefficient builder by tests/host_math/dbw_data_host.cpp, g++ -ffp-contract=off) against
the installed Pillow's Image.resize(BILINEAR), bit for bit; the uint8 -> float division against ToTensor; the keyed permutation
(exhaustively a bijection for every P up to 4096); and DeviceLoader's batch order and global-RNG draws against the installed
torch's own DataLoader and DistributedSampler.  The kernels themselves are tested in tests/test_device_data_gpu.py."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope='module')
def hm():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_data_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_data_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.hm_resample.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.hm_resample.restype = None
    L.hm_u8_to_unit.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    L.hm_u8_to_unit.restype = None
    L.hm_permutation.argtypes = [ctypes.c_uint64] * 4 + [ctypes.c_int64, ctypes.c_void_p]
    L.hm_permutation.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _host_resize(hm, img, out_h, out_w):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty((out_h, out_w, 3), np.uint8)
    hm.hm_resample(img.shape[0], img.shape[1], _p(img), out_h, out_w, _p(out))
    return out


def _pil_resize(img, out_h, out_w):
    return np.asarray(Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR))


# (in_h, in_w, out_h, out_w): the DTU and BlendedMVS shapes, a 2x downscale, odd and non-integer ratios, upscales, one-row
# and one-column outputs, one axis unchanged, sizes where a pass is skipped, and both sides of Pillow's pass-order switch
RESIZE_CASES = [
    (1200, 1600, 300, 400), (576, 768, 288, 384), (540, 960, 270, 480),
    (97, 131, 31, 45), (100, 100, 33, 67), (123, 77, 50, 50), (64, 48, 37, 29),
    (30, 40, 64, 81), (7, 5, 20, 13), (50, 60, 100, 30),
    (40, 50, 1, 17), (40, 50, 17, 1), (40, 50, 1, 1), (1, 9, 1, 4), (9, 1, 3, 1),
    (60, 80, 60, 33), (60, 80, 21, 80), (45, 45, 45, 45), (300, 400, 300, 400),
    (1200, 1600, 40, 53),
    # tall, narrow sources: Image.resize runs the vertical pass first when the height exceeds 100x the width and shrinks
    (1000, 3, 999, 5), (1000, 9, 300, 4), (400, 2, 50, 7), (1001, 10, 500, 3),
    (1000, 10, 999, 5), (1000, 3, 1500, 5), (1000, 3, 400, 3),
]


@pytest.mark.parametrize('in_h,in_w,out_h,out_w', RESIZE_CASES)
def test_resample_matches_pillow_bit_for_bit(hm, in_h, in_w, out_h, out_w):
    rng = np.random.default_rng(in_h * 7919 + in_w * 31 + out_h * 3 + out_w)
    img = rng.integers(0, 256, (in_h, in_w, 3), dtype=np.uint8)
    # smooth content as well as noise: the saturated and mid-range sums both occur
    yy, xx = np.mgrid[:in_h, :in_w]
    img[: in_h // 2] = ((np.stack([xx, yy, xx + yy], -1)[: in_h // 2] * 255) // max(in_h + in_w, 1)).astype(np.uint8)
    got, want = _host_resize(hm, img, out_h, out_w), _pil_resize(img, out_h, out_w)
    assert got.shape == want.shape
    np.testing.assert_array_equal(got, want)


def test_resample_extremes_match_pillow(hm):
    for v in (0, 255):
        img = np.full((33, 47, 3), v, np.uint8)
        np.testing.assert_array_equal(_host_resize(hm, img, 10, 13), _pil_resize(img, 10, 13))
    img = np.zeros((40, 40, 3), np.uint8)
    img[::2, ::2] = 255                                        # a checkerboard: the widest spread of tap values
    np.testing.assert_array_equal(_host_resize(hm, img, 13, 17), _pil_resize(img, 13, 17))


def test_u8_to_unit_is_totensors_division(hm):
    from torchvision.transforms import ToTensor
    x = np.arange(256, dtype=np.uint8)
    got = np.empty(256, np.float32)
    hm.hm_u8_to_unit(256, _p(x), _p(got))
    want = ToTensor()(Image.fromarray(np.repeat(x[None, :, None], 3, 2)))[0, 0].numpy()
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    assert not np.array_equal(got, (x.astype(np.float32) * np.float32(1 / 255)))        # the multiply would differ


def _perm(hm, P, n=None, seed=0, step=0, view=0):
    n = P if n is None else n
    out = np.empty(n, np.int64)
    hm.hm_permutation(P, seed, step, view, n, _p(out))
    return out


def test_permutation_is_a_bijection_for_every_size_up_to_4096(hm):
    for P in range(1, 4097):
        perm = _perm(hm, P, seed=P, step=3, view=P % 7)
        assert np.array_equal(np.sort(perm), np.arange(P)), P


def test_permutation_prefixes_have_no_duplicates_and_depend_on_the_key(hm):
    P = 2_500_000
    a = _perm(hm, P, 100_000, seed=1, step=0, view=0)
    assert len(np.unique(a)) == len(a) and a.min() >= 0 and a.max() < P
    for kw in (dict(seed=2, step=0, view=0), dict(seed=1, step=1, view=0), dict(seed=1, step=0, view=1)):
        b = _perm(hm, P, 100_000, **kw)
        assert len(np.unique(b)) == len(b)
        assert np.mean(a == b) < 1e-3
    np.testing.assert_array_equal(a, _perm(hm, P, 100_000, seed=1, step=0, view=0))
    # a uniform subset: the prefix's mean and spread are those of [0, P)
    assert abs(a.mean() / P - 0.5) < 0.01 and abs(a.std() / P - 12 ** -0.5) < 0.01


# ------------------------------------------------------------------ DeviceLoader's order and RNG draws, against torch
class _Items(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i


def _device_loader_epochs(n, bs, shuffle, epochs, **kw):
    from dbw_b200.data import DeviceLoader
    loader = DeviceLoader(_Items(n), bs, shuffle=shuffle, **kw)
    out = []
    for e in range(epochs):
        if 'rank' in kw:
            loader.sampler.set_epoch(e)
        _, batches = loader.index_batches()
        out.append(([list(b) for b in batches], torch.get_rng_state().clone(), len(loader)))
    return out


def _torch_loader_epochs(n, bs, shuffle, epochs, rank=None, world_size=None):
    from torch.utils.data import DataLoader, DistributedSampler
    ds = _Items(n)
    if rank is not None:
        sampler = DistributedSampler(ds, num_replicas=world_size, rank=rank, shuffle=shuffle)
        loader = DataLoader(ds, batch_size=bs, sampler=sampler, collate_fn=list)
    else:
        sampler, loader = None, DataLoader(ds, batch_size=bs, shuffle=shuffle, collate_fn=list)
    out = []
    for e in range(epochs):
        if sampler is not None:
            sampler.set_epoch(e)
        out.append(([list(b) for b in loader], torch.get_rng_state().clone(), len(loader)))
    return out


@pytest.mark.parametrize('n,bs', [(49, 4), (16, 4), (5, 8), (1, 1), (10, 3)])
@pytest.mark.parametrize('shuffle', [True, False])
def test_device_loader_order_and_rng_state_equal_torchs_dataloader(n, bs, shuffle):
    torch.manual_seed(1234)
    mine = _device_loader_epochs(n, bs, shuffle, 3)
    torch.manual_seed(1234)
    ref = _torch_loader_epochs(n, bs, shuffle, 3)
    for (b1, s1, l1), (b2, s2, l2) in zip(mine, ref):
        assert b1 == b2 and l1 == l2
        assert torch.equal(s1, s2)
    if shuffle and n > 2:
        assert mine[0][0] != mine[1][0]                        # a new order every epoch


@pytest.mark.parametrize('world_size', [1, 2, 3])
@pytest.mark.parametrize('shuffle', [True, False])
@pytest.mark.parametrize('n,bs', [(49, 4), (10, 3)])
def test_device_loader_follows_distributed_sampler(world_size, shuffle, n, bs):
    for rank in range(world_size):
        torch.manual_seed(7)
        mine = _device_loader_epochs(n, bs, shuffle, 3, rank=rank, world_size=world_size)
        torch.manual_seed(7)
        ref = _torch_loader_epochs(n, bs, shuffle, 3, rank=rank, world_size=world_size)
        for (b1, s1, l1), (b2, s2, l2) in zip(mine, ref):
            assert b1 == b2 and l1 == l2
            assert torch.equal(s1, s2)


def test_rng_draws_happen_when_dataloader_makes_them():
    """the base seed at iter(), the sampler's seed at the first batch: interleaved draws see the same state"""
    from torch.utils.data import DataLoader
    from dbw_b200.data import DeviceLoader

    def run(make):
        torch.manual_seed(99)
        it = make()
        a = torch.rand(1)
        first = next(it)
        return a, first, torch.rand(1)
    ours = run(lambda: (lambda p: (b for b in p[1]))(DeviceLoader(_Items(12), 5, shuffle=True).index_batches()))
    ref = run(lambda: iter(DataLoader(_Items(12), batch_size=5, shuffle=True, collate_fn=list)))
    assert torch.equal(ours[0], ref[0]) and list(ours[1]) == list(ref[1]) and torch.equal(ours[2], ref[2])


def test_reference_transform_detection():
    from torchvision.transforms import Compose, InterpolationMode, Normalize, Resize, ToTensor
    from dbw_b200.data import is_reference_transform

    class D:
        img_size = (300, 400)

    d = D()
    d.transform = Compose([Resize(d.img_size), ToTensor()])
    assert is_reference_transform(d)
    for t in (Compose([Resize(300), ToTensor()]), Compose([Resize((300, 401)), ToTensor()]),
              Compose([Resize(d.img_size, InterpolationMode.NEAREST), ToTensor()]),
              Compose([Resize(d.img_size), ToTensor(), Normalize([0.5] * 3, [0.5] * 3)]), None):
        d.transform = t
        assert not is_reference_transform(d)


def test_cabi_refuses_bad_arguments_before_any_launch():
    from dbw_b200 import _lib
    L = _lib.lib()
    nbytes = ctypes.c_size_t(0)
    assert L.dbw_resample_u8_workspace_bytes(1, 1200, 1600, 300, 400, ctypes.byref(nbytes)) == 0 and nbytes.value > 0
    assert L.dbw_resample_u8_workspace_bytes(0, 10, 10, 5, 5, ctypes.byref(nbytes)) != 0
    assert L.dbw_resample_u8(1, 10, 10, None, 5, 5, None, None, 0, None) != 0
    assert L.dbw_gather_views(4, 0, ctypes.c_void_p(8), None, 1, 1, None, None, 0, None) != 0
    assert L.dbw_gather_views(4, 2, ctypes.c_void_p(8), None, 1, 1, None, None, 0, None) != 0          # nothing to gather
    f = (_lib.DbwGatherField * 5)()
    assert L.dbw_gather_views(4, 2, ctypes.c_void_p(8), None, 1, 1, None, f, 5, None) != 0             # too many fields
    assert L.dbw_subsample_points(10, 3, ctypes.c_void_p(8), 4, 2, ctypes.c_void_p(8), 0, 0, 11, ctypes.c_void_p(8), None) != 0
    assert 'n_out' in L.dbw_last_error().decode()


def test_compat_load_ply_reads_a_point_cloud(tmp_path):
    """in a subprocess (the stand-ins must not leak into this session): load_ply returns float32 verts and no faces, and
    refuses a mesh rather than dropping its faces"""
    code = r'''
import sys; sys.path.insert(0, %r)
import numpy as np, torch, dbw_b200, dbw_b200.compat as compat
from dbw_b200.dtu_eval import write_ply
if 'pytorch3d' in compat.install():
    from pytorch3d.io import load_ply
    pts = torch.randn(57, 3)
    for binary in (True, False):
        write_ply(%r, pts.numpy(), binary=binary)
        verts, faces = load_ply(%r)
        assert verts.dtype == torch.float32 and torch.equal(verts, pts) and faces.shape == (0, 3) and faces.dtype == torch.int64
    open(%r, 'wb').write(b'ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n'
                         b'element face 1\nproperty list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n0 1 0\n3 0 1 2\n')
    try:
        load_ply(%r)
        raise SystemExit('a mesh was read as a point cloud')
    except NotImplementedError:
        pass
print('OK')
''' % (ROOT, str(tmp_path / 'a.ply'), str(tmp_path / 'a.ply'), str(tmp_path / 'm.ply'), str(tmp_path / 'm.ply'))
    res = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and 'OK' in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
