"""CPU: the evaluation's image scores without a GPU.  The float64 oracle (oracle/image_scores.py) against the reference's own
float32 SSIMLoss(padding=False) and mse2psnr frozen in tests/golden/image_scores.npz; the device math of the score kernel
(differentiable-blocksworld_b200/csrc/dbw_metrics_math.cuh) compiled for the host (tests/host_math/dbw_metrics_host.cpp,
g++ -ffp-contract=off) against the oracle, pixel by pixel; and the argument checks of the C-ABI and of dbw_b200.metrics,
which all fail before anything reaches a device.  The kernel itself is tested in tests/test_image_scores_gpu.py.

Bounds, set from the measured maxima.  On textured pairs the oracle reproduces the reference to 8.3e-7 in per-image SSIM and
1.0e-6 dB in PSNR.  On near-constant pairs the reference's own float32 sigma = E[x^2] - mu^2 cancels (the variance is below
the rounding of E[x^2]), so there it is 1.0e-4 from the float64 value; the host-compiled kernel math carries the same
float32 rounding (per pixel 1.4e-5 textured, 1.4e-4 near-constant)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import image_scores as O
from tests.golden.make_image_scores_golden import CASES, checksum, pairs

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, 'golden', 'image_scores.npz'))
NEAR_CONSTANT = {n for n, c in CASES.items() if c[3].startswith('flat')}
# name -> (per-image SSIM vs the reference, per-pixel host math vs the oracle, per-image host math vs the oracle)
BOUNDS = {n: (2e-4, 3e-4, 5e-6) if n in NEAR_CONSTANT else (1e-6, 3e-5, 1e-6) for n in CASES}
PSNR_DB = 2e-6


@pytest.fixture(scope='module')
def hm():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_metrics_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_metrics_host.cpp'), '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def test_window_is_the_references():
    from dbw_b200 import metrics
    assert np.array_equal(O.gaussian().numpy(), GOLDEN['window'])
    assert np.array_equal(np.float32(list(metrics._WINDOW)), GOLDEN['window'])


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_reproduces_the_references_scores(name):
    x, y = pairs(name)
    assert np.array_equal(checksum(x, y), GOLDEN[f'{name}/checksum'])       # the seeded pair is the one frozen
    ref_ssim = 1 - GOLDEN[f'{name}/ssim_loss'].astype(np.float64)
    err = np.abs(O.ssim(x, y).numpy() - ref_ssim).max()
    assert err <= BOUNDS[name][0], err
    ref_psnr, got = float(GOLDEN[f'{name}/psnr'][0]), O.psnr(x, y).item()
    if np.isinf(ref_psnr):                                                    # identical pair
        assert got == ref_psnr
    else:
        assert abs(got - ref_psnr) <= PSNR_DB, abs(got - ref_psnr)
    if name.startswith('same'):
        assert (ref_ssim == 1).all()


@pytest.mark.parametrize('name', list(CASES))
def test_device_math_matches_the_oracle_pixel_by_pixel(hm, name):
    x, y = pairs(name)
    B, C, H, W = x.shape
    got = np.zeros((B, C, H - 10, W - 10), np.float32)
    w = O.gaussian().numpy()
    for b in range(B):
        hm.hm_ssim_map(C, H, W, _p(x[b].numpy()), _p(y[b].numpy()), _p(w), _p(got[b]))
    want = O.ssim_map(x, y).numpy()
    assert np.abs(got - want).max() <= BOUNDS[name][1], np.abs(got - want).max()
    err_img = np.abs(got.reshape(B, -1).astype(np.float64).mean(1) - want.reshape(B, -1).mean(1)).max()
    assert err_img <= BOUNDS[name][2], err_img
    if name.startswith('same'):
        assert (got == 1).all()                                               # no FMA in the formula: exactly 1


def test_workspace_bytes_and_the_c_abi_checks():
    from dbw_b200 import _lib, metrics
    L = _lib.lib()
    assert hasattr(L, 'dbw_image_scores') and hasattr(L, 'dbw_image_scores_workspace_bytes')
    # 8 bytes x 2 sums per (32 x 32 output tile, view)
    assert L.dbw_image_scores_workspace_bytes(1, 11, 11) == 16
    assert L.dbw_image_scores_workspace_bytes(2, 42, 74) == 2 * 2 * 16             # 32 x 64 outputs: two tiles
    assert L.dbw_image_scores_workspace_bytes(3, 43, 43) == 3 * 4 * 16             # 33 x 33 outputs: 2 x 2 tiles
    assert L.dbw_image_scores_workspace_bytes(4, 576, 768) == 4 * 18 * 24 * 16
    for bad in ((1, 10, 11), (1, 11, 10), (0, 64, 64), (-1, 64, 64), (65536, 64, 64)):
        assert L.dbw_image_scores_workspace_bytes(*bad) == 0, bad
    fake, ws = ctypes.c_void_p(256), ctypes.c_void_p(512)                         # never dereferenced: the checks fail first
    win = metrics._WINDOW
    assert L.dbw_image_scores(1, 10, 64, fake, fake, win, fake, fake, ws, 1 << 20, None) != 0
    assert b'11' in L.dbw_last_error()
    assert L.dbw_image_scores(1, 64, 64, None, fake, win, fake, fake, ws, 1 << 20, None) != 0
    assert b'null' in L.dbw_last_error()
    assert L.dbw_image_scores(1, 64, 64, fake, fake, None, fake, fake, ws, 1 << 20, None) != 0
    assert L.dbw_image_scores(2, 64, 64, fake, fake, win, fake, fake, ws, 8 * 4 * 2 * 2 - 1, None) != 0
    assert b'workspace' in L.dbw_last_error()


def test_python_checks_raise_before_any_launch():
    from dbw_b200 import metrics
    from dbw_b200._lib import DbwError
    a = torch.rand(2, 3, 16, 16)
    with pytest.raises(DbwError, match='CUDA'):                                  # no CPU fallback
        metrics.image_scores(a, a)
    with pytest.raises(DbwError, match='CUDA'):
        metrics.ssim(a, a)
    with pytest.raises(DbwError, match='CUDA'):
        metrics.psnr(a, a)
    for bad_x, bad_y in ((torch.rand(2, 4, 16, 16),) * 2, (a, torch.rand(2, 3, 16, 17)), (a[0], a[0]),
                         (torch.rand(0, 3, 16, 16),) * 2):
        with pytest.raises(ValueError, match='B,3,H,W'):
            metrics.image_scores(bad_x, bad_y)
    for H, W in ((10, 16), (16, 10), (10, 10)):
        b = torch.rand(1, 3, H, W)
        with pytest.raises(ValueError, match='at least 11'):
            metrics.image_scores(b, b)
