"""CPU: cell maps (DbwMapDesc.reserved = DBW_MAP_CELLS(f, p_left)).  The raster kernels sample a box-decimated texture at its
f x f cells instead of at the atlas that repeats every cell over f x f texels and the circular padding; tap_to_cells
(csrc/dbw_math.cuh, compiled for the host by tests/host_math/dbw_cells_host.cpp) maps each bilinear tap of the logical atlas to
its cell.  Checked here against a torch expansion of random cells -- nearest upsampling + circular u padding, what
DBW_TEX_STAGE_EXPAND writes: every tap must read exactly the value its atlas texel holds, so renders stay bit-identical."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'host_math', 'dbw_cells_host.cpp')


@pytest.fixture(scope='module')
def hc():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_cells_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', '-Wno-unknown-pragmas', SRC, '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _expand(cells, f, p_left, p_right):
    """(M, CS, CS, 3) cells -> (M, TS, p_left + TS + p_right, 3) atlas: nearest upsample, circular padding along u"""
    up = F.interpolate(cells.permute(0, 3, 1, 2), scale_factor=f, mode='nearest')
    if p_left or p_right:
        up = F.pad(up, (p_left, p_right, 0, 0), mode='circular')
    return up.permute(0, 2, 3, 1).contiguous()


def _uv(n, seed):
    """random (u, v) plus the borders, the corners, the texel centres next to them and points outside [0, 1]"""
    g = np.random.default_rng(seed)
    uv = g.uniform(-0.05, 1.05, size=(n, 2))
    edge = np.array([0.0, 1.0, 1e-7, 1 - 1e-7, 0.5, -0.2, 1.2])
    grid = np.stack(np.meshgrid(edge, edge), -1).reshape(-1, 2)
    return np.ascontiguousarray(np.concatenate([uv, grid, g.uniform(0, 1, size=(n, 1)) * [1, 0], g.uniform(0, 1, size=(n, 1)) * [0, 1] + [1, 0]]),
                                dtype=np.float32)


@pytest.mark.parametrize('TS,p_left,p_right', [(256, 0, 0), (128, 0, 0), (256, 3, 5), (128, 3, 5), (128, 128, 128), (64, 1, 0)])
def test_cell_taps_read_what_the_expanded_atlas_holds(hc, TS, p_left, p_right):
    f, M = 8, 3
    CS, W = TS // f, TS + p_left + p_right
    g = torch.Generator().manual_seed(TS + p_left)
    cells = torch.rand(M, CS, CS, 3, generator=g)
    atlas = _expand(cells, f, p_left, p_right)
    assert atlas.shape == (M, TS, W, 3)
    flat_atlas, flat_cells = atlas.reshape(-1, 3).numpy(), cells.reshape(-1, 3).numpy()
    uv = _uv(4000, TS)
    n = len(uv)
    code = (p_left << 8) | f
    for m in range(M):
        texel, cell = np.empty((n, 4), np.int32), np.empty((n, 4), np.int32)
        w = np.empty((n, 4), np.float32)
        hc.hc_taps(_p(uv), n, m * TS * W, m * CS * CS, TS, W, code, _p(texel), _p(cell), _p(w))
        assert np.array_equal(texel < 0, cell < 0)                        # border taps stay absent, the others present
        assert (texel[:, 0] >= 0).all()
        ok = texel >= 0
        assert (cell[ok] >= m * CS * CS).all() and (cell[ok] < (m + 1) * CS * CS).all()
        assert np.array_equal(flat_atlas[texel[ok]], flat_cells[cell[ok]])  # bit for bit the value the atlas texel holds
        # the bilinear colour, written as the kernels write it, is identical too
        a = np.where(ok[..., None], flat_atlas[np.maximum(texel, 0)], 0).astype(np.float32)
        c = np.where(ok[..., None], flat_cells[np.maximum(cell, 0)], 0).astype(np.float32)
        col = lambda t: ((t[:, 0] * w[:, :1] + t[:, 1] * w[:, 1:2]) + t[:, 2] * w[:, 2:3]) + t[:, 3] * w[:, 3:4]
        assert np.array_equal(col(a), col(c))


def test_padded_columns_wrap_around(hc):
    """u at the first / last atlas columns (the circular padding) lands on the last / first source cell columns"""
    TS, f, p_left, p_right = 128, 8, 3, 5
    W, CS = TS + p_left + p_right, TS // f
    x = np.array([0.25, 1.25, 2.25, p_left + 0.25, W - p_right + 0.25, W - 1], np.float32)      # atlas columns (+ a quarter texel)
    uv = np.ascontiguousarray(np.stack([x / (W - 1), np.full_like(x, 0.5)], 1), dtype=np.float32)
    n = len(uv)
    texel, cell = np.empty((n, 4), np.int32), np.empty((n, 4), np.int32)
    w = np.empty((n, 4), np.float32)
    hc.hc_taps(_p(uv), n, 0, 0, TS, W, (p_left << 8) | f, _p(texel), _p(cell), _p(w))
    col = cell[:, 0] % CS
    assert list(col) == [CS - 1, CS - 1, CS - 1, 0, 0, (p_right - 1) // f]
