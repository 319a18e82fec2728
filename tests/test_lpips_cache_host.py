"""CPU: the LPIPS target cache's lookup math (csrc/dbw_lpips_cache.cuh compiled for the host) against a numpy
restatement -- the fingerprint, the candidate search with its bitwise confirmation, the route and miss compaction -- the
arena size against the tap shapes, and the C-ABI checks of the cache entries without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1


def fmix64(k):
    k = np.asarray(k, np.uint64)
    with np.errstate(over='ignore'):
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xff51afd7ed558ccd)
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xc4ceb9fe1a85ec53)
        k = k ^ (k >> np.uint64(33))
    return k


def fingerprint_np(img):
    """sum_i fmix64((i << 32) | bits_i) mod 2^64 over the image's floats in NCHW order"""
    u = np.ascontiguousarray(img, np.float32).reshape(-1).view(np.uint32).astype(np.uint64)
    i = np.arange(u.size, dtype=np.uint64)
    return int(sum(int(v) for v in fmix64((i << np.uint64(32)) | u))) & M64


def route_np(q_fp, q_img, c_fp, c_img):
    """(route (B,2), n_miss): the first cache entry with the same fingerprint AND the same bits, misses numbered in order"""
    B = len(q_fp)
    hit = [next((e for e in range(len(c_fp)) if c_fp[e] == q_fp[b] and np.array_equal(q_img[b].view(np.uint32),
                                                                                           c_img[e].view(np.uint32))), -1)
           for b in range(B)]
    route = np.full((B, 2), -1, np.int32)
    s = 0
    for b in range(B):
        if hit[b] >= 0:
            route[b, 0] = hit[b]
        else:
            route[b, 0], route[s, 1] = -(s + 1), b
            s += 1
    return route, s


@pytest.fixture(scope='module')
def hc(tmp_path_factory):
    so = str(tmp_path_factory.mktemp('lpips_cache_host') / 'libdbw_lpips_cache_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_lpips_cache_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.hc_fingerprint.restype = None
    L.hc_fingerprint.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]
    L.hc_lookup.restype = ctypes.c_int
    L.hc_lookup.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                            ctypes.c_int64, ctypes.c_void_p]
    return L


def _fp(hc, imgs):
    out = np.zeros(len(imgs), np.uint64)
    imgs = np.ascontiguousarray(imgs, np.float32)
    hc.hc_fingerprint(imgs.ctypes.data, imgs[0].size, len(imgs), out.ctypes.data)
    return out


def _lookup(hc, q_fp, q_img, c_fp, c_img):
    q_img, c_img = np.ascontiguousarray(q_img, np.float32), np.ascontiguousarray(c_img, np.float32)
    q_fp, c_fp = np.ascontiguousarray(q_fp, np.uint64), np.ascontiguousarray(c_fp, np.uint64)
    route = np.full((len(q_fp), 2), 12345, np.int32)
    n_miss = hc.hc_lookup(q_fp.ctypes.data, q_img.ctypes.data, len(q_fp), c_fp.ctypes.data, c_img.ctypes.data, len(c_fp),
                          q_img[0].size, route.ctypes.data)
    return route, n_miss


def test_fingerprint_is_the_numpy_restatement(hc):
    rng = np.random.default_rng(0)
    imgs = rng.random((3, 3, 7, 11), np.float32)
    imgs[2] = imgs[0]
    imgs[2, 1, 3, 4] = np.nextafter(imgs[0, 1, 3, 4], np.float32(2))       # one bit apart
    fp = _fp(hc, imgs)
    assert [int(v) for v in fp] == [fingerprint_np(x) for x in imgs]
    assert len(set(int(v) for v in fp)) == 3
    # position matters: two images with two values swapped differ
    sw = imgs[0].copy()
    sw.reshape(-1)[[0, 1]] = sw.reshape(-1)[[1, 0]]
    assert int(_fp(hc, sw[None])[0]) != int(fp[0])
    assert int(_fp(hc, np.zeros((1, 3, 4, 4), np.float32))[0]) == fingerprint_np(np.zeros((3, 4, 4), np.float32))


@pytest.mark.parametrize('case', ['mixed', 'all_hit', 'all_miss', 'duplicates', 'collisions', 'one_bit'])
def test_lookup_and_route_are_the_numpy_restatement(hc, case):
    rng = np.random.default_rng(len(case))
    N, B = 5, 9
    cache = rng.random((N, 3, 6, 5), np.float32)
    other = rng.random((B, 3, 6, 5), np.float32)
    if case == 'mixed':
        pick = rng.integers(0, 2, B).astype(bool)
        q = np.where(pick[:, None, None, None], cache[rng.integers(0, N, B)], other)
    elif case == 'all_hit':
        q = cache[rng.permutation(np.arange(B) % N)]
    elif case == 'all_miss':
        q = other
    elif case == 'duplicates':
        q = np.stack([cache[2], other[0], cache[2], cache[2], other[0], cache[4], other[1], cache[4], cache[2]])
    elif case == 'collisions':
        q = np.stack([cache[1], other[0], cache[3], other[1], cache[0], cache[1], other[2], other[3], cache[4]])
    else:
        q = cache[np.arange(B) % N].copy()
        q[3, 2, 1, 1] = np.nextafter(q[3, 2, 1, 1], np.float32(0))
    c_fp, q_fp = _fp(hc, cache), _fp(hc, q)
    if case == 'collisions':                 # a stub hash: every fingerprint equal, only the bitwise comparison decides
        c_fp[:], q_fp[:] = 7, 7
    route, n_miss = _lookup(hc, q_fp, q, c_fp, cache)
    want, want_miss = route_np([int(v) for v in q_fp], q, [int(v) for v in c_fp], cache)
    assert n_miss == want_miss and np.array_equal(route, want), (route, want)
    hits = route[:, 0] >= 0
    for b in range(B):                       # every hit is the same bits; every miss slot points back at its image
        if hits[b]:
            assert np.array_equal(q[b].view(np.uint32), cache[route[b, 0]].view(np.uint32))
        else:
            assert route[-route[b, 0] - 1, 1] == b
    assert (route[n_miss:, 1] == -1).all()
    if case == 'all_hit':
        assert n_miss == 0
    if case in ('all_miss', 'one_bit'):
        assert n_miss == (B if case == 'all_miss' else 1)


def test_first_of_equal_entries_wins(hc):
    rng = np.random.default_rng(5)
    cache = rng.random((4, 3, 4, 4), np.float32)
    cache[3] = cache[1]
    route, n_miss = _lookup(hc, _fp(hc, cache[[3, 1]]), cache[[3, 1]], _fp(hc, cache), cache)
    assert n_miss == 0 and route[:, 0].tolist() == [1, 1]


@pytest.mark.parametrize('H,W', [(300, 400), (576, 768), (37, 50), (16, 16), (17, 23)])
def test_arena_bytes_are_the_tap_shapes(H, W):
    from dbw_b200.perceptual import LPIPS
    m = LPIPS()
    taps = sum((H >> k) * (W >> k) * c for k, c in enumerate((64, 128, 256, 512, 512))) * 4
    per = taps + 8 + 3 * H * W * 4                        # the taps, a fingerprint, a copy of the image
    assert m.target_cache_bytes(H, W) == per
    assert m.target_cache_bytes(H, W, N=49) == 49 * per
    if (H, W) == (300, 400):
        assert taps == 58_470_400 and 59.9e6 < per < 60e6 and 2.93e9 < 49 * per < 2.94e9
    if (H, W) == (576, 768):
        assert 221e6 < per < 222e6


def test_cache_c_abi_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    b = ctypes.c_size_t(0)
    assert L.dbw_lpips_cache_bytes(15, 64, ctypes.byref(b)) != 0 and b'bad sizes' in L.dbw_last_error()
    assert L.dbw_lpips_cache_bytes(64, 64, None) != 0 and b'null pointer' in L.dbw_last_error()
    assert L.dbw_lpips_cache_bytes(64, 64, ctypes.byref(b)) == 0
    net = _lib.DbwLpipsNet()
    for f in ('conv_w', 'conv_b', 'lin_w'):
        arr = getattr(net, f)
        for i in range(len(arr)):
            arr[i] = 256                                   # non-null: the checks below fail before anything is launched
    net.shift = net.scale = net.prepared = 256
    cache = _lib.DbwLpipsTargetCache(256, 4, 48, 64, 1)
    p = ctypes.c_void_p(256)
    # registration
    assert L.dbw_lpips_cache_targets(ctypes.byref(net), p, None, 2, p, 1 << 40, None) != 0
    assert b'null pointer' in L.dbw_last_error()
    assert L.dbw_lpips_cache_targets(ctypes.byref(net), p, ctypes.byref(cache), 0, p, 1 << 40, None) != 0
    assert b'bad sizes' in L.dbw_last_error()
    assert L.dbw_lpips_cache_targets(ctypes.byref(net), None, ctypes.byref(cache), 2, p, 1 << 40, None) != 0
    empty = _lib.DbwLpipsTargetCache(256, 0, 48, 64, 1)
    assert L.dbw_lpips_cache_targets(ctypes.byref(net), p, ctypes.byref(empty), 2, p, 1 << 40, None) != 0
    assert L.dbw_lpips_cache_targets(ctypes.byref(net), p, ctypes.byref(cache), 2, p, 16, None) != 0
    assert b'workspace too small' in L.dbw_last_error()
    # the cached forward and backward: sizes, null pointers, then the cache against the call
    fwd = lambda c, H, W, norm, route=p: L.dbw_lpips_forward_cached(ctypes.byref(net), c, p, p, 2, H, W, norm, 0, 1, p, p, route,
                                                                     None, p, 1 << 40, None)
    assert fwd(ctypes.byref(cache), 8, 64, 1) != 0 and b'bad sizes' in L.dbw_last_error()
    assert fwd(ctypes.byref(cache), 48, 64, 1, route=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert fwd(None, 48, 64, 1) != 0 and b'bad cache' in L.dbw_last_error()
    assert fwd(ctypes.byref(cache), 48, 96, 1) != 0 and b'bad cache' in L.dbw_last_error()         # another W
    assert fwd(ctypes.byref(cache), 32, 64, 1) != 0 and b'bad cache' in L.dbw_last_error()         # another H
    assert fwd(ctypes.byref(cache), 48, 64, 0) != 0 and b'bad cache' in L.dbw_last_error()         # another normalize
    assert fwd(ctypes.byref(empty), 48, 64, 1) != 0 and b'bad cache' in L.dbw_last_error()
    bwd = lambda c, H, W, route=p: L.dbw_lpips_backward_cached(ctypes.byref(net), c, route, p, 2, H, W, 1, 0, p, p, 1 << 40, None)
    assert bwd(ctypes.byref(cache), 48, 64, route=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert bwd(ctypes.byref(cache), 48, 80) != 0 and b'bad cache' in L.dbw_last_error()
    assert bwd(None, 48, 64) != 0 and b'bad cache' in L.dbw_last_error()
    assert ctypes.sizeof(_lib.DbwLpipsTargetCache) == 32


def test_model_refuses_to_cache_for_another_perceptual_term():
    import torch
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from tests.test_model_gpu import CFG
    from copy import deepcopy
    model = DifferentiableBlocksWorld((48, 64), **deepcopy(CFG))
    model.set_perceptual_loss(lambda imgs, rec: (imgs - rec).abs().mean())
    with pytest.raises(TypeError, match='not PerceptualTerm'):
        model.cache_perceptual_targets(torch.zeros(2, 3, 48, 64))
