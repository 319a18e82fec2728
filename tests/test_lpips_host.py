"""CPU: the LPIPS module's state-dict names and constructors, the input-gradient weight layout, the dropout hash (the
device header compiled for the host against the numpy restatement of oracle/lpips.py) and the C-ABI checks of
dbw_lpips_* without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lpips as OL

HERE = os.path.dirname(os.path.abspath(__file__))


def _want_keys():
    keys = {'scaling_layer.shift': (1, 3, 1, 1), 'scaling_layer.scale': (1, 3, 1, 1)}
    for s, idx, chans in ((1, (0, 2), (3, 64, 64)), (2, (5, 7), (64, 128, 128)), (3, (10, 12, 14), (128, 256, 256, 256)),
                          (4, (17, 19, 21), (256, 512, 512, 512)), (5, (24, 26, 28), (512, 512, 512, 512))):
        for j, i in enumerate(idx):
            keys[f'net.slice{s}.{i}.weight'] = (chans[j + 1], chans[j], 3, 3)
            keys[f'net.slice{s}.{i}.bias'] = (chans[j + 1],)
    for k, c in enumerate((64, 128, 256, 512, 512)):
        keys[f'lin{k}.model.1.weight'] = (1, c, 1, 1)
        keys[f'lins.{k}.model.1.weight'] = (1, c, 1, 1)
    return keys


def test_state_dict_names_and_shapes_are_lpips():
    from dbw_b200.perceptual import LPIPS
    sd = LPIPS().state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == _want_keys()
    assert torch.equal(sd['scaling_layer.shift'].flatten(), torch.tensor([-.030, -.088, -.188]))
    assert torch.equal(sd['scaling_layer.scale'].flatten(), torch.tensor([.458, .448, .450]))
    assert not any(p.requires_grad for p in LPIPS().parameters())


def test_from_state_dict_strips_prefixes_and_raises_on_bad_keys():
    from dbw_b200.dbw import PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    sd = OL.random_state_dict(1)
    wrapped = {'perceptual_loss.loss.' + k: v for k, v in sd.items() if not k.startswith('lins.')}
    wrapped['blocks.something'] = torch.zeros(3)                    # the rest of a model_state
    m = LPIPS.from_state_dict(wrapped)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    term = PerceptualTerm(m)
    assert set(term.state_dict()) == {'loss.' + k for k in _want_keys()}
    assert LPIPS.from_state_dict({'module.' + k: v for k, v in sd.items()}).state_dict().keys() == sd.keys()
    bad = dict(sd)
    del bad['net.slice3.12.bias']
    with pytest.raises(KeyError):
        LPIPS.from_state_dict(bad)
    bad = dict(sd)
    bad['net.slice3.12.weight'] = torch.zeros(256, 256, 1, 1)
    with pytest.raises(ValueError):
        LPIPS.from_state_dict(bad)


def test_from_files_renames_torchvision_and_lpips_weights(tmp_path):
    from torchvision.models import vgg16
    from dbw_b200.perceptual import LPIPS
    torch.manual_seed(3)
    tv = vgg16(weights=None).state_dict()                            # features.N.* and classifier.*
    lin = {f'lin{k}.model.1.weight': torch.randn(1, c, 1, 1).abs() for k, c in enumerate((64, 128, 256, 512, 512))}
    torch.save(tv, tmp_path / 'vgg16.pth')
    torch.save(lin, tmp_path / 'vgg.pth')
    m = LPIPS.from_files(tmp_path / 'vgg16.pth', tmp_path / 'vgg.pth')
    sd = m.state_dict()
    for s, i in ((1, 0), (2, 7), (3, 14), (4, 17), (5, 28)):
        assert torch.equal(sd[f'net.slice{s}.{i}.weight'], tv[f'features.{i}.weight'])
        assert torch.equal(sd[f'net.slice{s}.{i}.bias'], tv[f'features.{i}.bias'])
    for k in range(5):
        assert torch.equal(sd[f'lins.{k}.model.1.weight'], lin[f'lin{k}.model.1.weight'])
    del tv['features.26.bias']
    torch.save(tv, tmp_path / 'broken.pth')
    with pytest.raises(KeyError):
        LPIPS.from_files(tmp_path / 'broken.pth', tmp_path / 'vgg.pth')


@pytest.mark.parametrize('ci,co', [(64, 64), (64, 128), (256, 512), (3, 64)])
def test_dgrad_weights_are_the_input_gradient(ci, co):
    from dbw_b200.perceptual import dgrad_weight, kmajor
    g = torch.Generator().manual_seed(ci + co)
    w = torch.randn(co, ci, 3, 3, generator=g, dtype=torch.float64)
    gy = torch.randn(2, co, 9, 7, generator=g, dtype=torch.float64)
    want = torch.nn.grad.conv2d_input((2, ci, 9, 7), w, gy, padding=1)
    got = F.conv2d(gy, dgrad_weight(w), padding=1)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    # the K-major operand: column (ky*3 + kx)*C_in + ci of row co
    km = kmajor(w)
    assert km.shape == (co, 9 * ci) and km[5, (2 * 3 + 1) * ci + 2] == w[5, 2, 2, 1]


def test_tf32_rounding_is_nearest_ties_away():
    from dbw_b200.perceptual import tf32_round
    one_ulp = 2.0 ** -10                                            # TF32 spacing at 1
    x = torch.tensor([1.0, 1 + one_ulp / 2, 1 + one_ulp / 2 - 2 ** -23, -(1 + one_ulp / 2), 1 + 3 * one_ulp / 2], dtype=torch.float32)
    assert tf32_round(x).tolist() == [1.0, 1 + one_ulp, 1.0, -(1 + one_ulp), 1 + 2 * one_ulp]
    r = tf32_round(torch.randn(10000))
    assert not (r.view(torch.int32) & 0x1fff).any()
    assert torch.equal(OL.tf32(r.double()), r.double())


@pytest.fixture(scope='module')
def hl(tmp_path_factory):
    so = str(tmp_path_factory.mktemp('lpips_host') / 'libdbw_lpips_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_lpips_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.hl_mask.restype = None
    L.hl_mask.argtypes = [ctypes.c_uint32, ctypes.c_uint32] + [ctypes.c_int] * 4 + [ctypes.c_void_p]
    return L


@pytest.mark.parametrize('seed,tap,shape', [(0, 0, (2, 64, 17, 23)), (0xfffffffe, 4, (3, 512, 1, 1)),
                                            (12345, 2, (1, 256, 75, 100))])
def test_numpy_mask_is_the_device_hash(hl, seed, tap, shape):
    out = np.empty(shape, np.uint8)
    hl.hl_mask(seed, tap, *shape, out.ctypes.data)
    assert np.array_equal(OL.mask_np(seed, tap, *shape), out * 2.0)


def test_mask_keep_rate_and_independence():
    m = OL.mask_np(7, 1, 4, 128, 40, 50) / 2                        # 1.024e6 Bernoulli(1/2) draws
    n = m.size
    assert abs(m.mean() - 0.5) < 3 * 0.5 / np.sqrt(n)
    # neighbouring channels, pixels, images, taps and seeds are not correlated
    for a, b in ((m[:, 1:], m[:, :-1]), (m[:, :, :, 1:], m[:, :, :, :-1]), (m[1:], m[:-1])):
        assert abs((a == b).mean() - 0.5) < 3 * 0.5 / np.sqrt(a.size)
    for other in (OL.mask_np(7, 2, 4, 128, 40, 50) / 2, OL.mask_np(8, 1, 4, 128, 40, 50) / 2):
        assert abs((other == m).mean() - 0.5) < 3 * 0.5 / np.sqrt(n)


def test_lpips_c_abi_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    ws, prep = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert ctypes.sizeof(_lib.DbwLpipsNet) == 34 * 8
    assert L.dbw_lpips_workspace_bytes(1, 15, 64, 1, ctypes.byref(ws), ctypes.byref(prep)) != 0 and b'bad sizes' in L.dbw_last_error()
    assert L.dbw_lpips_workspace_bytes(0, 64, 64, 1, ctypes.byref(ws), ctypes.byref(prep)) != 0
    assert L.dbw_lpips_workspace_bytes(1, 400, 400, 1, ctypes.byref(ws), ctypes.byref(prep)) == 0
    ws_fwd = ctypes.c_size_t(0)
    assert L.dbw_lpips_workspace_bytes(1, 400, 400, 0, ctypes.byref(ws_fwd), ctypes.byref(prep)) == 0
    acts = sum(c * (400 >> lv) ** 2 for c, lv in ((64, 0), (64, 0), (128, 1), (128, 1), (256, 2), (256, 2), (256, 2),
                                                  (512, 3), (512, 3), (512, 3), (512, 4), (512, 4), (512, 4))) * 4
    taps = sum(c * (400 >> lv) ** 2 for lv, c in enumerate((64, 128, 256, 512, 512))) * 4
    scratch = 2 * 400 * 400 * 64 * 4
    assert acts + taps + scratch < ws.value < acts + taps + scratch + 2 ** 20  # rec's activations, imgs' taps, scratch
    assert 172e6 < acts < 174e6                                             # ~173 MB per 400x400 view
    # without a backward to follow, rec keeps only its taps, like imgs
    assert 2 * taps + scratch < ws_fwd.value < 2 * taps + scratch + 2 ** 20
    n_w = sum(9 * ci * co for ci, co in ((64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512),
                                         (512, 512), (512, 512), (512, 512), (512, 512), (512, 512)))
    assert prep.value == 2 * n_w * 4
    net = _lib.DbwLpipsNet()
    assert L.dbw_lpips_forward(ctypes.byref(net), None, None, 1, 32, 32, 1, 0, 1, None, None, None, 0, None) != 0
    assert b'null pointer' in L.dbw_last_error()
    assert L.dbw_lpips_backward(ctypes.byref(net), None, 1, 32, 32, 1, 0, None, None, 0, None) != 0
    assert L.dbw_lpips_prepare_weights(None, None) != 0
    assert L.dbw_lpips_conv3x3(None, None, None, None, None, 1, 8, 8, 48, 64, 1, None) != 0 and b'bad sizes' in L.dbw_last_error()
    assert L.dbw_lpips_conv3x3(None, None, None, None, None, 1, 8, 8, 64, 192, 1, None) != 0
    assert L.dbw_lpips_maxpool(None, None, 1, 8, 8, 6, None) != 0


def test_lpips_module_refuses_what_it_does_not_implement():
    from dbw_b200._lib import DbwError
    from dbw_b200.perceptual import LPIPS
    m = LPIPS()
    x = torch.zeros(1, 3, 32, 32)
    with pytest.raises(DbwError):
        m(x, x)                                                               # CPU: no fallback
    with pytest.raises(DbwError):
        m(x.requires_grad_(True), x.detach())                                 # no gradient to in0
