"""CPU: the VGG16 feature-reconstruction loss (perceptual.PerceptualLoss, dbw_vgg_loss_* of csrc/dbw_lpips.cu) without a GPU.
The float64 oracle against the reference's own forward frozen in tests/golden/vgg_perceptual.npz, the module's names and
constructors, the model's wiring without the ImageNet weights, the options struct's C layout and the C-ABI checks."""
import ctypes
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import _vgg_oracle as OV
from tests.golden.make_vgg_perceptual_golden import StandIn, weight_checksum

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'vgg_perceptual.npz')


@pytest.fixture(scope='module')
def golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


@pytest.fixture(scope='module')
def sd(golden):
    sd = OV.random_state_dict(json.loads(str(golden['meta']))['weight_seed'])
    assert np.allclose(weight_checksum(sd), golden['weight_checksum'], rtol=1e-12, atol=0)    # the frozen weights
    return sd


@pytest.mark.parametrize('shape', [0, 1])
@pytest.mark.parametrize('name', list(OV.OPTION_SETS))
def test_oracle_reproduces_the_reference_forward(golden, sd, name, shape):
    imgs, rec = (torch.from_numpy(golden[f's{shape}__{k}']) for k in ('imgs', 'rec'))
    o = OV.options(**OV.OPTION_SETS[name])
    B = imgs.shape[0]
    v, g = OV.value_and_grad(sd, imgs, rec, **o, grad_value=torch.full((B,), 1.0 / B))
    want_v = float(golden[f's{shape}__{name}__value'])
    want_g = torch.from_numpy(golden[f's{shape}__{name}__grad']).double()
    assert abs(float(v.mean()) - want_v) <= 1e-5 * abs(want_v), (name, float(v.mean()), want_v)
    assert float((g - want_g).norm() / want_g.norm()) < 1e-4


def test_state_dict_names_and_shapes_are_the_references():
    from dbw_b200.perceptual import PerceptualLoss
    ref = StandIn(OV.random_state_dict(0))
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    for kw in ({}, dict(feature_levels=[1]), dict(feature_levels=[2, 5], sum_channels=True)):
        m = PerceptualLoss(**kw)
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == want
        assert list(m.state_dict()) == list(ref.state_dict())
        assert not any(p.requires_grad for p in m.parameters())
    assert torch.equal(m.mean_rgb, ref.mean_rgb) and torch.equal(m.std_rgb, ref.std_rgb)
    with pytest.raises(NotImplementedError):
        PerceptualLoss(requires_grad=True)


def test_a_model_state_with_the_prefix_loads(tmp_path):
    from dbw_b200.perceptual import PerceptualLoss
    sd = OV.random_state_dict(1)
    state = {'perceptual_loss.' + k: v for k, v in sd.items()}
    state['blocks.something'] = torch.zeros(3)                       # the rest of a model_state
    m = PerceptualLoss.from_state_dict(state, feature_levels=[2, 4], sum_channels=True)
    assert m.feature_levels == [2, 4] and m.sum_channels
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    holder = torch.nn.Module()
    holder.perceptual_loss = m
    assert set(holder.state_dict()) == set(state) - {'blocks.something'}
    bad = dict(sd)
    del bad['slice3.12.bias']
    with pytest.raises(KeyError):
        PerceptualLoss.from_state_dict(bad)
    bad = dict(sd)
    bad['slice5.28.weight'] = torch.zeros(512, 512, 1, 1)
    with pytest.raises(ValueError):
        PerceptualLoss.from_state_dict(bad)
    # torchvision's file
    from torchvision.models import vgg16
    torch.manual_seed(4)
    tv = vgg16(weights=None).state_dict()
    torch.save(tv, tmp_path / 'vgg16.pth')
    m = PerceptualLoss.from_files(tmp_path / 'vgg16.pth', feature_levels=[1, 2])
    for s, i in ((1, 0), (2, 7), (3, 14), (4, 17), (5, 28)):
        assert torch.equal(m.state_dict()[f'slice{s}.{i}.weight'], tv[f'features.{i}.weight'])
    assert m.feature_levels == [1, 2]


def test_make_perceptual_without_the_weights_warns_and_never_downloads(tmp_path, monkeypatch):
    import urllib.request
    from dbw_b200 import dbw
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path))

    def no_network(*a, **k):
        raise AssertionError('network access')
    monkeypatch.setattr(urllib.request, 'urlopen', no_network)
    monkeypatch.setattr(torch.hub, 'download_url_to_file', no_network)
    with pytest.warns(RuntimeWarning, match='DROPPED'):
        assert dbw._make_perceptual('perceptual') is None
    # with the file in the hub cache: the module, unwrapped
    from torchvision.models import vgg16
    (tmp_path / 'checkpoints').mkdir()
    torch.save(vgg16(weights=None).state_dict(), tmp_path / 'checkpoints' / 'vgg16-397923af.pth')
    from dbw_b200.perceptual import PerceptualLoss
    m = dbw._make_perceptual('perceptual')
    assert type(m) is PerceptualLoss and m.feature_levels == [3]


def test_module_refuses_what_it_does_not_implement():
    from dbw_b200._lib import DbwError
    from dbw_b200.perceptual import PerceptualLoss
    m = PerceptualLoss()
    x = torch.zeros(1, 3, 32, 32)
    with pytest.raises(DbwError):
        m(x, x)                                                      # CPU: no fallback
    with pytest.raises(DbwError):
        m(x.clone().requires_grad_(True), x)                         # no gradient to imgs
    with pytest.raises(DbwError):
        PerceptualLoss(feature_levels=[0, 3])
    with pytest.raises(DbwError):
        PerceptualLoss(feature_levels=[])


def test_cache_perceptual_targets_refuses_this_term():
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.perceptual import PerceptualLoss
    from types import SimpleNamespace
    with pytest.raises(TypeError):
        DifferentiableBlocksWorld.cache_perceptual_targets(SimpleNamespace(perceptual_loss=PerceptualLoss()), torch.zeros(1, 3, 16, 16))


def test_options_struct_has_the_c_layout(tmp_path):
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    cls = _lib.DbwVggLossOptions
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(DbwVggLossOptions));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DbwVggLossOptions, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls) == 16
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _ws(L, B, H, W, levels, save=1, **kw):
    from dbw_b200 import _lib
    o = _lib.DbwVggLossOptions(levels, kw.get('ni', 1), kw.get('nf', 1), kw.get('sc', 0))
    n = ctypes.c_size_t(0)
    return L.dbw_vgg_loss_workspace_bytes(B, H, W, ctypes.byref(o), save, ctypes.byref(n)), n.value


def test_vgg_loss_c_abi_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    # the default relu3_3 at 400x400: rec's 7 activations, imgs' one tap, two scratch tensors, partials and constants
    rc, ws = _ws(L, 1, 400, 400, 0b100)
    assert rc == 0
    acts = sum(c * (400 >> lv) ** 2 for c, lv in ((64, 0), (64, 0), (128, 1), (128, 1), (256, 2), (256, 2), (256, 2))) * 4
    tap = 256 * 100 * 100 * 4
    scratch = 2 * 400 * 400 * 64 * 4
    assert acts + tap + scratch < ws < acts + tap + scratch + 2 ** 16
    rc, ws_fwd = _ws(L, 1, 400, 400, 0b100, save=0)
    assert rc == 0 and 2 * tap + scratch < ws_fwd < 2 * tap + scratch + 2 ** 16
    lp, prep = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert L.dbw_lpips_workspace_bytes(1, 400, 400, 1, ctypes.byref(lp), ctypes.byref(prep)) == 0
    # all five levels: LPIPS's layout with the 2568 constants (2624 floats aligned) in place of its 64-float seed region
    assert _ws(L, 1, 400, 400, 0b11111)[1] == lp.value + (2624 - 64) * 4
    assert _ws(L, 1, 400, 400, 0b01010)[1] < _ws(L, 1, 400, 400, 0b11010)[1]
    # levels 0 and >= 32, and images below what the deepest level needs, fail loudly
    for levels in (0, 32, 64, -1):
        assert _ws(L, 1, 64, 64, levels)[0] != 0 and b'bad options' in L.dbw_last_error()
    for levels, size in ((0b1, 1), (0b100, 4), (0b10000, 16), (0b10001, 16)):
        assert _ws(L, 1, size, size, levels)[0] == 0
        assert _ws(L, 1, size - 1, size, levels)[0] != 0 if size > 1 else _ws(L, 1, 0, size, levels)[0] != 0
        assert _ws(L, 1, size, size - 1, levels)[0] != 0 if size > 1 else True
    assert _ws(L, 0, 64, 64, 0b100)[0] != 0
    assert L.dbw_vgg_loss_workspace_bytes(1, 64, 64, None, 1, ctypes.byref(ctypes.c_size_t(0))) != 0
    o = _lib.DbwVggLossOptions(0b100, 1, 1, 0)
    net = _lib.DbwLpipsNet()
    assert L.dbw_vgg_loss_forward(ctypes.byref(net), ctypes.byref(o), None, None, 1, 32, 32, 1, None, None, 0, None) != 0
    assert b'null pointer' in L.dbw_last_error()
    assert L.dbw_vgg_loss_backward(ctypes.byref(net), ctypes.byref(o), None, 1, 32, 32, None, None, 0, None) != 0
    assert b'null pointer' in L.dbw_last_error()
