"""CPU: the optimiser (dbw_b200/optim.py, csrc/dbw_optim.cu).

1. The C-ABI: ctypes mirrors of DbwAdamSegment / DbwAdamGroup have gcc's layout, and dbw_adam_step validates its arguments
   without a GPU.
2. The per-element update of csrc/dbw_optim_math.cuh compiled for the host (tests/host_math/dbw_optim_host.cpp) against a
   float64 restatement and against torch.optim.Adam(foreach=False) on CPU fp32: two groups, weight decay, a skipped tensor,
   and step counts up to 1e5 (the bias corrections).
3. BucketAdam's state dict is torch.optim.Adam's, in both directions; schedulers drive its param_groups as they drive Adam's;
   create_optimizer splits the groups as the reference's factory does."""
import ctypes
import os
import shutil
import subprocess
from copy import deepcopy

import numpy as np
import pytest
import torch

from tests import _refextract

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------ 1. C-ABI
def test_adam_structs_have_the_c_layout(tmp_path):
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    structs = {'DbwAdamSegment': _lib.DbwAdamSegment, 'DbwAdamGroup': _lib.DbwAdamGroup}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
             '  printf("max %d %d\\n", DBW_ADAM_MAX_SEGMENTS, DBW_ADAM_MAX_GROUPS);']
    for name, cls in structs.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{name}.{field} %zu\\n", offsetof({name}, {field}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert out[0].split()[1:] == [str(_lib.ADAM_MAX_SEGMENTS), str(_lib.ADAM_MAX_GROUPS)]
    got = dict(l.split() for l in out[1:])
    for name, cls in structs.items():
        assert int(got[name]) == ctypes.sizeof(cls), name
        for field, _ in cls._fields_:
            assert int(got[f'{name}.{field}']) == getattr(cls, field).offset, f'{name}.{field}'


def test_adam_step_validates_its_arguments_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    assert 'dbw_adam_step' in _lib.EXPORTS
    groups = (_lib.DbwAdamGroup * 1)(_lib.DbwAdamGroup(0.9, 0.999, 1e-8, 0.))
    fake = ctypes.c_void_p(256)          # never dereferenced: every call below is refused before a launch
    bad_sizes = [dict(n_segments=0), dict(n_segments=65), dict(n_groups=0), dict(n_groups=9), dict(n_total=0), dict(n_total=-4)]
    for kw in bad_sizes:
        a = dict(n_segments=1, n_total=16, n_groups=1)
        a.update(kw)
        rc = L.dbw_adam_step(fake, a['n_segments'], a['n_total'], groups, a['n_groups'], fake, fake, None)
        assert rc != 0 and b'dbw_adam_step: bad sizes' in L.dbw_last_error(), kw
    for null in range(4):
        ptrs = [fake, groups, fake, fake]
        ptrs[null] = None
        rc = L.dbw_adam_step(ptrs[0], 1, 16, ptrs[1], 1, ptrs[2], ptrs[3], None)
        assert rc != 0 and b'null pointer' in L.dbw_last_error(), null


# ------------------------------------------------------------------ 2. the update, on the host
@pytest.fixture(scope='module')
def ho():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_optim_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_optim_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.ho_adam_step.restype = None
    L.ho_adam_step.argtypes = [ctypes.c_int64] + [ctypes.c_void_p] * 4 + [ctypes.c_double] * 4 + [ctypes.c_float, ctypes.c_int64]
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class _HostAdam:
    """the kernel's arithmetic over a list of numpy tensors: state per tensor, a tensor whose gradient is None is skipped"""

    def __init__(self, ho, params, group_of, groups):
        self.ho, self.p, self.group_of, self.groups = ho, params, group_of, groups
        self.m = [np.zeros_like(p) for p in params]
        self.v = [np.zeros_like(p) for p in params]
        self.t = [0] * len(params)

    def step(self, grads):
        for i, g in enumerate(grads):
            if g is None:
                continue
            self.t[i] += 1
            o = self.groups[self.group_of[i]]
            self.ho.ho_adam_step(self.p[i].size, _p(self.p[i]), _p(np.ascontiguousarray(g)), _p(self.m[i]), _p(self.v[i]),
                                 o['betas'][0], o['betas'][1], o['eps'], o['weight_decay'], o['lr'], self.t[i])


def _adam64(p, g, m, v, t, lr, betas, eps, weight_decay):
    """torch.optim.Adam's single-tensor update restated in float64; lr as the kernel reads it (a float)"""
    b1, b2 = betas
    if weight_decay != 0:
        g = g + weight_decay * p
    m = m + (1 - b1) * (g - m)
    v = b2 * v + (1 - b2) * g * g
    p = p - (float(np.float32(lr)) / (1 - b1 ** t)) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps)
    return p, m, v


GROUPS = [dict(lr=5e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.),
          dict(lr=5e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=1e-2)]
SHAPES = [((7, 3), 0), ((1,), 0), ((5,), 0), ((33, 5), 1), ((4, 4, 3), 1)]          # (shape, group); tensor 2 never gets a gradient
SKIPPED = 2


def _problem(seed):
    rng = np.random.default_rng(seed)
    params = [rng.normal(size=s).astype(np.float32) for s, _ in SHAPES]
    grads = [[None if i == SKIPPED else (rng.normal(size=s) * rng.uniform(0.01, 3)).astype(np.float32) for i, (s, _) in enumerate(SHAPES)]
             for _ in range(200)]
    return params, grads


def test_host_update_matches_float64_and_torch_adam_over_200_steps(ho):
    params, grads = _problem(0)
    group_of = [g for _, g in SHAPES]
    mine = _HostAdam(ho, [p.copy() for p in params], group_of, GROUPS)
    tp = [torch.nn.Parameter(torch.from_numpy(p.copy())) for p in params]
    ref = torch.optim.Adam([dict(params=[q for q, g in zip(tp, group_of) if g == k], **GROUPS[k]) for k in range(2)], foreach=False)
    p64 = [p.astype(np.float64) for p in params]
    m64 = [np.zeros_like(p) for p in p64]
    v64 = [np.zeros_like(p) for p in p64]
    for t, gs in enumerate(grads, start=1):
        # per step, from the same state: the host build against torch's CPU fp32 Adam
        for q, p, m, v in zip(tp, mine.p, mine.m, mine.v):
            with torch.no_grad():
                q.copy_(torch.from_numpy(p))
            if q in ref.state:
                ref.state[q]['exp_avg'].copy_(torch.from_numpy(m))
                ref.state[q]['exp_avg_sq'].copy_(torch.from_numpy(v))
        for q, g in zip(tp, gs):
            q.grad = None if g is None else torch.from_numpy(g.copy())
        mine.step(gs)
        ref.step()
        for i, q in enumerate(tp):
            if gs[i] is None:
                assert q not in ref.state and mine.t[i] == 0
                continue
            st = ref.state[q]
            assert int(st['step']) == mine.t[i] == t
            for name, a, b in (('p', mine.p[i], q.detach().numpy()), ('m', mine.m[i], st['exp_avg'].numpy()),
                               ('v', mine.v[i], st['exp_avg_sq'].numpy())):
                assert np.abs(a - b).max() <= 2e-7 * np.abs(b).max(), (t, i, name)
        # free-running float64
        for i, g in enumerate(gs):
            if g is not None:
                p64[i], m64[i], v64[i] = _adam64(p64[i], g.astype(np.float64), m64[i], v64[i], t, **GROUPS[group_of[i]])
    for i in range(len(SHAPES)):
        for name, a, b in (('p', mine.p[i], p64[i]), ('m', mine.m[i], m64[i]), ('v', mine.v[i], v64[i])):
            if i == SKIPPED:
                assert np.array_equal(a, b.astype(np.float32)), name          # untouched: still the initial values, zero moments
            else:
                # what no fp32 Adam escapes over 200 steps (torch's drifts as far): the parameter is rounded once per step, a
                # random walk of half-ulps, and (float)0.999 is 1.3e-8 off beta2, which the second moment compounds every step
                tol = 1e-6 if name == 'm' else 4e-6
                assert np.abs(a - b).max() <= tol * np.abs(b).max(), (i, name, np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize('t', [1, 2, 10, 1000, 6931, 99999, 100000])
def test_host_bias_corrections_up_to_1e5_steps(ho, t):
    """one step at counter t from a given state: where 1 - beta2^t runs from 1e-3 to 1 and beta1^t underflows past fp32"""
    rng = np.random.default_rng(t)
    for o in GROUPS:
        p = rng.normal(size=257).astype(np.float32)
        g = rng.normal(size=257).astype(np.float32)
        m = (0.1 * rng.normal(size=257)).astype(np.float32)
        v = (0.1 * rng.uniform(0.01, 1, size=257)).astype(np.float32)
        ref = _adam64(p.astype(np.float64), g.astype(np.float64), m.astype(np.float64), v.astype(np.float64), t, **o)
        ho.ho_adam_step(p.size, _p(p), _p(g), _p(m), _p(v), o['betas'][0], o['betas'][1], o['eps'], o['weight_decay'], o['lr'], t)
        for name, a, b in zip('pmv', (p, m, v), ref):
            assert np.abs(a - b).max() <= 2e-7 * np.abs(b).max(), (name, o['lr'])


# ------------------------------------------------------------------ 3. the optimiser class
def _params(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g)) for s in ((3, 2), (5,), (2, 2, 3), (1,))]


def _two_groups(ps):
    return [dict(params=ps[:2]), dict(params=ps[2:], lr=0.05, weight_decay=0.01, betas=(0.8, 0.99))]


def test_constructor_refuses_what_the_kernel_does_not_do():
    from dbw_b200.optim import BucketAdam
    from dbw_b200._lib import DbwError
    ps = _params()
    for kw in (dict(amsgrad=True), dict(maximize=True)):
        with pytest.raises(NotImplementedError):
            BucketAdam(ps, **kw)
    with pytest.raises(NotImplementedError):
        BucketAdam([dict(params=ps[:2]), dict(params=ps[2:], amsgrad=True)])
    with pytest.raises(ValueError):
        BucketAdam([torch.nn.Parameter(torch.zeros(3, dtype=torch.float64))])
    with pytest.raises(ValueError):
        BucketAdam([torch.nn.Parameter(torch.zeros(2)) for _ in range(65)])
    with pytest.raises(ValueError):
        BucketAdam(ps, betas=(1.0, 0.999))
    opt = BucketAdam(ps)
    with pytest.raises(RuntimeError):
        opt.add_param_group(dict(params=[torch.nn.Parameter(torch.zeros(2))]))
    for p in ps:
        p.grad = torch.ones_like(p)
    with pytest.raises(DbwError):          # no CPU path
        opt.step()


def test_state_is_views_of_flat_buffers():
    from dbw_b200.optim import BucketAdam
    ps = _params()
    opt = BucketAdam(_two_groups(ps), lr=0.005)
    assert opt.exp_avg.dtype == opt.exp_avg_sq.dtype == torch.float32 and opt.steps.dtype == torch.int64
    assert opt.exp_avg.numel() == sum((p.numel() + 3) // 4 * 4 for p in ps)
    for i, p in enumerate(ps):
        st = opt.state[p]
        assert st['exp_avg'].shape == p.shape and st['exp_avg_sq'].shape == p.shape
        assert st['exp_avg'].untyped_storage().data_ptr() == opt.exp_avg.untyped_storage().data_ptr()
        assert st['exp_avg'].data_ptr() % 16 == 0 and st['exp_avg_sq'].data_ptr() % 16 == 0
        st['step'].fill_(i + 1)
    assert opt.steps.tolist() == [1, 2, 3, 4]


def test_state_dict_round_trips_with_torch_adam_in_both_directions():
    from dbw_b200.optim import BucketAdam
    ps = _params()
    adam = torch.optim.Adam(_two_groups(ps), lr=0.005)
    for k in range(3):          # the last parameter gets no gradient: torch keeps no state for it
        for p in ps[:3]:
            p.grad = torch.randn(p.shape, generator=torch.Generator().manual_seed(k))
        adam.step()
    sd = adam.state_dict()
    assert sorted(sd['state']) == [0, 1, 2]

    mine = BucketAdam(_two_groups(ps), lr=0.1)          # options come from the loaded dict
    mine.load_state_dict(deepcopy(sd))
    assert mine.steps.tolist() == [3, 3, 3, 0]
    assert [g['lr'] for g in mine.param_groups] == [0.005, 0.05] and mine.param_groups[1]['betas'] == (0.8, 0.99)
    for i, p in enumerate(ps[:3]):
        assert torch.equal(mine.state[p]['exp_avg'], sd['state'][i]['exp_avg'])
        assert torch.equal(mine.state[p]['exp_avg_sq'], sd['state'][i]['exp_avg_sq'])
    assert not mine.state[ps[3]]['exp_avg'].any()

    back = mine.state_dict()
    assert set(back) == {'state', 'param_groups'} and sorted(back['state']) == [0, 1, 2]
    for i in range(3):
        a, b = back['state'][i], sd['state'][i]
        assert set(a) == set(b) == {'step', 'exp_avg', 'exp_avg_sq'}
        assert a['step'].dtype == b['step'].dtype and a['step'].device == b['step'].device and a['step'].shape == b['step'].shape
        assert all(torch.equal(a[k], b[k]) for k in a)
        assert a['exp_avg'].data_ptr() != mine.state[ps[i]]['exp_avg'].data_ptr()          # a copy, not a view of the flat buffer
    for a, b in zip(back['param_groups'], sd['param_groups']):
        assert a == b          # same keys, same values, same parameter indices

    fresh = torch.optim.Adam(_two_groups(ps), lr=0.1)
    fresh.load_state_dict(back)
    again = fresh.state_dict()
    assert all(torch.equal(again['state'][i][k], sd['state'][i][k]) for i in range(3) for k in ('step', 'exp_avg', 'exp_avg_sq'))
    # and the loaded torch optimiser steps on from there exactly as the original does
    for p in ps[:3]:
        p.grad = torch.ones_like(p)
    snap = [p.detach().clone() for p in ps]
    adam.step()
    after = [p.detach().clone() for p in ps]
    with torch.no_grad():
        for p, s in zip(ps, snap):
            p.copy_(s)
    fresh.step()
    assert all(torch.equal(p, a) for p, a in zip(ps, after))


def test_load_state_dict_refuses_other_groups_and_shapes():
    from dbw_b200.optim import BucketAdam
    ps = _params()
    mine = BucketAdam(_two_groups(ps))
    with pytest.raises(ValueError):
        mine.load_state_dict(torch.optim.Adam(ps).state_dict())          # one group of four, not two of two
    other = torch.optim.Adam(_two_groups([torch.nn.Parameter(torch.zeros(2, 3)) for _ in ps]))
    for g in other.param_groups:
        for p in g['params']:
            p.grad = torch.ones_like(p)
    other.step()
    with pytest.raises(ValueError):
        mine.load_state_dict(other.state_dict())
    sd = torch.optim.Adam(_two_groups(ps), amsgrad=True).state_dict()
    with pytest.raises(NotImplementedError):
        mine.load_state_dict(sd)


def _rates(opt, make_scheduler, n):
    sched = make_scheduler(opt)
    opt._opt_called = True          # silences torch's step-order warning; no optimiser step is taken here
    out = [[g['lr'] for g in opt.param_groups]]
    for _ in range(n):
        sched.step()
        out.append([g['lr'] for g in opt.param_groups])
    return out


@pytest.mark.parametrize('make', [lambda o: torch.optim.lr_scheduler.MultiStepLR(o, milestones=[3, 5], gamma=0.2),
                                  lambda o: torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=6),
                                  lambda o: torch.optim.lr_scheduler.ExponentialLR(o, gamma=0.9)],
                         ids=['multi_step', 'cosine_annealing', 'exponential'])
def test_torch_schedulers_drive_the_param_groups_as_they_drive_adams(make):
    from dbw_b200.optim import BucketAdam
    ps = _params()
    assert _rates(BucketAdam(_two_groups(ps), lr=0.005), make, 8) == _rates(torch.optim.Adam(_two_groups(ps), lr=0.005), make, 8)


class _Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        for n, s in (('S', (4, 3)), ('alpha_logit', (4,)), ('texture_bkg', (1, 4, 4, 3)), ('T', (4, 3)), ('textures', (4, 2, 2, 3))):
            setattr(self, n, torch.nn.Parameter(torch.zeros(s)))


CFG = {'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}


def test_create_optimizer_splits_the_texture_group():
    from dbw_b200.optim import BucketAdam, create_optimizer
    model = _Toy()
    opt = create_optimizer(deepcopy(CFG), model)
    assert isinstance(opt, BucketAdam)
    assert [[id(p) for p in g['params']] for g in opt.param_groups] == [[id(model.S), id(model.alpha_logit), id(model.T)],
                                                                       [id(model.texture_bkg), id(model.textures)]]
    assert [g['lr'] for g in opt.param_groups] == [0.005, 0.05]
    one = create_optimizer({'training': {'optimizer': {'name': 'adam', 'lr': 0.01, 'weight_decay': 0.1}}}, model)
    assert len(one.param_groups) == 1 and one.param_groups[0]['weight_decay'] == 0.1 and len(one.param_groups[0]['params']) == 5
    for name in ('sgd', 'adamw', None):
        with pytest.raises(NotImplementedError):
            create_optimizer({'training': {'optimizer': {'name': name, 'lr': 0.01}}}, model)


@pytest.mark.skipif(not _refextract.have_reference(), reason='DBW_REFERENCE names no reference checkout')
def test_reference_factory_and_scheduler_see_the_same_optimiser():
    """the reference's own create_optimizer and MultiStepLR (read from the checkout, not copied): the same group split, and the
    same rates through the warm-up and a milestone, whether they drive torch.optim.Adam or BucketAdam"""
    from bisect import bisect_right
    from collections import Counter
    from dbw_b200.optim import create_optimizer
    quiet = lambda *a, **k: None
    ns = _refextract.extract('src/optimizer.py', ['create_optimizer', 'get_optimizer'],
                             {'deepcopy': deepcopy, 'print_log': quiet,
                              **{n: getattr(torch.optim, n) for n in ('SGD', 'Adam', 'AdamW', 'ASGD', 'Adamax', 'Adadelta', 'Adagrad', 'RMSprop')}})
    sched = _refextract.extract('src/scheduler.py', ['MultiStepLR'],
                                {'Counter': Counter, 'bisect_right': bisect_right, 'print_log': quiet,
                                 '_LRScheduler': torch.optim.lr_scheduler._LRScheduler})['MultiStepLR']
    model = _Toy()
    theirs, mine = ns['create_optimizer'](deepcopy(CFG), model), create_optimizer(deepcopy(CFG), model)
    assert isinstance(theirs, torch.optim.Adam)
    assert [[id(p) for p in g['params']] for g in theirs.param_groups] == [[id(p) for p in g['params']] for g in mine.param_groups]
    make = lambda o: sched(o, milestones=[6], gamma=[0.1, 0.5], warmup=4)
    a, b = _rates(theirs, make, 9), _rates(mine, make, 9)
    assert a == b
    assert a[1] == [0.005 / 2, 0.05 / 2] and a[3] == a[5] == [0.005, 0.05] and a[6] == a[9] == [0.005 * 0.1, 0.05 * 0.5]
