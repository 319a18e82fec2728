"""CPU: what tests/test_vgg_matrix_gpu.py relies on, without a GPU.

  - its restatement of the workspace layout adds up to dbw_vgg_loss_workspace_bytes for every level subset, with and
    without save_for_backward, at its case shapes and the extremes, and the sizes a subset cannot run at are refused;
  - the plain single-head entry points refuse bad sizes, channel counts and null pointers;
  - dbw_vgg_loss_forward and dbw_vgg_loss_backward refuse a workspace one float short, on the host, before any launch;
  - its per-element bounds hold for a CPU float32 evaluation of every step (the same operation on the same float32
    inputs, the convolutions accumulated as the tensor cores do), through the whole loss of each of its cases that is
    small enough for a CPU, and each relative-L2 bar sits between HEADROOM x and 32 x the worst deviation of that
    evaluation from float64 over those cases."""
import ctypes
import functools

import pytest
import torch
import torch.nn.functional as F

from tests import test_lpips_matrix_gpu as M
from tests import test_vgg_matrix_gpu as V

# a bar is at least HEADROOM x the float32 evaluation's relative-L2 deviation and at most 32 x it (the bars are 8 x; CPUs
# differ in their float32 summation order)
HEADROOM = 4

EXTREME_SHAPES = [(1, 1, 1), (65535, 1, 1), (1, 32767, 16), (1, 16, 32767), (65535, 16, 16)]
SHAPES = sorted({(c.B, c.H, c.W) for c in V.CASES.values()} | set(EXTREME_SHAPES))


def _bytes(B, H, W, levels, save):
    from dbw_b200 import _lib
    n = ctypes.c_size_t(0)
    o = _lib.DbwVggLossOptions(V.mask_of(levels), 1, 1, 0)
    return _lib.lib().dbw_vgg_loss_workspace_bytes(B, H, W, ctypes.byref(o), save, ctypes.byref(n)), n.value


@pytest.mark.parametrize('B,H,W', SHAPES)
@pytest.mark.parametrize('save', [0, 1])
def test_layout_restatement_adds_up_to_the_workspace_size(B, H, W, save):
    for levels in V.SUBSETS.values():
        rc, n = _bytes(B, H, W, levels, save)
        if min(H, W) < 1 << V.deepest(levels):
            assert rc != 0, levels                                   # the deepest level's tap would be empty
            continue
        assert rc == 0, levels
        L = V.layout(B, H, W, levels, save)
        assert n == L.total * 4, levels
        last = M.TAP_LAYER[V.deepest(levels)]
        assert all(L.act[l] is None for l in range(last + 1, 13))
        assert all((L.act[M.TAP_LAYER[k]] is not None) == (k + 1 in levels or (save and M.TAP_LAYER[k] <= last)) for k in range(5))
        assert all((L.tap0[k] is not None) == (k + 1 in levels) for k in range(5))
        assert all((L.chunks[k] > 0) == (k + 1 in levels) for k in range(5))
        assert L.partials + L.part_off[4] + B * L.chunks[4] <= L.consts and L.consts + 2568 <= L.total


def test_plain_head_entries_refuse_bad_arguments_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)                                   # never dereferenced: validation fails before any launch
    fwd = lambda B, H, W, C, f0=p, f1=p, part=p: L.dbw_vgg_head_forward(f0, f1, 0.5, B, H, W, C, part, None)  # noqa: E731
    bwd = lambda B, H, W, C, f0=p, f1=p, gv=p, g=p: L.dbw_vgg_head_backward(f0, f1, 0.5, B, H, W, C, gv, 1, g, None)  # noqa: E731
    for f in (fwd, bwd):
        for args in ((0, 8, 8, 64), (65536, 8, 8, 64), (1, 0, 8, 64), (1, 8, 0, 64), (1, 32768, 8, 64), (1, 8, 32768, 64),
                     (1, 8, 8, 96), (1, 8, 8, 1024), (1, 8, 8, 32), (1, 8, 8, 0), (1, -1, 8, 64)):
            assert f(*args) != 0 and b'bad sizes' in L.dbw_last_error(), args
        assert f(1, 8, 8, 64, f0=None) != 0 and b'null pointer' in L.dbw_last_error()
        assert f(1, 8, 8, 64, f1=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert fwd(1, 8, 8, 64, part=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert bwd(1, 8, 8, 512, gv=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert bwd(1, 8, 8, 512, g=None) != 0 and b'null pointer' in L.dbw_last_error()


@pytest.mark.parametrize('levels', [(1,), (2, 4), (1, 2, 3, 4, 5)])
def test_loss_refuses_a_workspace_one_float_short(levels):
    from dbw_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)
    net = _lib.DbwLpipsNet()
    for i in range(13):
        net.conv_w[i] = net.conv_b[i] = 16
    net.shift = net.scale = net.prepared = 16
    for save in (0, 1):
        rc, n = _bytes(2, 16, 24, levels, save)
        assert rc == 0
        o = _lib.DbwVggLossOptions(V.mask_of(levels), 1, 1, 0)
        assert L.dbw_vgg_loss_forward(ctypes.byref(net), ctypes.byref(o), p, p, 2, 16, 24, save, p, p, n - 4, None) != 0
        assert b'workspace too small' in L.dbw_last_error()
    assert L.dbw_vgg_loss_backward(ctypes.byref(net), ctypes.byref(o), p, 2, 16, 24, p, p, n - 4, None) != 0
    assert b'workspace too small' in L.dbw_last_error()


# the GPU module's cases small enough for the CPU (the others differ in size, not in kind)
HOST_CASES = [n for n, c in V.CASES.items() if c.B * c.H * c.W <= 20000]


@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = V.CASES[name]
    return V.make_images(case, 'cpu')


@functools.lru_cache(maxsize=None)
def float32_walk(name):
    """one case of the GPU module stepped in float32 on the CPU as that module steps the kernels (each step's float32
    result feeds the next; the convolutions on the tensor-core model M.TC32).  {kind: (worst error / bound, worst
    relative L2 against float64)}"""
    case = V.CASES[name]
    B, H, W, levels = case.B, case.H, case.W, case.levels
    ni, nf, sc = case.normalize_input, case.normalize_features, case.sum_channels
    want = [k + 1 in levels for k in range(5)]
    last = M.TAP_LAYER[V.deepest(levels)]
    in0, in1 = _inputs(name)
    gv = M.grad_values(B, 'cpu')
    hw = M.level_sizes(H, W)
    out = {}

    def step(kind, fn, *args, dtype=torch.float32):
        """fn(*args, dtype) against fn(*args, float64): record the deviation, return the float32 result"""
        got = fn(*args, dtype)[0]
        want_, bound = fn(*args, torch.float64)
        err = (got.double() - want_).abs()
        assert bool((err <= bound).all()), (name, kind)
        r0, e0 = out.get(kind, (0.0, 0.0))
        out[kind] = (max(r0, float((err / bound.clamp_min(1e-300)).max())), max(e0, M.rel_l2(got, want_)))
        return got

    def features(sd, x, upto):
        acts = [step('first', M.oracle_first, x, V.input_sd(sd, ni), False)]
        for l in range(1, upto + 1):
            a = acts[-1]
            if M.LEVEL[l] != M.LEVEL[l - 1]:
                a = F.max_pool2d(a, 2, 2)
            acts.append(step(V.kind_of(case, 'conv', l), M.oracle_conv, a, M.conv_weight(sd, l), sd[M.SLICE_KEY[l] + '.bias'],
                             True, None, dtype=M.TC32))
        return acts

    sd = M.dead5_state_dict(features(M.state_dict('base'), in1, 12)[11]) if case.sd == 'dead5' else M.state_dict(case.sd)
    f0 = features(sd, in0, last)
    acts = features(sd, in1, last)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(t.shape[0], -1, t.shape[1])          # noqa: E731  NCHW -> (n, P, C)
    parts, sizes = [], []
    for k in range(5):
        if not want[k]:
            continue
        w = V.head_weight(k, sc)
        a, b = flat(f0[M.TAP_LAYER[k]]), flat(acts[M.TAP_LAYER[k]])
        if nf:
            lin = torch.full((M.TAP_C[k],), w)
            parts.append(step(V.kind_of(case, 'head', k), lambda *z: tuple(map(M.chunk_sums, M.oracle_head(*z))), a, b, lin, None))
        else:
            parts.append(step('plain_head', lambda *z: tuple(map(M.chunk_sums, V.oracle_plain_head(*z))), a, b, w))
        sizes.append(hw[k][0] * hw[k][1])
    step('vgg_value', M.oracle_value, parts, sizes)
    G = None
    for l in range(last, 0, -1):
        lv = M.LEVEL[l]
        if l == M.TAP_LAYER[lv]:
            g_in = None
            if l != last:
                x = acts[l].clone().requires_grad_(True)
                F.max_pool2d(x, 2, 2).backward(G)
                G = x.grad
                g_in = flat(G)
            h, w = hw[lv]
            if want[lv]:
                a, b = flat(f0[l]), flat(acts[l])
                wt = V.head_weight(lv, sc)
                if nf:
                    G = step(V.kind_of(case, 'head_bwd', lv), M.oracle_head_backward, a, b, torch.full((M.TAP_C[lv],), wt), None, gv,
                             g_in)
                else:
                    G = step('plain_head_bwd', V.oracle_plain_head_backward, a, b, wt, gv, g_in)
                G = G.view(B, h, w, -1).permute(0, 3, 1, 2)
            else:
                G = torch.where(acts[l] > 0, G, torch.zeros_like(G))
        mask = None if M.LEVEL[l - 1] != lv else acts[l - 1]
        G = step('conv_bwd', M.oracle_conv, G, M.conv_weight(sd, l, bwd=True), None, False, mask, dtype=M.TC32)
    step('dgrad', M.oracle_dgrad, G, V.input_sd(sd, ni), False)
    return out


@functools.lru_cache(maxsize=None)
def value_deviation(name):
    """(worst error / bound, relative L2) of the value step in float32 at the chunk counts of every case, the large ones
    included: the deviation of an in-order sum grows with its length, and hardly depends on the positive partials summed"""
    case = V.CASES[name]
    hw = [s for k, s in enumerate(M.level_sizes(case.H, case.W)) if k + 1 in case.levels]
    g = torch.Generator().manual_seed(case.B * case.H * case.W)
    n = len(case.images) if case.images else case.B
    parts = [torch.rand(n, M.chunks(h, w), generator=g).float() for h, w in hw]
    got = M.oracle_value(parts, [h * w for h, w in hw], torch.float32)[0]
    want, bound = M.oracle_value(parts, [h * w for h, w in hw], torch.float64)
    err = (got.double() - want).abs()
    assert bool((err <= bound).all()), name
    return float((err / bound).max()), M.rel_l2(got, want)


def float32_deviations():
    """{kind: (worst error / bound, worst relative L2)} over HOST_CASES (and, for the value, every case)"""
    out = {}
    walks = [float32_walk(name) for name in HOST_CASES] + [{'vgg_value': value_deviation(name)} for name in V.CASES]
    for w in walks:
        for kind, (r, e) in w.items():
            r0, e0 = out.get(kind, (0.0, 0.0))
            out[kind] = (max(r0, r), max(e0, e))
    return out


@pytest.mark.parametrize('name', HOST_CASES)
def test_every_bound_holds_for_a_float32_evaluation(name):
    worst = float32_walk(name)                                      # asserts every element of every step against its bound
    assert set(worst) <= set(V.BARS)
    assert all(ratio <= 1 for ratio, _ in worst.values()), worst


@pytest.mark.parametrize('kind', sorted(V.BARS))
def test_bar_sits_a_fixed_multiple_above_float32_rounding(kind):
    assert set(float32_deviations()) == set(V.BARS)
    dev, bar = float32_deviations()[kind][1], V.BARS[kind]
    assert HEADROOM * dev <= bar, f'{kind}: float32 deviates by {dev:.3g}; bar {bar:.3g} leaves less than {HEADROOM}x'
    assert bar <= 32 * dev, f'{kind}: bar {bar:.3g} is loose for a float32 deviation of {dev:.3g}'
