"""GPU: the VGG16 feature loss of csrc/dbw_lpips.cu (dbw_vgg_loss_*) one step at a time, each step against the float64
oracle on the kernel's own float32 inputs.

Each case runs the real `dbw_vgg_loss_forward(save_for_backward=1)` and `dbw_vgg_loss_backward` on a workspace whose layout
(include/dbw_render.h) `layout` restates, with a sentinel tail past `workspace_bytes` that neither call may touch.  Then:

  forward   act[l], l <= last (the tap layer of the deepest requested level; no region exists past it), against the float64
            layer applied to the workspace's act[l-1] (max-pooled first where a pool sits in between; the pool itself, by
            `dbw_lpips_maxpool`, equal to F.max_pool2d bit for bit); imgs' taps against rec's taps of a second forward with
            in1 := in0, bit for bit; the constants region holds exactly w = 1 or 1 / C_k per level, then shift 0 and scale 1;
            a forward without save_for_backward gives the same taps and value bit for bit;
  heads     each requested level's head by its single-head entry (`dbw_vgg_head_forward`, or `dbw_lpips_head_forward` with
            train = 0 and lin = the constants' w when the features are normalised) on the workspace's taps: its partials
            equal the forward's bit for bit, and each 64-pixel chunk is checked against the float64 head; value[b] against
            the float64 reduction of the kernel's own partials of the requested levels;
  backward  replayed with the single-step entries (maxpool_backward, the head backward with accumulate = !deepest,
            torch.where(act > 0, g, 0) for the tap of a level not requested, the input-gradient conv3x3 with the
            act[l-1] > 0 mask unless a pool follows, dgrad_last with the net's scale or 1).  The replay's gradient must equal
            the real call's bit for bit (the kernels are deterministic: a difference is orchestration), and every step is
            checked against the float64 step on the replay's input.

The convolutions, the first layer, the last input gradient, the normalised head (`head`, `head_bwd`) and the pools take the
per-element bounds of tests/test_lpips_matrix_gpu.py, whose oracle steps this module imports; the first layer and dgrad_last
see (x - mean_rgb) / std_rgb, or the identity transform (x - 0) / 1, never LPIPS's 2x - 1.  The plain head, u = 2^-24,
eta = 2^-150, every bound evaluated in float64 from the same float32 operands and doubled for the second-order terms:

  plain_head      per pixel w sum_c (f0 - f1)^2: the difference errs by u |e|, its square by 2u e^2 + u e^2; NPL = C / 32
                  FMAs per lane, the 5-level shuffle tree, the warp's 8 pixels, then the 8 warps add NPL + 5 + 8 + 8
                  roundings of sum |w| e^2.  Bound 2 |w| sum_c ((NPL + 24) u e^2 + eta) per pixel, summed over the chunk.
  plain_head_bwd  k = 2w (gv / HW): 2w is exact, gv / HW and the product one rounding each; k (u1 - f0) adds one for the
                  difference and one for the product; the accumulate (or the FMA it may be fused into) one of the result.
                  Bound 2 (4u |k (u1 - f0)| + u |k (u1 - f0) + g_in| + eta), then * [u1 > 0], exact.
  vgg_value       lpips_reduce_kernel: each requested level's partials summed in chunk order (chunks_k - 1 roundings), the fp32
                  1 / (H_k W_k) and the product (2), the levels in order (up to 5): tests/test_lpips_matrix_gpu.py's value
                  bound 2 (chunks_k + 7) u sum_k sum_c |partial_c| / (H_k W_k) over the requested levels.

No ReLU or pool decision can differ from the oracle's, since both sides read the same fp32 tensors; each comparison is one
step deep.  At B = 65535 the kernels run on the whole batch and the oracle on images 0, 32767 and 65534.

A worst-case bound lets a small systematic error through, so every array also meets a relative-L2 bar: BARS[kind], about
8 x the worst deviation of a CPU float32 evaluation of the same step over this module's cases that fit a CPU (the
convolutions on the tensor-core model; tests/test_vgg_matrix_host.py checks that each bar sits between 4 x and 32 x it).
Arrays that cancel by construction have kinds of their own (`kind_of`): layer 12 of 'dead5', whose bias nearly cancels the
convolution; the normalised heads of 'near', where n0 - n1 cancels; the relu5_3 head backward of 'dead5', whose nearly dead
pixels divide by a tiny norm."""
import ctypes
import functools
import time
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import test_lpips_matrix_gpu as M

pytestmark = pytest.mark.gpu
DEV = M.DEV
U, ETA = M.U, M.ETA
CIN, COUT, LEVEL, TAP_LAYER, TAP_C = M.CIN, M.COUT, M.LEVEL, M.TAP_LAYER, M.TAP_C
N_CONSTS = 5 * 512 + 8
MEAN_RGB = (0.485, 0.456, 0.406)
STD_RGB = (0.229, 0.224, 0.225)

# relative-L2 bars per step kind: about 8 x the worst deviation of the CPU float32 evaluation of
# tests/test_vgg_matrix_host.py over the arrays of that kind (the '_cancel' kinds: see `kind_of`)
BARS = {'first': 9e-7, 'conv': 1e-4, 'conv_bwd': 1.1e-4, 'dgrad': 1.3e-6, 'head': 5.5e-6, 'head_bwd': 2.5e-5, 'plain_head': 7.5e-7,
        'plain_head_bwd': 4.5e-7, 'vgg_value': 7.5e-7, 'conv_cancel': 6e-4, 'head_cancel': 4.5e-4, 'head_bwd_cancel': 1.1e-3}


# ------------------------------------------------------------------------------------------------ workspace layout
def deepest(levels):
    """0-based index of the deepest requested level (levels: 1-based, as the options' bits k - 1)"""
    return max(levels) - 1


def mask_of(levels):
    return sum(1 << (k - 1) for k in set(levels))


Layout = namedtuple('Layout', 'act tap0 s0 s1 partials part_off chunks consts total')


def layout(B, H, W, levels, save):
    """the workspace layout of include/dbw_render.h, offsets in floats (None where a region is absent)"""
    hw = M.level_sizes(H, W)
    want = [k + 1 in levels for k in range(5)]
    last = TAP_LAYER[deepest(levels)]
    o, act = 0, []
    for l in range(13):
        lv = LEVEL[l]
        if l > last or (not save and not (l == TAP_LAYER[lv] and want[lv])):
            act.append(None)
            continue
        act.append(o)
        o += M._align64(B * hw[lv][0] * hw[lv][1] * COUT[l])
    tap0 = []
    for k in range(5):
        tap0.append(o if want[k] else None)
        if want[k]:
            o += M._align64(B * hw[k][0] * hw[k][1] * TAP_C[k])
    big = M._align64(B * H * W * 64)
    s0, s1 = o, o + big
    o += 2 * big
    partials, part_off, chunks, p = o, [], [], 0
    for k in range(5):
        chunks.append(M.chunks(*hw[k]) if want[k] else 0)
        part_off.append(p)
        p += B * chunks[k]
    o += M._align64(p)
    return Layout(tuple(act), tuple(tap0), s0, s1, partials, tuple(part_off), tuple(chunks), o, o + M._align64(N_CONSTS))


def head_weight(k, sum_channels):
    """w of level k (0-based): 1, or 1 / C_k in float32 (exact: C_k is a power of 2)"""
    return 1.0 if sum_channels else float(np.float32(1.0 / TAP_C[k]))


# ------------------------------------------------------------------------------------------------ float64 steps
def input_sd(sd, normalize_input):
    """sd (LPIPS names) with the first layer's transform the loss applies: (x - mean_rgb) / std_rgb, or the identity of the
    constants region, (x - 0) / 1; for tests/test_lpips_matrix_gpu.py's oracle_first and oracle_dgrad with normalize = 0"""
    shift, scale = (torch.tensor(MEAN_RGB), torch.tensor(STD_RGB)) if normalize_input else (torch.zeros(3), torch.ones(3))
    return dict(sd, **{'scaling_layer.shift': shift.view(1, 3, 1, 1), 'scaling_layer.scale': scale.view(1, 3, 1, 1)})


def vgg_state_dict(sd):
    """the PerceptualLoss names of an LPIPS-named state dict's convolutions, with the ImageNet statistics"""
    out = {'mean_rgb': torch.tensor(MEAN_RGB), 'std_rgb': torch.tensor(STD_RGB)}
    for key in M.SLICE_KEY:
        for n in ('weight', 'bias'):
            out[f'{key[len("net."):]}.{n}'] = sd[f'{key}.{n}']
    return out


def oracle_plain_head(f0, f1, w, dtype):
    """per-pixel plain head w sum_c (f0 - f1)^2 of (n, P, C) features: (values (n, P) in dtype, bounds (n, P))"""
    C = f0.shape[-1]
    e = f0.to(dtype) - f1.to(dtype)
    val = (w * e * e).sum(-1)
    e64 = f0.double() - f1.double()
    bound = 2 * abs(w) * ((C // 32 + 24) * U * e64 * e64 + ETA).sum(-1)
    return val, bound


def oracle_plain_head_backward(f0, f1, w, gv, g_in, dtype):
    """(d sum_b gv[b] mean_p plain head / d f1 + g_in) * [f1 > 0] of (n, P, C) features, gv (n,), g_in (n, P, C) or None"""
    P = f0.shape[1]
    k = 2 * w * (gv.to(dtype) / P).view(-1, 1, 1)
    v = k * (f1.to(dtype) - f0.to(dtype))
    if g_in is not None:
        v = v + g_in.to(dtype)
    keep = f1 > 0
    a = 2 * w * (gv.double() / P).view(-1, 1, 1) * (f1.double() - f0.double())
    t = a if g_in is None else a + g_in.double()
    return v * keep, 2 * (4 * U * a.abs() + U * t.abs() + ETA) * keep


# ------------------------------------------------------------------------------------------------ cases
Case = namedtuple('Case', 'B H W levels normalize_input normalize_features sum_channels inputs sd images',
                  defaults=('random', 'base', None))
ALL = (1, 2, 3, 4, 5)
# the 8 combinations of (normalize_input, normalize_features, sum_channels), round robin over the 31 level subsets: each
# combination meets at least three subsets
COMBOS = [(ni, nf, sc) for ni in (1, 0) for nf in (1, 0) for sc in (0, 1)]
SUBSETS = {m: tuple(k + 1 for k in range(5) if m >> k & 1) for m in range(1, 32)}
CASES = {f'2x16x24_L{m:02d}': Case(2, 16, 24, SUBSETS[m], *COMBOS[(m - 1) % 8]) for m in range(1, 32)}
CASES.update({
    # each level's smallest images: relu1_2 on 1x1, 1xW and Hx1; a pool to 1x1 dropping a row or a column; deepest 3, 5
    'L1_2x1x1': Case(2, 1, 1, (1,), 1, 1, 0),
    'L1_3x1x37': Case(3, 1, 37, (1,), 0, 0, 1),
    'L1_3x37x1': Case(3, 37, 1, (1,), 1, 0, 0),
    'L12_2x2x3': Case(2, 2, 3, (1, 2), 0, 1, 0),
    'L12_2x3x2': Case(2, 3, 2, (1, 2), 1, 0, 1),
    'L23_2x4x4': Case(2, 4, 4, (2, 3), 1, 1, 1),
    'L135_2x16x16': Case(2, 16, 16, (1, 3, 5), 1, 0, 0),
    'L45_2x17x31': Case(2, 17, 31, (4, 5), 0, 1, 0),
    # odd floors at every pool; M = 1921 = 15 * 128 + 1 (a 1-row conv tile) and H W = 1921 = 30 * 64 + 1 (a 1-pixel head
    # chunk) at level 0
    '2x17x23': Case(2, 17, 23, ALL, 1, 1, 0),
    '1x17x113': Case(1, 17, 113, ALL, 0, 0, 0),
    # the training shape: the reference's default options, and every level
    '4x300x400': Case(4, 300, 400, (3,), 1, 1, 0),
    '4x300x400_L1-5': Case(4, 300, 400, ALL, 1, 0, 1),
    # the head grid's y limit
    '65535x1x1': Case(65535, 1, 1, (1,), 1, 0, 0, images=(0, 32767, 65534)),
    'same': Case(2, 17, 23, ALL, 1, 0, 0, inputs='same'),            # e = 0: value and gradient exactly 0
    'near': Case(2, 33, 47, ALL, 1, 1, 0, inputs='near'),            # in1 within 1e-6 of in0: cancellation in n0 - n1
    'near_plain': Case(2, 33, 47, (2, 4), 0, 0, 1, inputs='near'),
    'black': Case(2, 32, 48, ALL, 0, 1, 0, inputs='black'),          # relu(bias) features, many all-zero vectors
    'dead5': Case(2, 64, 96, (4, 5), 1, 1, 0, sd='dead5'),           # relu5_3 all zero at some pixels (r1 == 0)
})


def kind_of(case, kind, k):
    """the bar kind of the array of step `kind` at layer or level k (0-based) of `case`: the arrays that cancel by
    construction (see the module docstring) get a '_cancel' kind"""
    if (kind == 'conv' and case.sd == 'dead5' and k == 12) or (kind in ('head', 'head_bwd') and case.inputs == 'near') or \
            (kind == 'head_bwd' and case.sd == 'dead5' and k == 4):
        return kind + '_cancel'
    return kind


def make_images(case, device=DEV):
    if case.inputs == 'black':
        z = torch.zeros(case.B, 3, case.H, case.W, device=device)
        return z, z.clone()
    return M.make_images(case, device)


def options(case):
    from dbw_b200 import _lib
    return _lib.DbwVggLossOptions(mask_of(case.levels), case.normalize_input, case.normalize_features, case.sum_channels)


def make_net(sd):
    from dbw_b200.perceptual import PerceptualLoss
    m = PerceptualLoss.from_state_dict(vgg_state_dict(sd)).to(DEV)
    m._prepare()
    return m


@functools.lru_cache(maxsize=None)
def _net(kind):
    return make_net(M.state_dict(kind))


# ------------------------------------------------------------------------------------------------ C-ABI calls
SENTINEL = 7.25
TAIL = 64


def workspace_floats(case, save):
    n = ctypes.c_size_t(0)
    M._call('dbw_vgg_loss_workspace_bytes', case.B, case.H, case.W, ctypes.byref(options(case)), int(save), ctypes.byref(n))
    assert n.value % 4 == 0
    return n.value // 4


def run_forward(net, case, in0, in1, save):
    """the real forward: (workspace (floats, with a sentinel tail past workspace_bytes), value)"""
    B, H, W = case.B, case.H, case.W
    n = workspace_floats(case, save)
    assert n == layout(B, H, W, case.levels, save).total
    ws = torch.full((n + TAIL,), float('nan'), device=DEV)
    ws[n:] = SENTINEL
    value = torch.full((B,), float('nan'), device=DEV)
    M._call('dbw_vgg_loss_forward', ctypes.byref(net._net_struct()), ctypes.byref(options(case)), M._vp(in0), M._vp(in1), B, H, W,
            int(save), M._vp(value), M._vp(ws), n * 4, M._st())
    return ws, value


def tail_intact(ws, case, save):
    return bool((ws[layout(case.B, case.H, case.W, case.levels, save).total:] == SENTINEL).all())


def act_view(ws, Lw, l, B, H, W):
    h, w = M.level_sizes(H, W)[LEVEL[l]]
    return ws[Lw.act[l]:Lw.act[l] + B * h * w * COUT[l]].view(B, h, w, COUT[l])


def tap0_view(ws, Lw, k, B, H, W):
    h, w = M.level_sizes(H, W)[k]
    return ws[Lw.tap0[k]:Lw.tap0[k] + B * h * w * TAP_C[k]].view(B, h, w, TAP_C[k])


def bwd_weight(net, l):
    """the prepared input-gradient copy of layer l"""
    n_w = 9 * CIN[l] * COUT[l]
    o = sum(2 * 9 * CIN[i] * COUT[i] for i in range(1, l)) + n_w
    return net.prepared[o:o + n_w]


# ------------------------------------------------------------------------------------------------ the test
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report():
    torch.cuda.init()
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    print(f'\n{time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.2f} GiB allocated; '
          'worst error / bound and relative L2 per step kind over the cases:')
    for kind, (ratio, rel) in sorted(WORST.items()):
        print(f'  {kind:15s} error/bound {ratio:.3f}   rel L2 {rel:.2e} (bar {BARS.get(kind, 0):.0e})')


class Checker:
    """tests/test_lpips_matrix_gpu.py's Checker, with this module's bars and report"""
    def __init__(self, name):
        self.name, self.worst = name, {}

    def __call__(self, kind, got, want, bound, where=''):
        got, want = got.double(), want.double()
        err = (got - want).abs()
        ok = err <= bound                                          # NaN fails
        ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
        rel = M.rel_l2(got, want)
        assert bool(ok.all()), f'{self.name} {kind} {where}: {int((~ok).sum())} elements outside the bound, worst ratio {ratio:.3g}'
        assert rel <= BARS[kind], f'{self.name} {kind} {where}: relative L2 {rel:.3g} above {BARS[kind]:.1g}'
        for d in (self.worst, WORST):
            r0, e0 = d.get(kind, (0.0, 0.0))
            d[kind] = (max(r0, ratio), max(e0, rel))


def case_net(case, in1):
    """(LPIPS-named state dict, PerceptualLoss module) of a case; 'dead5' sets layer 12's bias from rec's relu5_2"""
    if case.sd != 'dead5':
        return M.state_dict(case.sd), _net(case.sd)
    c5 = case._replace(levels=(5,))
    ws = run_forward(_net('base'), c5, in1, in1, True)[0]
    Lw = layout(case.B, case.H, case.W, c5.levels, True)
    sd = M.dead5_state_dict(M.nchw(act_view(ws, Lw, 11, case.B, case.H, case.W)))
    del ws
    return sd, make_net(sd)


@pytest.mark.parametrize('name', list(CASES))
def test_loss_step_by_step_against_float64(name):
    case = CASES[name]
    B, H, W, levels = case.B, case.H, case.W, case.levels
    ni, nf, sc = case.normalize_input, case.normalize_features, case.sum_channels
    want = [k + 1 in levels for k in range(5)]
    last = TAP_LAYER[deepest(levels)]
    in0, in1 = make_images(case)
    sd, net = case_net(case, in1)
    sdi = input_sd(sd, ni)
    idx = torch.tensor(case.images if case.images else range(B), device=DEV)
    n_img = len(idx)
    hw = M.level_sizes(H, W)
    Lw = layout(B, H, W, levels, True)
    check = Checker(name)
    gv = M.grad_values(B)

    ws, value = run_forward(net, case, in0, in1, True)
    grad_real = torch.full((B, 3, H, W), float('nan'), device=DEV)
    M._call('dbw_vgg_loss_backward', ctypes.byref(net._net_struct()), ctypes.byref(options(case)), M._vp(gv), B, H, W,
            M._vp(grad_real), M._vp(ws), Lw.total * 4, M._st())
    assert tail_intact(ws, case, True), f'{name}: written past workspace_bytes'
    assert all(Lw.act[l] is None for l in range(last + 1, 13)) and all(Lw.act[l] is not None for l in range(last + 1))

    # ---- constants: w per level, then the identity transform
    consts = ws[Lw.consts:Lw.consts + N_CONSTS]
    for k in range(5):
        assert bool((consts[512 * k:512 * k + TAP_C[k]] == head_weight(k, sc)).all()), f'{name}: the weight of level {k + 1}'
    assert torch.equal(consts[5 * 512:], torch.tensor([0.0] * 4 + [1.0] * 4, device=DEV)), f'{name}: shift and scale'

    # ---- forward: every layer from the workspace's previous layer
    A = lambda l: act_view(ws, Lw, l, B, H, W)                                     # noqa: E731
    check('first', M.nchw(A(0)[idx]), *M.oracle_first(in1[idx], sdi, False, torch.float64), 'layer 0')
    for l in range(1, last + 1):
        x = A(l - 1)
        if LEVEL[l] != LEVEL[l - 1]:
            h, w = hw[LEVEL[l - 1]]
            pooled = torch.full((B, h // 2, w // 2, CIN[l]), float('nan'), device=DEV)
            M._call('dbw_lpips_maxpool', M._vp(x), M._vp(pooled), B, h, w, CIN[l], M._st())
            assert torch.equal(M.nchw(pooled[idx]), F.max_pool2d(M.nchw(x[idx]), 2, 2)), f'{name}: pool before layer {l}'
            x = pooled
        w_, bound = M.oracle_conv(M.nchw(x[idx]), M.conv_weight(sd, l), sd[M.SLICE_KEY[l] + '.bias'], True, None, torch.float64)
        check(kind_of(case, 'conv', l), M.nchw(A(l)[idx]), w_, bound, f'layer {l}')
        del x, w_, bound
    # imgs keeps only its requested taps: they are rec's taps of a forward with in1 := in0
    ws2 = run_forward(net, case, in0, in0, True)[0]
    for k in range(5):
        if want[k]:
            assert torch.equal(tap0_view(ws, Lw, k, B, H, W), act_view(ws2, Lw, TAP_LAYER[k], B, H, W)), f'{name}: imgs tap {k}'
    del ws2
    # without save_for_backward: the same taps and value, bit for bit
    ws0, value0 = run_forward(net, case, in0, in1, False)
    assert tail_intact(ws0, case, False), f'{name}: written past workspace_bytes without save_for_backward'
    L0 = layout(B, H, W, levels, False)
    assert torch.equal(value0, value), f'{name}: the value depends on save_for_backward'
    for k in range(5):
        if want[k]:
            assert torch.equal(tap0_view(ws0, L0, k, B, H, W), tap0_view(ws, Lw, k, B, H, W)), f'{name}: imgs tap {k}, unsaved'
            assert torch.equal(act_view(ws0, L0, TAP_LAYER[k], B, H, W), A(TAP_LAYER[k])), f'{name}: rec tap {k}, unsaved'
    del ws0

    # ---- heads and the value
    flat = lambda t: t[idx].reshape(n_img, -1, t.shape[-1])                         # noqa: E731
    parts, sizes = [], []
    for k in range(5):
        if not want[k]:
            continue
        h, w = hw[k]
        f0, f1 = tap0_view(ws, Lw, k, B, H, W), A(TAP_LAYER[k])
        part = torch.full((B, M.chunks(h, w)), float('nan'), device=DEV)
        if nf:
            lin = consts[512 * k:512 * k + TAP_C[k]]
            M._call('dbw_lpips_head_forward', M._vp(f0), M._vp(f1), M._vp(lin), B, h, w, TAP_C[k], k, 0, None, M._vp(part), M._st())
            val, bnd = M.oracle_head(flat(f0), flat(f1), lin, None, torch.float64)
        else:
            M._call('dbw_vgg_head_forward', M._vp(f0), M._vp(f1), head_weight(k, sc), B, h, w, TAP_C[k], M._vp(part), M._st())
            val, bnd = oracle_plain_head(flat(f0), flat(f1), head_weight(k, sc), torch.float64)
        o = Lw.partials + Lw.part_off[k]
        assert torch.equal(part.flatten(), ws[o:o + part.numel()]), f'{name}: head {k} partials differ from the forward'
        check(kind_of(case, 'head' if nf else 'plain_head', k), part[idx], M.chunk_sums(val), M.chunk_sums(bnd), f'level {k + 1}')
        parts.append(part[idx])
        sizes.append(h * w)
    # the value sums the requested levels' partials only: an unrequested level has no chunks to contribute
    assert Lw.partials + Lw.part_off[4] + B * Lw.chunks[4] <= Lw.consts
    check('vgg_value', value[idx], *M.oracle_value(parts, sizes, torch.float64))
    if case.inputs in ('same', 'black'):
        assert not value.any()

    # ---- backward, replayed with the single-step entries
    G = None
    for l in range(last, 0, -1):
        lv = LEVEL[l]
        h, w = hw[lv]
        act = A(l)
        if l == TAP_LAYER[lv]:
            g_in = None
            if l != last:
                gin = torch.full((B, h, w, COUT[l]), float('nan'), device=DEV)
                M._call('dbw_lpips_maxpool_backward', M._vp(act), M._vp(G), M._vp(gin), B, h, w, COUT[l], M._st())
                x = M.nchw(act[idx]).contiguous().requires_grad_(True)
                F.max_pool2d(x, 2, 2).backward(M.nchw(G[idx]))
                assert torch.equal(M.nchw(gin[idx]), x.grad), f'{name}: pool backward after layer {l}'
                G, g_in = gin, flat(gin).clone()
            else:
                G = torch.full((B, h, w, COUT[l]), float('nan'), device=DEV)
            if want[lv]:
                f0 = tap0_view(ws, Lw, lv, B, H, W)
                if nf:
                    lin = consts[512 * lv:512 * lv + TAP_C[lv]]
                    M._call('dbw_lpips_head_backward', M._vp(f0), M._vp(act), M._vp(lin), B, h, w, TAP_C[lv], lv, 0, None, M._vp(gv),
                            int(l != last), M._vp(G), M._st())
                    w_, bound = M.oracle_head_backward(flat(f0), flat(act), lin, None, gv[idx], g_in, torch.float64)
                else:
                    M._call('dbw_vgg_head_backward', M._vp(f0), M._vp(act), head_weight(lv, sc), B, h, w, TAP_C[lv], M._vp(gv),
                            int(l != last), M._vp(G), M._st())
                    w_, bound = oracle_plain_head_backward(flat(f0), flat(act), head_weight(lv, sc), gv[idx], g_in, torch.float64)
                check(kind_of(case, 'head_bwd' if nf else 'plain_head_bwd', lv), flat(G), w_, bound, f'level {lv + 1}')
                del w_, bound
            else:                                                  # the ReLU of a tap whose level is not requested
                G = torch.where(act > 0, G, torch.zeros_like(G))
            del g_in
        after_pool = LEVEL[l - 1] != lv
        mask = None if after_pool else A(l - 1)
        out = torch.full((B, h, w, CIN[l]), float('nan'), device=DEV)
        M._call('dbw_lpips_conv3x3', M._vp(G), M._vp(bwd_weight(net, l)), None, M._vp(mask), M._vp(out), B, h, w, COUT[l], CIN[l], 0,
                M._st())
        w_, bound = M.oracle_conv(M.nchw(G[idx]), M.conv_weight(sd, l, bwd=True), None, False,
                                  None if mask is None else M.nchw(mask[idx]), torch.float64)
        check('conv_bwd', M.nchw(out[idx]), w_, bound, f'layer {l}')
        G = out
        del w_, bound
    grad = torch.full((B, 3, H, W), float('nan'), device=DEV)
    scale = net.std_rgb if ni else torch.ones(3, device=DEV)
    M._call('dbw_lpips_dgrad_last', M._vp(G), M._vp(net._convs()[0].weight), M._vp(scale), 0, M._vp(grad), B, H, W, M._st())
    check('dgrad', grad[idx], *M.oracle_dgrad(M.nchw(G[idx]), sdi, False, torch.float64))
    assert torch.equal(grad, grad_real), f'{name}: the replayed backward differs from dbw_vgg_loss_backward'
    if case.inputs in ('same', 'black'):
        assert not grad_real.any()
    if case.sd == 'dead5':
        r1 = A(12).abs().amax(-1)
        assert bool((r1 == 0).any()) and bool((r1 > 0).any()), 'no pixel of relu5_3 is all zero'
    print(f'{name}: ' + ', '.join(f'{k} {r:.3f} / {e:.1e}' for k, (r, e) in sorted(check.worst.items())))
    torch.cuda.synchronize()
