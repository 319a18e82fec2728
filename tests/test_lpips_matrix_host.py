"""CPU: what tests/test_lpips_matrix_gpu.py relies on, without a GPU.

  - its restatement of the workspace layout adds up to dbw_lpips_workspace_bytes;
  - the single-head entry points refuse bad sizes, channel counts, taps and null pointers;
  - its per-element bounds hold for a CPU float32 evaluation of every step (the same operation on the same float32
    inputs, the convolutions accumulated as the tensor cores do), through the whole term of each of its cases that is
    small enough for a CPU, and each relative-L2 bar sits between HEADROOM x and 32 x the worst deviation of that
    evaluation from float64 over those cases."""
import ctypes
import functools

import pytest
import torch
import torch.nn.functional as F

from oracle import lpips as OL
from tests import test_lpips_matrix_gpu as M

# a bar is at least HEADROOM x the float32 evaluation's relative-L2 deviation and at most 32 x it (the bars are 8 x; CPUs
# differ in their float32 summation order)
HEADROOM = 4

EXTREME_SHAPES = [(1, 16, 16), (65535, 16, 16), (1, 32767, 16), (1, 16, 32767), (2, 1023, 1025), (49, 400, 400)]


@pytest.mark.parametrize('B,H,W', sorted({(c.B, c.H, c.W) for c in M.CASES.values()} | set(EXTREME_SHAPES)))
@pytest.mark.parametrize('save', [0, 1])
def test_layout_restatement_adds_up_to_the_workspace_size(B, H, W, save):
    from dbw_b200 import _lib
    ws, prep = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert _lib.lib().dbw_lpips_workspace_bytes(B, H, W, save, ctypes.byref(ws), ctypes.byref(prep)) == 0
    L = M.layout(B, H, W, save)
    assert ws.value == L.total * 4
    assert (L.act[0] is not None) == bool(save) and all(L.act[l] is not None for l in M.TAP_LAYER)
    assert L.seed + 64 == L.total and L.partials + L.part_off[4] + B * M.chunks(H >> 4, W >> 4) <= L.seed


def test_head_entries_refuse_bad_arguments_without_a_gpu():
    from dbw_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)                                   # never dereferenced: validation fails before any launch
    fwd = lambda B, H, W, C, tap, train=1, seed=p, f0=p, part=p: L.dbw_lpips_head_forward(  # noqa: E731
        f0, p, p, B, H, W, C, tap, train, seed, part, None)
    bwd = lambda B, H, W, C, tap, train=1, seed=p, gv=p, g=p: L.dbw_lpips_head_backward(  # noqa: E731
        p, p, p, B, H, W, C, tap, train, seed, gv, 1, g, None)
    for f in (fwd, bwd):
        for args in ((0, 8, 8, 64, 0), (65536, 8, 8, 64, 0), (1, 0, 8, 64, 0), (1, 8, 0, 64, 0), (1, 32768, 8, 64, 0),
                     (1, 8, 32768, 64, 0), (1, 8, 8, 96, 0), (1, 8, 8, 1024, 0), (1, 8, 8, 32, 0), (1, 8, 8, 64, -1),
                     (1, 8, 8, 64, 5)):
            assert f(*args) != 0 and b'bad sizes' in L.dbw_last_error(), args
    assert fwd(1, 8, 8, 64, 0, f0=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert fwd(1, 8, 8, 64, 0, part=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert fwd(1, 8, 8, 64, 0, seed=None) != 0 and b'null pointer' in L.dbw_last_error()      # train needs the seed
    assert bwd(1, 8, 8, 512, 4, gv=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert bwd(1, 8, 8, 512, 4, g=None) != 0 and b'null pointer' in L.dbw_last_error()
    assert bwd(1, 8, 8, 512, 4, seed=None) != 0 and b'null pointer' in L.dbw_last_error()


# the GPU module's cases small enough for the CPU (the others differ in size, not in kind)
HOST_CASES = [n for n, c in M.CASES.items() if c.B * c.H * c.W <= 20000]


@functools.lru_cache(maxsize=None)
def float32_walk(name):
    """one case of the GPU module stepped in float32 on the CPU as that module steps the kernels (each step's float32
    result feeds the next; the convolutions on the tensor-core model M.TC32).  {kind: (worst error / bound, worst
    relative L2 against float64)}"""
    case = M.CASES[name]
    B, H, W = case.B, case.H, case.W
    in0, in1 = M.make_images(case, 'cpu')
    gv = M.grad_values(B, 'cpu')
    hw = M.level_sizes(H, W)
    out = {}

    def step(kind, fn, *args, dtype=torch.float32):
        """fn(*args, dtype) against fn(*args, float64): record the deviation, return the float32 result"""
        got = fn(*args, dtype)[0]
        want, bound = fn(*args, torch.float64)
        err = (got.double() - want).abs()
        assert bool((err <= bound).all()), (name, kind)
        r0, e0 = out.get(kind, (0.0, 0.0))
        out[kind] = (max(r0, float((err / bound.clamp_min(1e-300)).max())), max(e0, M.rel_l2(got, want)))
        return got

    def features(sd, x):
        acts = [step('first', M.oracle_first, x, sd, case.normalize)]
        for l in range(1, 13):
            a = acts[-1]
            if M.LEVEL[l] != M.LEVEL[l - 1]:
                a = F.max_pool2d(a, 2, 2)
            acts.append(step(M.kind_of(case, 'conv', l), M.oracle_conv, a, M.conv_weight(sd, l), sd[M.SLICE_KEY[l] + '.bias'],
                             True, None, dtype=M.TC32))
        return acts

    sd = M.dead5_state_dict(features(M.state_dict('base'), in1)[11]) if case.sd == 'dead5' else M.state_dict(case.sd)
    f0 = features(sd, in0)
    f0 = [f0[l] for l in M.TAP_LAYER]
    acts = features(sd, in1)
    lin = [sd[f'lin{k}.model.1.weight'].flatten() for k in range(5)]
    masks = [None] * 5
    if case.train:
        masks = [torch.from_numpy(OL.mask_np(case.seed, k, B, M.TAP_C[k], *hw[k])).permute(0, 2, 3, 1).reshape(B, -1, M.TAP_C[k])
                 for k in range(5)]
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(t.shape[0], -1, t.shape[1])          # noqa: E731  NCHW -> (n, P, C)
    parts = [step(M.kind_of(case, 'head', k), lambda *a: tuple(map(M.chunk_sums, M.oracle_head(*a))), flat(f0[k]), flat(acts[M.TAP_LAYER[k]]),
                  lin[k], masks[k]) for k in range(5)]
    step('value', M.oracle_value, parts, [h * w for h, w in hw])
    G = None
    for l in range(12, 0, -1):
        lv = M.LEVEL[l]
        if l == M.TAP_LAYER[lv]:
            g_in = None
            if lv < 4:
                x = acts[l].clone().requires_grad_(True)
                F.max_pool2d(x, 2, 2).backward(G)
                g_in = flat(x.grad)
            h, w = hw[lv]
            G = step(M.kind_of(case, 'head_bwd', lv), M.oracle_head_backward, flat(f0[lv]), flat(acts[l]), lin[lv], masks[lv], gv, g_in)
            G = G.view(B, h, w, -1).permute(0, 3, 1, 2)
        mask = None if M.LEVEL[l - 1] != lv else acts[l - 1]
        G = step('conv_bwd', M.oracle_conv, G, M.conv_weight(sd, l, bwd=True), None, False, mask, dtype=M.TC32)
    step('dgrad', M.oracle_dgrad, G, sd, case.normalize)
    return out


@functools.lru_cache(maxsize=None)
def value_deviation(name):
    """(worst error / bound, relative L2) of the value step in float32 at the chunk counts of every case, the large ones
    included: the deviation of an in-order sum grows with its length, and hardly depends on the positive partials summed"""
    case = M.CASES[name]
    hw = M.level_sizes(case.H, case.W)
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
    walks = [float32_walk(name) for name in HOST_CASES] + [{'value': value_deviation(name)} for name in M.CASES]
    for walk in walks:
        for kind, (r, e) in walk.items():
            r0, e0 = out.get(kind, (0.0, 0.0))
            out[kind] = (max(r0, r), max(e0, e))
    return out


@pytest.mark.parametrize('name', HOST_CASES)
def test_every_bound_holds_for_a_float32_evaluation(name):
    worst = float32_walk(name)                              # asserts every element of every step against its bound
    assert set(worst) <= set(M.BARS)
    assert all(ratio <= 1 for ratio, _ in worst.values()), worst


@pytest.mark.parametrize('kind', sorted(M.BARS))
def test_bar_sits_a_fixed_multiple_above_float32_rounding(kind):
    assert set(float32_deviations()) == set(M.BARS)
    dev, bar = float32_deviations()[kind][1], M.BARS[kind]
    assert HEADROOM * dev <= bar, f'{kind}: float32 deviates by {dev:.3g}; bar {bar:.3g} leaves less than {HEADROOM}x'
    assert bar <= 32 * dev, f'{kind}: bar {bar:.3g} is loose for a float32 deviation of {dev:.3g}'
