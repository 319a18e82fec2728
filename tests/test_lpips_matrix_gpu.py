"""GPU: the LPIPS term of csrc/dbw_lpips.cu one step at a time, each step against the float64 oracle on the kernel's own
float32 inputs.

Each case runs the real `dbw_lpips_forward(save_for_backward=1)` and `dbw_lpips_backward` on a workspace whose layout
(include/dbw_render.h) `layout` restates.  Then:

  forward   act[l] of the workspace against the float64 layer applied to the workspace's act[l-1] (max-pooled first where
            a pool sits in between; the pool itself, by `dbw_lpips_maxpool`, must equal F.max_pool2d bit for bit); imgs'
            taps against rec's taps of a second forward with in1 := in0, bit for bit;
  heads     `dbw_lpips_head_forward` on the workspace's taps and seed: its partials equal the forward's bit for bit, and
            each 64-pixel chunk is checked against the float64 head; value[b] against the float64 reduction of the
            kernel's own partials;
  backward  replayed with the single-step entries on the forward's workspace (head backward, maxpool_backward, the
            input-gradient conv3x3 with the `act[l-1] > 0` mask, dgrad_last).  The replay's gradient must equal the real
            call's bit for bit (the kernels are deterministic: a difference is orchestration), and every step is checked
            against the float64 step on the replay's input.

No ReLU or pool decision can differ from the oracle's, since both sides read the same fp32 tensors; each comparison is one
step deep.  At B = 49 the kernels run on the whole batch and the oracle on images 0, 24 and 48 (every step is per image).

Per-element bounds, u = 2^-24, all evaluated in float64 from the same float32 operands:

  conv      2 (K + 2) u sum_k |a_k b_k| (+ |bias|), K = 9 C_in, on the TF32-rounded operands (the kernel rounds the
            activation or incoming gradient as it leaves shared memory, the weights once): an fp32 accumulation of K terms
            errs by at most (K - 1) u sum |terms| with round-to-nearest; 2u per addition also admits the tensor cores'
            truncation, + 2 covers the bias and a last rounding.  ReLU and the [act > 0] mask are 1-Lipschitz and exact.
  first     2 (27 + 4) u sum |x' w| (+ |bias|): 27 FMAs after the scaling x' = (x - shift) / scale (2 roundings, 4 with
            normalize's 2x - 1).
  dgrad     2 (576 + 4) u sum |g w| / scale (* 2): 576 FMAs, then the chain factor (2 roundings).
  heads     first-order running error of the kernel's own arithmetic, doubled for the second-order terms.  With
            NPL = C / 32 terms per lane, a warp sum of squares s = ||f||^2 (NPL FMAs, a 5-level shuffle tree) errs by
            sigma s, sigma = (NPL + 5) u + (C + 31) eta / s (eta = 2^-150, the absolute error of a rounding into the
            subnormals); r = sqrt(s) by sigma / 2 + u; d = r + eps by delta_d = sigma / 2 + 2u; n = f / d by delta_d + u
            relative (+ eta); e = n0 - n1 by |dn0| + |dn1| + u |e|.  Forward: e^2 by 2 |e| |de| + u e^2, and the sum of
            |w| e^2 over the chunk passes NPL + 5 + 8 + 8 roundings (lane, warp tree, the warp's 8 pixels, the 8 warps).
            Backward: w * grad_value / HW carries 2u, q = -2 w e adds u; q / d1 by |dq| / d1 + |q / d1| (delta_d + u);
            dot = sum q u1 by sum |dq| |u1| + (NPL + 5) u sum |q u1| (+ (C + 31) eta); den = d1 d1 r1 by
            2 delta_d + sigma / 2 + 3u (+ eta / den); k = dot / den by |d dot| / den + |k| (delta_den + u); then
            u1 k, the difference and the accumulation one rounding each.
  value     2 (chunks_k + 7) u sum_k sum_c |partial_c| / (H_k W_k): the chunk sum in order, the fp32 1 / (H_k W_k) and its
            product, the five taps.
  pool      exact (forward and backward are selections).

A worst-case bound lets a small systematic error through (a 1e-3 scale of a layer sits well inside 2 (K + 2) u for
K = 4608).  So every array also meets a relative-L2 bar: BARS[kind], about 8 x the worst deviation of a CPU float32
evaluation of the same step over the arrays of that kind (tests/test_lpips_matrix_host.py checks that each bar sits between
4 x and 32 x it).  Arrays that cancel by construction have kinds of their own (`kind_of`), so that they do not set the bar
of the well-conditioned ones: layer 12 of 'dead5', whose bias nearly cancels the convolution; every head of 'near', where
n0 - n1 cancels; the relu5_3 head backward of 'dead5', whose nearly dead pixels divide by a tiny norm.  For the
convolutions the float32 evaluation models the tensor cores (TC32: 8 products per step into an accumulator truncated
toward zero), whose accumulation is coarser than round-to-nearest float32: on an H100 80GB HBM3 at 700 W, over this
module's cases, the kernels deviate from float64 by 10 to 25 x what a round-to-nearest float32 convolution does, and by
0.5 to 1 x what TC32 does.  The value is evaluated in float32 as the kernel sums it: each tap's partials in chunk
order."""
import ctypes
import functools
import time
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lpips as OL

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
U = 2.0 ** -24
ETA = 2.0 ** -150
EPS = float(np.float32(1e-10))            # the kernels' LP_EPS, as the float32 they add

# the network as csrc/dbw_lpips.cu lays it out
CIN = (3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512)
COUT = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
LEVEL = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)
TAP_LAYER = (1, 3, 6, 9, 12)
TAP_C = (64, 128, 256, 512, 512)
HEAD_PIX = 64
SLICE_KEY = ('net.slice1.0', 'net.slice1.2', 'net.slice2.5', 'net.slice2.7', 'net.slice3.10', 'net.slice3.12', 'net.slice3.14',
             'net.slice4.17', 'net.slice4.19', 'net.slice4.21', 'net.slice5.24', 'net.slice5.26', 'net.slice5.28')

# relative-L2 bars per step kind: about 8 x the worst deviation of the CPU float32 evaluation of
# tests/test_lpips_matrix_host.py over the arrays of that kind (the '_cancel' kinds: see `kind_of`)
BARS = {'first': 9e-7, 'conv': 1e-4, 'conv_bwd': 1.1e-4, 'dgrad': 1.3e-6, 'head': 1e-5, 'head_bwd': 3e-5, 'value': 1.1e-6,
        'conv_cancel': 6e-4, 'head_cancel': 6e-4, 'head_bwd_cancel': 4e-4}


# ------------------------------------------------------------------------------------------------ workspace layout
def _align64(n):
    return (n + 63) // 64 * 64


def level_sizes(H, W):
    return [(H >> k, W >> k) for k in range(5)]


def chunks(H, W):
    return (H * W + HEAD_PIX - 1) // HEAD_PIX


Layout = namedtuple('Layout', 'act tap0 s0 s1 partials part_off seed total')


def layout(B, H, W, save):
    """the workspace layout of include/dbw_render.h, offsets in floats (act[l] None where the region is absent)"""
    hw = level_sizes(H, W)
    o, act = 0, []
    for l in range(13):
        if not save and l not in TAP_LAYER:
            act.append(None)
            continue
        h, w = hw[LEVEL[l]]
        act.append(o)
        o += _align64(B * h * w * COUT[l])
    tap0 = []
    for k in range(5):
        tap0.append(o)
        o += _align64(B * hw[k][0] * hw[k][1] * TAP_C[k])
    big = _align64(B * H * W * 64)
    s0, s1 = o, o + big
    o += 2 * big
    partials, part_off, p = o, [], 0
    for k in range(5):
        part_off.append(p)
        p += B * chunks(*hw[k])
    o += _align64(p)
    seed = o
    return Layout(tuple(act), tuple(tap0), s0, s1, partials, tuple(part_off), seed, o + 64)


# ------------------------------------------------------------------------------------------------ float64 steps
# Every oracle step takes the kernel's float32 inputs (NCHW for the convolutions, (n, P, C) for the heads) and returns the
# step in `dtype` (float64 here; float32 for the deviations of the host module) and its per-element bound in float64.
def conv_weight(sd, l, bwd=False):
    """the TF32-rounded weight of layer l (1..12) as the kernels hold it: the forward copy, or the input-gradient copy
    W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx]"""
    w = sd[SLICE_KEY[l] + '.weight'].double()
    return OL.tf32(w.flip(2, 3).transpose(0, 1) if bwd else w)


TC32 = 'tc32'


def _conv_tc32(xr, wr, b):
    """a float32 model of the tensor cores' accumulation: the products of the TF32 operands summed 8 at a time (one mma
    k-step, in the kernel's K order (ky, kx, ci)) into an fp32 accumulator truncated toward zero; the bias then added with
    rounding to nearest, as the epilogue adds it"""
    n, C, h, w = xr.shape
    A = F.unfold(xr, 3, padding=1).view(n, C, 9, h * w).permute(0, 3, 2, 1).reshape(n * h * w, 9 * C)
    Wk = wr.permute(0, 2, 3, 1).reshape(wr.shape[0], 9 * C)
    acc = torch.zeros(n * h * w, wr.shape[0], dtype=torch.float64, device=xr.device)
    for j in range(0, 9 * C, 8):
        s = acc + A[:, j:j + 8] @ Wk[:, j:j + 8].T
        t = s.float()
        acc = torch.where(t.double().abs() > s.abs(), torch.nextafter(t, torch.zeros_like(t)), t).double()
    out = acc.float() if b is None else acc.float() + b.float()
    return out.view(n, h, w, -1).permute(0, 3, 1, 2)


def oracle_conv(x, wr, bias, relu, mask, dtype):
    """one tensor-core layer: x (n, C_in, h, w) fp32 values, wr TF32-rounded; mask (n, C_out, h, w) or None.  dtype TC32:
    the float32 model of the tensor cores (the host module's float32 evaluation)"""
    xr = OL.tf32(x.double())
    dev = x.device
    wr = wr.to(dev)
    b = None if bias is None else bias.to(dev).double()
    if dtype == TC32:
        out = _conv_tc32(xr, wr, b)
    else:
        out = F.conv2d(xr.to(dtype), wr.to(dtype), None if b is None else b.to(dtype), padding=1)
    bound = OL.conv_abs_bound(xr, wr, b) * (2 * (9 * x.shape[1] + 2) * U)
    if relu:
        out = out.relu()
    if mask is not None:
        keep = mask > 0
        out, bound = out * keep, bound * keep
    return out, bound


def oracle_first(x, sd, normalize, dtype):
    dev = x.device
    w, b = sd['net.slice1.0.weight'].to(dev).double(), sd['net.slice1.0.bias'].to(dev).double()
    shift, scale = (sd[f'scaling_layer.{n}'].to(dev).double().view(1, 3, 1, 1) for n in ('shift', 'scale'))
    xs = 2 * x.double() - 1 if normalize else x.double()
    xs = (xs - shift) / scale
    out = F.conv2d(xs.to(dtype), w.to(dtype), b.to(dtype), padding=1).relu()
    return out, OL.conv_abs_bound(xs, w, b) * (2 * (27 + 4) * U)


def oracle_dgrad(gz, sd, normalize, dtype):
    """the last input gradient: gz (n, 64, H, W) -> d rec (n, 3, H, W)"""
    dev = gz.device
    w = sd['net.slice1.0.weight'].to(dev).double()
    f = (2.0 if normalize else 1.0) / sd['scaling_layer.scale'].to(dev).double().view(1, 3, 1, 1)
    shape = (gz.shape[0], 3, gz.shape[2], gz.shape[3])
    out = torch.nn.grad.conv2d_input(shape, w.to(dtype), gz.to(dtype), padding=1) * f.to(dtype)
    bound = torch.nn.grad.conv2d_input(shape, w.abs(), gz.double().abs(), padding=1) * f * (2 * (576 + 4) * U)
    return out, bound


def _normed(f, dtype):
    """s = ||f||^2, r, d = r + eps, n = f / d of (n, P, C) features, in dtype"""
    f = f.to(dtype)
    s = (f * f).sum(-1, keepdim=True)
    r = s.sqrt()
    d = r + EPS
    return s, r, d, f / d


def _norm_errors(f):
    """float64 (sigma, delta_d, |dn|) of the kernel's normalisation of f (n, P, C): see the module docstring"""
    C = f.shape[-1]
    s, r, d, n = _normed(f, torch.float64)
    sigma = (C // 32 + 5) * U + torch.where(s > 0, (C + 31) * ETA / s.clamp_min(1e-300), torch.zeros_like(s))
    delta_d = sigma / 2 + 2 * U
    return sigma, delta_d, (delta_d + U) * n.abs() + ETA


def _wmask(lin, mask, dtype):
    """the head's channel weights per element: lin, or lin * {0, 2} in training"""
    w = lin.to(dtype).view(1, 1, -1)
    return w if mask is None else w * mask.to(dtype)


def oracle_head(f0, f1, lin, mask, dtype):
    """per-pixel head sum_j w_j (n0_j - n1_j)^2 of (n, P, C) features: (values (n, P) in dtype, bounds (n, P))"""
    C = f0.shape[-1]
    n0, n1 = _normed(f0, dtype)[3], _normed(f1, dtype)[3]
    e = n0 - n1
    val = (_wmask(lin, mask, dtype) * e * e).sum(-1)
    e64 = _normed(f0, torch.float64)[3] - _normed(f1, torch.float64)[3]
    de = _norm_errors(f0)[2] + _norm_errors(f1)[2] + U * e64.abs()
    aw = _wmask(lin, mask, torch.float64).abs()
    bound = 2 * (aw * ((C // 32 + 22) * U * e64 * e64 + 2 * e64.abs() * de + ETA)).sum(-1)
    return val, bound


def chunk_sums(per_pixel):
    """(n, P) -> (n, ceil(P / 64)): the 64-pixel chunks of the head CTAs"""
    n, P = per_pixel.shape
    c = chunks(P, 1)
    return F.pad(per_pixel, (0, c * HEAD_PIX - P)).view(n, c, HEAD_PIX).sum(-1)


def oracle_head_backward(f0, f1, lin, mask, gv, g_in, dtype):
    """(d sum_b gv[b] mean_p head / d f1 + g_in) * [f1 > 0] of (n, P, C) features, gv (n,), g_in (n, P, C) or None"""
    C, P = f0.shape[-1], f0.shape[1]

    def grad(dt):
        s1, r1, d1, n1 = _normed(f1, dt)
        e = _normed(f0, dt)[3] - n1
        u1 = f1.to(dt)
        q = -2 * _wmask(lin, mask, dt) * (gv.to(dt) / P).view(-1, 1, 1) * e
        dot = (q * u1).sum(-1, keepdim=True)
        k = torch.where(r1 > 0, dot / (d1 * d1 * r1), torch.zeros_like(dot))
        v = q / d1 - u1 * k
        return v, q, dot, k, d1, r1, e

    v, *_ = grad(dtype)
    if g_in is not None:
        v = v + g_in.to(dtype)
    v = v * (f1 > 0)
    v64, q, dot, k, d1, r1, e = grad(torch.float64)
    u1 = f1.double()
    sigma1, dd1 = _norm_errors(f1)[:2]
    de = _norm_errors(f0)[2] + _norm_errors(f1)[2] + U * e.abs()
    dq = (2 * _wmask(lin, mask, torch.float64) * (gv.double() / P).view(-1, 1, 1)).abs() * (de + 3 * U * e.abs())
    da = dq / d1 + (q / d1).abs() * (dd1 + U)
    ddot = (dq * u1.abs()).sum(-1, keepdim=True) + (C // 32 + 5) * U * (q * u1).abs().sum(-1, keepdim=True) + (C + 31) * ETA
    den = d1 * d1 * r1
    dden = 2 * dd1 + sigma1 / 2 + 3 * U + ETA / den.clamp_min(1e-300)
    dk = torch.where(r1 > 0, ddot / den.clamp_min(1e-300) + k.abs() * (dden + U), torch.zeros_like(k))
    db = u1.abs() * dk + U * (u1 * k).abs() + ETA
    bound = da + db + U * v64.abs() + ETA
    if g_in is not None:
        bound = bound + U * (v64 + g_in.double()).abs() + ETA
    return v, 2 * bound * (f1 > 0)


def oracle_value(parts, hw, dtype):
    """value per image from the kernel's partials [(n, chunks_k)] * 5 and the tap sizes H_k W_k, summed in dtype as the
    kernel sums: each tap's partials in chunk order, times 1 / (H_k W_k) rounded to dtype, the taps in order"""
    val = sum(p.to(dtype).cumsum(-1)[..., -1] * torch.tensor(1 / n, dtype=dtype) for p, n in zip(parts, hw))
    bound = 2 * U * sum((p.shape[-1] + 7) * p.double().abs().sum(-1) / n for p, n in zip(parts, hw))
    return val, bound


def rel_l2(got, want):
    d, n = float((got.double() - want.double()).norm()), float(want.double().norm())
    return d / n if n > 0 else (0.0 if d == 0 else float('inf'))


# ------------------------------------------------------------------------------------------------ state dicts and inputs
@functools.lru_cache(maxsize=None)
def state_dict(kind):
    """'base': oracle/lpips.py's random weights; 'tiny': layer 12 scaled by 1e-20 (|relu5_3| ~ 1e-20, d1 d1 r1 subnormal);
    'linzero': every other lin weight exactly 0 ('dead5' is built per case from the base weights)"""
    sd = OL.random_state_dict(0)
    if kind == 'tiny':
        for n in ('weight', 'bias'):
            sd[f'{SLICE_KEY[12]}.{n}'] = sd[f'{SLICE_KEY[12]}.{n}'] * 1e-20
    elif kind == 'linzero':
        for k in range(5):
            w = sd[f'lin{k}.model.1.weight'].clone()
            w.view(-1)[::2] = 0.0
            sd[f'lin{k}.model.1.weight'] = sd[f'lins.{k}.model.1.weight'] = w
    return sd


def make_net(sd):
    from dbw_b200.perceptual import LPIPS
    net = LPIPS.from_state_dict(sd).to(DEV)
    net._prepare()
    return net


@functools.lru_cache(maxsize=None)
def _net(kind):
    return make_net(state_dict(kind))


def make_images(case, device=DEV):
    B, H, W = case.B, case.H, case.W
    g = torch.Generator().manual_seed(B * 100003 + H * 101 + W)
    if case.inputs == 'constant':
        a = torch.full((B, 3, H, W), 0.3)
        b = torch.full((B, 3, H, W), 0.7)
        b[:, 1] = 0.2
    else:
        a = torch.rand(B, 3, H, W, generator=g)
        if case.inputs == 'same':
            b = a.clone()
        elif case.inputs == 'near':
            b = (a + 1e-6 * (2 * torch.rand(B, 3, H, W, generator=g) - 1)).clamp(0, 1)
        else:
            b = (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)
    return a.to(device), b.to(device)


def grad_values(B, device=DEV):
    """non-unit, zero and negative entries"""
    return torch.tensor([[1.5, -0.75, 0.0, 1.0, 0.25][b % 5] for b in range(B)], dtype=torch.float32, device=device)


# ------------------------------------------------------------------------------------------------ C-ABI calls
def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    from dbw_b200 import _lib
    _lib.check(getattr(_lib.lib(), name)(*args), name)


def run_forward(net, in0, in1, normalize, train, seed):
    """the real forward with save_for_backward: (workspace (floats), value, seed buffer after the call)"""
    B, _, H, W = in1.shape
    Lw = layout(B, H, W, True)
    ws = torch.full((Lw.total,), float('nan'), device=DEV)
    value = torch.full((B,), float('nan'), device=DEV)
    sbuf = torch.tensor([seed], dtype=torch.int64).to(torch.int32).to(DEV)       # uint32 bits in an int32
    s = ctypes.byref(net._net_struct())
    _call('dbw_lpips_forward', s, _vp(in0), _vp(in1), B, H, W, int(normalize), int(train), 1, _vp(sbuf), _vp(value), _vp(ws),
          Lw.total * 4, _st())
    return ws, value, sbuf


def act_view(ws, Lw, l, B, H, W):
    h, w = level_sizes(H, W)[LEVEL[l]]
    return ws[Lw.act[l]:Lw.act[l] + B * h * w * COUT[l]].view(B, h, w, COUT[l])


def tap0_view(ws, Lw, k, B, H, W):
    h, w = level_sizes(H, W)[k]
    return ws[Lw.tap0[k]:Lw.tap0[k] + B * h * w * TAP_C[k]].view(B, h, w, TAP_C[k])


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ cases
Case = namedtuple('Case', 'B H W normalize train seed inputs sd images', defaults=('random', 'base', None))
CASES = {
    # relu5_3 is 1x1; every tap below relu1_2 fits one head chunk; level 0 is M = 256 = 2 conv tiles exactly
    '1x16x16': Case(1, 16, 16, True, True, 0),
    '2x17x23': Case(2, 17, 23, False, False, 0x7fffffff),            # odd floors at every pool
    '3x33x47': Case(3, 33, 47, True, True, 0xffffffff),
    'wide': Case(2, 16, 1024, True, True, 5),                       # relu5_3 1x64: one full chunk
    'tall': Case(2, 1024, 16, True, False, 6),
    # M = 1921 = 15 * 128 + 1 (a 1-row conv tile) and H W = 1921 = 30 * 64 + 1 (a 1-pixel head chunk) at level 0
    '1x17x113': Case(1, 17, 113, False, True, 0xffffffff),
    '1x300x400': Case(1, 300, 400, True, True, 1234),
    '4x300x400': Case(4, 300, 400, True, True, 0x7fffffff),           # the training shape
    '49x400x400': Case(49, 400, 400, True, True, 3, images=(0, 24, 48)),
    'same': Case(2, 17, 23, True, True, 11, inputs='same'),         # e = 0: value and gradient exactly 0
    'near': Case(2, 33, 47, True, False, 12, inputs='near'),        # in1 within 1e-6 of in0: cancellation in e
    'constant': Case(2, 32, 48, True, True, 13, inputs='constant'),  # ties in the pool windows
    'dead5': Case(2, 64, 96, True, False, 14, sd='dead5'),          # relu5_3 all zero at some pixels (r1 == 0)
    'tiny': Case(2, 33, 47, True, True, 15, sd='tiny'),
    'linzero': Case(2, 17, 23, False, True, 16, sd='linzero'),
}

WORST = {}


def kind_of(case, kind, k):
    """the bar kind of the array of step `kind` at layer or tap k of `case`: the arrays that cancel by construction
    (see the module docstring) get a '_cancel' kind"""
    if (kind == 'conv' and case.sd == 'dead5' and k == 12) or (kind in ('head', 'head_bwd') and case.inputs == 'near') or \
            (kind == 'head_bwd' and case.sd == 'dead5' and k == 4):
        return kind + '_cancel'
    return kind


@pytest.fixture(scope='module', autouse=True)
def _report():
    torch.cuda.init()
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    print(f'\n{time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.1f} GiB allocated; '
          'worst error / bound and relative L2 per step kind over the cases:')
    for kind, (ratio, rel) in sorted(WORST.items()):
        print(f'  {kind:9s} error/bound {ratio:.3f}   rel L2 {rel:.2e} (bar {BARS.get(kind, 0):.0e})')


def dead5_state_dict(act11):
    """the base weights with a layer-12 bias that zeroes every relu5_3 channel at about half of the pixels of rec, whose
    relu5_2 is act11 (n, 512, h, w)"""
    sd = dict(state_dict('base'))
    z = F.conv2d(act11.double(), sd[SLICE_KEY[12] + '.weight'].to(act11.device).double(), padding=1).amax(1)
    sd[SLICE_KEY[12] + '.bias'] = torch.full((512,), -float(z.flatten().median()), dtype=torch.float32)
    return sd


class Checker:
    def __init__(self, name):
        self.name, self.worst = name, {}

    def __call__(self, kind, got, want, bound, where=''):
        got, want = got.double(), want.double()
        err = (got - want).abs()
        ok = err <= bound                                          # NaN fails
        ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
        rel = rel_l2(got, want)
        assert bool(ok.all()), f'{self.name} {kind} {where}: {int((~ok).sum())} elements outside the bound, worst ratio {ratio:.3g}'
        assert rel <= BARS[kind], f'{self.name} {kind} {where}: relative L2 {rel:.3g} above {BARS[kind]:.1g}'
        for d in (self.worst, WORST):
            r0, e0 = d.get(kind, (0.0, 0.0))
            d[kind] = (max(r0, ratio), max(e0, rel))


@pytest.mark.parametrize('name', list(CASES))
def test_term_step_by_step_against_float64(name):
    case = CASES[name]
    B, H, W, normalize, train, seed = case.B, case.H, case.W, case.normalize, case.train, case.seed
    in0, in1 = make_images(case)
    if case.sd == 'dead5':
        ws = run_forward(_net('base'), in1, in1, True, False, 0)[0]
        sd = dead5_state_dict(nchw(act_view(ws, layout(B, H, W, True), 11, B, H, W)))
        del ws
        net = make_net(sd)
    else:
        sd, net = state_dict(case.sd), _net(case.sd)
    idx = torch.tensor(case.images if case.images else range(B), device=DEV)
    n_img = len(idx)
    hw = level_sizes(H, W)
    Lw = layout(B, H, W, True)
    check = Checker(name)
    gv = grad_values(B)

    ws, value, sbuf = run_forward(net, in0, in1, normalize, train, seed)
    grad_real = torch.full((B, 3, H, W), float('nan'), device=DEV)
    _call('dbw_lpips_backward', ctypes.byref(net._net_struct()), _vp(gv), B, H, W, int(normalize), int(train), _vp(grad_real),
          _vp(ws), Lw.total * 4, _st())
    seed_slot = ws[Lw.seed:Lw.seed + 1]
    assert int(seed_slot.view(torch.int32).item()) & 0xffffffff == seed
    assert int(sbuf.item()) & 0xffffffff == (seed + 1) & 0xffffffff            # the int32 sign flip and the uint32 wrap

    # ---- forward: every layer from the workspace's previous layer
    A = lambda l: act_view(ws, Lw, l, B, H, W)                                     # noqa: E731
    check('first', nchw(A(0)[idx]), *oracle_first(in1[idx], sd, normalize, torch.float64), 'layer 0')
    for l in range(1, 13):
        x = A(l - 1)
        if LEVEL[l] != LEVEL[l - 1]:
            h, w = hw[LEVEL[l - 1]]
            pooled = torch.full((B, h // 2, w // 2, CIN[l]), float('nan'), device=DEV)
            _call('dbw_lpips_maxpool', _vp(x), _vp(pooled), B, h, w, CIN[l], _st())
            assert torch.equal(nchw(pooled[idx]), F.max_pool2d(nchw(x[idx]), 2, 2)), f'{name}: pool before layer {l}'
            x = pooled
        want, bound = oracle_conv(nchw(x[idx]), conv_weight(sd, l), sd[SLICE_KEY[l] + '.bias'], True, None, torch.float64)
        check(kind_of(case, 'conv', l), nchw(A(l)[idx]), want, bound, f'layer {l}')
        del x, want, bound
    # imgs keeps only its taps: they are rec's taps of a forward with in1 := in0
    ws2 = run_forward(net, in0, in0, normalize, train, seed)[0]
    for k in range(5):
        assert torch.equal(tap0_view(ws, Lw, k, B, H, W), act_view(ws2, Lw, TAP_LAYER[k], B, H, W)), f'{name}: imgs tap {k}'
    del ws2

    # ---- heads and the value
    seed_used = int(seed_slot.view(torch.int32).item()) & 0xffffffff
    lin = [sd[f'lin{k}.model.1.weight'].flatten().to(DEV) for k in range(5)]
    masks = [None] * 5
    if train:
        masks = [torch.from_numpy(OL.mask_np(seed_used, k, B, TAP_C[k], *hw[k], images=idx.tolist())).to(DEV)
                 .permute(0, 2, 3, 1).reshape(n_img, -1, TAP_C[k]) for k in range(5)]
    parts = []
    for k in range(5):
        h, w = hw[k]
        f0, f1 = tap0_view(ws, Lw, k, B, H, W), A(TAP_LAYER[k])
        part = torch.full((B, chunks(h, w)), float('nan'), device=DEV)
        _call('dbw_lpips_head_forward', _vp(f0), _vp(f1), _vp(lin[k]), B, h, w, TAP_C[k], k, int(train), _vp(seed_slot),
              _vp(part), _st())
        o = Lw.partials + Lw.part_off[k]
        assert torch.equal(part.flatten(), ws[o:o + part.numel()]), f'{name}: head {k} partials differ from the forward'
        val, bnd = oracle_head(f0[idx].reshape(n_img, h * w, -1), f1[idx].reshape(n_img, h * w, -1), lin[k], masks[k],
                               torch.float64)
        check(kind_of(case, 'head', k), part[idx], chunk_sums(val), chunk_sums(bnd), f'tap {k}')
        parts.append(part[idx])
    check('value', value[idx], *oracle_value(parts, [h * w for h, w in hw], torch.float64))
    if case.inputs == 'same':
        assert not value.any()

    # ---- backward, replayed with the single-step entries
    prep = net.prepared
    G = None
    for l in range(12, 0, -1):
        lv = LEVEL[l]
        h, w = hw[lv]
        act = A(l)
        if l == TAP_LAYER[lv]:
            if lv < 4:
                gin = torch.full((B, h, w, COUT[l]), float('nan'), device=DEV)
                _call('dbw_lpips_maxpool_backward', _vp(act), _vp(G), _vp(gin), B, h, w, COUT[l], _st())
                x = nchw(act[idx]).contiguous().requires_grad_(True)
                F.max_pool2d(x, 2, 2).backward(nchw(G[idx]))
                assert torch.equal(nchw(gin[idx]), x.grad), f'{name}: pool backward after layer {l}'
                G, g_in = gin, gin[idx].reshape(n_img, h * w, -1).clone()
            else:
                G, g_in = torch.full((B, h, w, COUT[l]), float('nan'), device=DEV), None
            f0 = tap0_view(ws, Lw, lv, B, H, W)
            _call('dbw_lpips_head_backward', _vp(f0), _vp(act), _vp(lin[lv]), B, h, w, TAP_C[lv], lv, int(train),
                  _vp(seed_slot), _vp(gv), int(lv < 4), _vp(G), _st())
            want, bound = oracle_head_backward(f0[idx].reshape(n_img, h * w, -1), act[idx].reshape(n_img, h * w, -1), lin[lv],
                                               masks[lv], gv[idx], g_in, torch.float64)
            check(kind_of(case, 'head_bwd', lv), G[idx].reshape(n_img, h * w, -1), want, bound, f'tap {lv}')
            del want, bound, g_in
        after_pool = LEVEL[l - 1] != lv
        mask = None if after_pool else A(l - 1)
        out = torch.full((B, h, w, CIN[l]), float('nan'), device=DEV)
        n_w = 9 * CIN[l] * COUT[l]
        o = sum(2 * 9 * CIN[i] * COUT[i] for i in range(1, l)) + n_w                 # the input-gradient copy of layer l
        _call('dbw_lpips_conv3x3', _vp(G), _vp(prep[o:o + n_w]), None, _vp(mask), _vp(out), B, h, w, COUT[l], CIN[l], 0, _st())
        want, bound = oracle_conv(nchw(G[idx]), conv_weight(sd, l, bwd=True), None, False,
                                  None if mask is None else nchw(mask[idx]), torch.float64)
        check('conv_bwd', nchw(out[idx]), want, bound, f'layer {l}')
        G = out
        del want, bound
    grad = torch.full((B, 3, H, W), float('nan'), device=DEV)
    _call('dbw_lpips_dgrad_last', _vp(G), _vp(net.net.convs()[0].weight), _vp(net.scaling_layer.scale), int(normalize), _vp(grad),
          B, H, W, _st())
    check('dgrad', grad[idx], *oracle_dgrad(nchw(G[idx]), sd, normalize, torch.float64))
    assert torch.equal(grad, grad_real), f'{name}: the replayed backward differs from dbw_lpips_backward'
    if case.inputs == 'same':
        assert not grad_real.any()
    if case.sd == 'dead5':
        r1 = A(12).abs().amax(-1)
        assert bool((r1 == 0).any()) and bool((r1 > 0).any()), 'no pixel of relu5_3 is all zero'
    print(f'{name}: ' + ', '.join(f'{k} {r:.3f} / {e:.1e}' for k, (r, e) in sorted(check.worst.items())))
    torch.cuda.synchronize()
