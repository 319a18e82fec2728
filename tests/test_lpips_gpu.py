"""GPU: the LPIPS kernels of csrc/dbw_lpips.cu against the float64 restatement of oracle/lpips.py.

Single layers are checked per element against the TF32-emulated oracle (the same rounded operands, products summed in
float64) within c * sum_k |a_k b_k|, the bound of an fp32 accumulation of K terms: c = 2 (K + 2) 2^-24 allows a
rounding (or a truncation, 2u) per addition.  The whole term is checked in relative terms, because 13 layers of fp32
activations re-rounded to TF32 can flip single roundings between the kernels and the oracle."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lpips as OL

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
U = 2.0 ** -24


def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from dbw_b200 import _lib
    return _lib


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


@pytest.fixture(scope='module')
def sd():
    return OL.random_state_dict(0)


@pytest.fixture(scope='module')
def net(sd):
    from dbw_b200.perceptual import LPIPS
    return LPIPS.from_state_dict(sd).to(DEV)


# ------------------------------------------------------------------------------------------------ single layers
SHAPES = [(64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 512), (512, 512),      # forward
          (128, 64), (256, 128), (512, 256)]                                                    # input gradient only


@pytest.mark.parametrize('B,H,W', [(1, 13, 21), (3, 11, 9)])
@pytest.mark.parametrize('ci,co', SHAPES)
def test_conv_layer_against_tf32_oracle(ci, co, B, H, W):
    from dbw_b200.perceptual import kmajor, tf32_round
    g = torch.Generator().manual_seed(ci * 7 + co + B)
    x = torch.randn(B, ci, H, W, generator=g).relu()
    w = torch.randn(co, ci, 3, 3, generator=g) * (2.0 / (9 * ci)) ** 0.5
    b = torch.randn(co, generator=g) * 0.1
    mask = torch.randn(B, co, H, W, generator=g)
    L = _lib()
    for use_bias, relu, use_mask in ((True, 1, False), (False, 0, True)):        # forward epilogue, input-gradient epilogue
        out = torch.empty(B, H, W, co, device=DEV)
        bb = b.to(DEV) if use_bias else None
        mm = nhwc(mask).to(DEV) if use_mask else None
        xd, wd = nhwc(x).to(DEV), kmajor(tf32_round(w)).to(DEV)        # held: the kernel runs after the call returns
        L.check(L.lib().dbw_lpips_conv3x3(_vp(xd), _vp(wd), _vp(bb), _vp(mm), _vp(out), B, H, W, ci, co, relu, _st()), 'conv3x3')
        xr, wr = OL.tf32(x.double()), OL.tf32(w.double())
        want = F.conv2d(xr, wr, b.double() if use_bias else None, padding=1)
        bound = OL.conv_abs_bound(xr, wr, b.double() if use_bias else None) * 2 * (9 * ci + 2) * U
        if relu:
            want = want.relu()
        if use_mask:
            want = want * (mask.double() > 0)
        got = nchw(out.cpu()).double()
        err = (got - want).abs()
        assert (err <= bound + 1e-30).all(), (ci, co, float((err / (bound + 1e-30)).max()))


@pytest.mark.parametrize('normalize', [True, False])
def test_first_layer_and_last_input_gradient(sd, normalize):
    L = _lib()
    g = torch.Generator().manual_seed(11)
    B, H, W = 3, 17, 23
    x = torch.rand(B, 3, H, W, generator=g)
    w, b = sd['net.slice1.0.weight'], sd['net.slice1.0.bias']
    shift, scale = sd['scaling_layer.shift'].flatten(), sd['scaling_layer.scale'].flatten()
    out = torch.empty(B, H, W, 64, device=DEV)
    xd, wd, bd, shd, scd = (t.to(DEV) for t in (x, w, b, shift, scale))
    L.check(L.lib().dbw_lpips_conv_first(_vp(xd), _vp(wd), _vp(bd), _vp(shd), _vp(scd), int(normalize), _vp(out), B, H, W, _st()),
            'conv_first')
    xs = ((2 * x.double() - 1) if normalize else x.double())
    xs = (xs - shift.double()[None, :, None, None]) / scale.double()[None, :, None, None]
    want = F.conv2d(xs, w.double(), b.double(), padding=1).relu()
    bound = OL.conv_abs_bound(xs, w.double(), b.double()) * 2 * (27 + 4) * U
    assert ((nchw(out.cpu()).double() - want).abs() <= bound).all()
    # the last input gradient: d rec = d x' * (2 if normalize) / scale
    gz = torch.randn(B, 64, H, W, generator=g)
    gin = torch.empty(B, 3, H, W, device=DEV)
    gzd = nhwc(gz).to(DEV)
    L.check(L.lib().dbw_lpips_dgrad_last(_vp(gzd), _vp(wd), _vp(scd), int(normalize), _vp(gin), B, H, W, _st()), 'dgrad_last')
    f = (2.0 if normalize else 1.0) / scale.double()[None, :, None, None]
    want = torch.nn.grad.conv2d_input((B, 3, H, W), w.double(), gz.double(), padding=1) * f
    bound = torch.nn.grad.conv2d_input((B, 3, H, W), w.double().abs(), gz.double().abs(), padding=1) * f * 2 * (576 + 4) * U
    assert ((gin.cpu().double() - want).abs() <= bound).all()


@pytest.mark.parametrize('H,W', [(7, 9), (8, 8), (75, 37), (3, 2)])
def test_maxpool_floor_and_dropped_rows(H, W):
    L = _lib()
    g = torch.Generator().manual_seed(H * W)
    B, C = 2, 64
    x = torch.randn(B, C, H, W, generator=g).relu()                      # post-ReLU values, zeros included
    out = torch.empty(B, H // 2, W // 2, C, device=DEV)
    xd = nhwc(x).to(DEV)
    L.check(L.lib().dbw_lpips_maxpool(_vp(xd), _vp(out), B, H, W, C, _st()), 'maxpool')
    xr = x.clone().requires_grad_(True)
    want = F.max_pool2d(xr, 2, 2)
    assert torch.equal(nchw(out.cpu()), want.detach())
    go = torch.randn(want.shape, generator=g)
    want.backward(go)
    gin = torch.full((B, H, W, C), float('nan'), device=DEV)
    god = nhwc(go).to(DEV)
    L.check(L.lib().dbw_lpips_maxpool_backward(_vp(xd), _vp(god), _vp(gin), B, H, W, C, _st()), 'pool bwd')
    got = nchw(gin.cpu())
    # windows of all zeros: torch routes to the first element, the kernel too; values are exact copies
    assert torch.equal(got, xr.grad)
    if H % 2:
        assert not got[:, :, H - 1].any()
    if W % 2:
        assert not got[:, :, :, W - 1].any()


# ------------------------------------------------------------------------------------------------ whole term
def _images(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g)
    return a, (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)


def _run(net, a, b, train, seed=1234, grad_value=None):
    net.train(train)
    net.seed.fill_(seed)
    x = b.to(DEV).requires_grad_(True)
    v = net(a.to(DEV), x, normalize=True)
    gv = torch.ones(v.shape[0]) if grad_value is None else grad_value
    (v.flatten() * gv.to(DEV)).sum().backward()
    return v.flatten().detach().cpu().double(), x.grad.cpu().double()


def _rel(a, b):
    return float((a - b).norm() / b.norm())


# thresholds.  Value: against the TF32-emulated oracle the kernels differ by fp32 accumulation and by the TF32
# roundings that an fp32 ulp of an activation flips (measured <= 3e-5 on an H100); against exact fp64, by TF32 itself.
# Gradient (relative L2): d value / d rec of a random VGG16 is ill-conditioned -- it passes 24 TF32 layers and every ReLU
# and pool decision, and those flip wherever fp32 and fp64 activations straddle 0 or tie.  Measured on an H100 80GB HBM3
# at 700 W: 1.2e-2 .. 3.5e-2 against the emulated oracle, 4.9e-2 against exact fp64 at 4 x 300x400, where cuDNN's own
# TF32 gradient of the same term is 4.9e-2 from exact fp64.  A missing term or a wrong mask is an O(1) error.
TOL = dict(tf32=dict(value=1e-4, grad=6e-2), exact=dict(value=1e-2, grad=1e-1))


@pytest.mark.parametrize('B,H,W', [(1, 300, 400), (1, 288, 384), (2, 64, 96), (2, 17, 23)])
@pytest.mark.parametrize('train', [False, True])
def test_whole_term_against_oracle(net, sd, B, H, W, train):
    a, b = _images(B, H, W, H + W)
    gv = torch.linspace(0.5, 1.5, B)
    v, g = _run(net, a, b, train, 1234, gv)
    assert int(net.seed.item()) == 1235                               # every forward advances the seed, eval mode too
    seed = 1234 if train else None
    for mode in ('tf32', 'exact'):
        wv, wg = OL.value_and_grad(sd, a.to(DEV), b.to(DEV), normalize=True, mode=mode, seed=seed, grad_value=gv)   # fp64
        wv, wg = wv.cpu(), wg.cpu()
        ev, eg = float(((v - wv).abs() / wv.abs()).max()), _rel(g, wg)
        print(f'{B}x{H}x{W} train={train} {mode}: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
        assert ev < TOL[mode]['value'] and eg < TOL[mode]['grad'], (mode, ev, eg)


def test_train_mode_mean_approaches_eval(net):
    """the heads are linear in the mask and E[mask] = 1, so E[value_train] = value_eval exactly"""
    a, b = _images(1, 17, 23, 5)
    net.eval()
    with torch.no_grad():
        ev = float(net(a.to(DEV), b.to(DEV), normalize=True))
        net.train()
        net.seed.fill_(0)
        vals = torch.stack([net(a.to(DEV), b.to(DEV), normalize=True).flatten() for _ in range(400)]).cpu().double()
    assert int(net.seed.item()) == 400
    assert len(set(vals.flatten().tolist())) > 390                   # fresh masks every call
    m, s = float(vals.mean()), float(vals.std())
    assert abs(m - ev) < 4 * s / 20, (m, ev, s)


def test_cuda_graph_replay_draws_fresh_masks(net):
    a, b = _images(2, 32, 48, 9)
    a, b = a.to(DEV), b.to(DEV)
    net.train()
    with torch.no_grad():
        net.seed.fill_(100)
        eager = [net(a, b, normalize=True).clone() for _ in range(3)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            net(a, b, normalize=True)                                # warm-up outside the graph
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = net(a, b, normalize=True)
        net.seed.fill_(100)
        replayed = []
        for _ in range(3):
            graph.replay()
            replayed.append(out.clone())
        torch.cuda.synchronize()
    assert int(net.seed.item()) == 103
    for e, r in zip(eager, replayed):
        assert torch.equal(e, r)
    assert not torch.equal(replayed[0], replayed[1])


def test_state_dict_round_trip_under_model_names(net):
    from dbw_b200.dbw import PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    holder = torch.nn.Module()
    holder.perceptual_loss = PerceptualTerm(net)
    state = holder.state_dict()
    assert all(k.startswith('perceptual_loss.loss.') for k in state)
    again = LPIPS.from_state_dict(state).to(DEV).eval()
    net.eval()
    a, b = _images(2, 40, 56, 3)
    with torch.no_grad():
        assert torch.equal(net(a.to(DEV), b.to(DEV), normalize=True), again(a.to(DEV), b.to(DEV), normalize=True))


@pytest.mark.parametrize('tap', range(5))
def test_each_tap_alone_against_oracle(sd, tap):
    """one head at a time (the other lin weights zeroed): a wrong gradient confined to one tap cannot hide behind the
    others' share of the gradient norm.  A deep tap alone averages over few pixels (relu5_3 is 4x6 here) after up to 12
    TF32 layers.  Measured on an H100 80GB HBM3 against the emulated oracle: values within 8.6e-4, gradients within
    6.9e-2 relative L2 (relu5_3; relu1_2 3e-5).  Bounds 2e-3 and 1.5e-1 keep a factor of 2; a wrong mask, channel
    or norm term in one head is an O(1) error."""
    from dbw_b200.perceptual import LPIPS
    one = dict(sd)
    for k in range(5):
        if k != tap:
            one[f'lin{k}.model.1.weight'] = torch.zeros_like(sd[f'lin{k}.model.1.weight'])
            one[f'lins.{k}.model.1.weight'] = one[f'lin{k}.model.1.weight']
    net1 = LPIPS.from_state_dict(one).to(DEV)
    a, b = _images(2, 64, 96, 31 + tap)
    for train in (False, True):
        v, g = _run(net1, a, b, train, 77)
        wv, wg = OL.value_and_grad(one, a.to(DEV), b.to(DEV), normalize=True, mode='tf32', seed=77 if train else None)
        ev, eg = float(((v - wv.cpu()).abs() / wv.cpu().abs()).max()), _rel(g, wg.cpu())
        print(f'tap {tap} train={train}: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
        assert ev < 2e-3 and eg < 1.5e-1, (tap, train, ev, eg)


def test_prepared_weights_are_the_rounded_forward_and_flipped_copies(net):
    """the device layout written by dbw_lpips_prepare_weights, element for element: per layer 1..12 the K-major forward
    copy [co][ky][kx][ci], then the input-gradient copy [ci][2-ky][2-kx][co], both TF32-rounded"""
    from dbw_b200.perceptual import dgrad_weight, kmajor, tf32_round
    net._prepare()
    prep = net.prepared.cpu()
    o = 0
    for conv in net.net.convs()[1:]:
        w = tf32_round(conv.weight.detach().cpu())
        for want in (kmajor(w), kmajor(dgrad_weight(w))):
            n = want.numel()
            assert torch.equal(prep[o:o + n].view_as(want), want)
            o += n
    assert o == prep.numel()


def test_forward_without_backward_keeps_only_the_taps(net):
    """under no_grad the forward keeps only rec's taps (a smaller workspace) and gives the same values bit for bit"""
    a, b = _images(2, 40, 56, 4)
    a, b = a.to(DEV), b.to(DEV)
    net.eval()
    assert net._bytes(2, 40, 56, False)[0] < net._bytes(2, 40, 56, True)[0]
    with torch.no_grad():
        v0 = net(a, b, normalize=True)
    v1 = net(a, b.clone().requires_grad_(True), normalize=True)
    assert torch.equal(v0, v1.detach())
