"""Times the LPIPS kernels (csrc/dbw_lpips.cu) and prints one JSON line with the card's name and power limit:

  layers   each 3x3 convolution shape of the VGG16 trunk at the DTU training shape (4 x 300x400 before the pools), forward
           and input gradient: kernel time (CUDA events), TFLOP/s from shapes and the share of the 495 TFLOP/s dense TF32
           of the H100 SXM data sheet; beside it F.conv2d with bias (cuDNN, allow_tf32) on the same tensors, NCHW and
           channels_last, alternating with the kernel in one process.  The kernel's time includes its fused bias + ReLU
           epilogue; cuDNN's includes the bias but not a ReLU (that would be one more elementwise kernel)
  term     LPIPS forward + backward (d/d rec) at 4 x 300x400 and 49 x 400x400 (the bench.py shape), the kernels against
           the same term restated in torch (cuDNN, TF32, oracle/lpips.py in float32 with its weights resident on the GPU),
           NCHW and channels_last
  step     one training step of the scene model at 4 x 300x400 (model(inp) + backward, coarse phase, 10 blocks): with the
           built-in LPIPS term at weight 0.1, and with the RGB loss alone (the fused loss epilogue)

--check compares the term's value and gradient of both with the float64 oracle at 4 x 300x400 (eval mode).

    python scripts/bench_lpips.py [--check] [--repeat 20]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import warnings

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TF32 = 495e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def timed(fn, repeat):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeat):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeat


def layers(repeat):
    from dbw_b200 import _lib
    from dbw_b200.perceptual import kmajor, tf32_round
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    B, rows = 4, []
    for ci, co, h, w in ((64, 64, 300, 400), (64, 128, 150, 200), (128, 128, 150, 200), (128, 256, 75, 100), (256, 256, 75, 100),
                         (256, 512, 37, 50), (512, 512, 37, 50), (512, 512, 18, 25),
                         (128, 64, 150, 200), (256, 128, 75, 100), (512, 256, 37, 50)):
        x = torch.randn(B, h, w, ci, device='cuda').relu_()
        wt = torch.randn(co, ci, 3, 3, device='cuda') * (2.0 / (9 * ci)) ** 0.5
        bias = torch.randn(co, device='cuda') * 0.1
        km = kmajor(tf32_round(wt))
        out = torch.empty(B, h, w, co, device='cuda')
        x_nchw, x_cl = x.permute(0, 3, 1, 2).contiguous(), x.permute(0, 3, 1, 2)
        w_cl = wt.contiguous(memory_format=torch.channels_last)

        def ours():
            _lib.check(_lib.lib().dbw_lpips_conv3x3(vp(x), vp(km), vp(bias), None, vp(out), B, h, w, ci, co, 1, st), 'conv3x3')
        t = dict(ours=[], nchw=[], channels_last=[])
        for _ in range(3):                               # alternate
            t['ours'].append(timed(ours, repeat))
            t['nchw'].append(timed(lambda: F.conv2d(x_nchw, wt, bias, padding=1), repeat))
            t['channels_last'].append(timed(lambda: F.conv2d(x_cl, w_cl, bias, padding=1), repeat))
        flop = 2.0 * B * h * w * co * 9 * ci
        ms = {k: min(v) for k, v in t.items()}
        rows.append(dict(C_in=ci, C_out=co, HxW=f'{h}x{w}', ms=round(ms['ours'], 4), tflops=round(flop / ms['ours'] / 1e9, 1),
                         share_of_tf32_peak=round(flop / ms['ours'] / 1e-3 / PEAK_TF32, 3),
                         cudnn_nchw_ms=round(ms['nchw'], 4), cudnn_channels_last_ms=round(ms['channels_last'], 4)))
        print(json.dumps(rows[-1]), file=sys.stderr)
    return rows


def term(B, H, W, repeat, sd, check):
    from oracle import lpips as OL
    from dbw_b200.perceptual import LPIPS
    net = LPIPS.from_state_dict(sd).cuda().eval()
    # the restatement's weights live on the GPU, in each memory format, before anything is timed
    sd_nchw = {k: v.cuda() for k, v in sd.items()}
    sd_cl = {k: v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v for k, v in sd_nchw.items()}
    g = torch.Generator().manual_seed(B)
    a = torch.rand(B, 3, H, W, generator=g)
    b = (a + 0.2 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)
    a, b = a.cuda(), b.cuda()
    res = {}

    def ours():
        x = b.detach().requires_grad_(True)
        v = net(a, x, normalize=True)
        v.sum().backward()
        return v.detach().flatten(), x.grad

    def cudnn(channels_last=False):
        x = b.detach().requires_grad_(True)
        v = OL.lpips(sd_cl if channels_last else sd_nchw, a, x, normalize=True, dtype=torch.float32, channels_last=channels_last)
        v.sum().backward()
        return v.detach().flatten(), x.grad
    t_o, t_c, t_cl = [], [], []
    for _ in range(3):
        t_o.append(timed(ours, repeat))
        t_c.append(timed(cudnn, repeat))
        t_cl.append(timed(lambda: cudnn(True), repeat))
    res.update(shape=f'{B}x{H}x{W}', ms=round(min(t_o), 3), cudnn_nchw_ms=round(min(t_c), 3),
               cudnn_channels_last_ms=round(min(t_cl), 3),
               tflop=round(3 * 2 * B * sum(9 * ci * co * (H >> lv) * (W >> lv) for ci, co, lv in (
                   (3, 64, 0), (64, 64, 0), (64, 128, 1), (128, 128, 1), (128, 256, 2), (256, 256, 2), (256, 256, 2),
                   (256, 512, 3), (512, 512, 3), (512, 512, 3), (512, 512, 4), (512, 512, 4), (512, 512, 4))) / 1e12, 2))
    if check:
        vo, go = ours()
        vc, gc = cudnn(True)
        vx, gx = OL.value_and_grad(sd_nchw, a, b, normalize=True, mode='exact')
        rel = lambda u, w: float((u.double() - w).norm() / w.norm())
        res.update(value_rel_err=rel(vo, vx), grad_rel_err=rel(go, gx), cudnn_value_rel_err=rel(vc, vx), cudnn_grad_rel_err=rel(gc, gx))
    torch.cuda.empty_cache()
    return res


def step(repeat, sd):
    """ms of model(inp) + backward at 4 x 300x400, with the LPIPS term and without it"""
    from oracle import dbw_path as D
    from dbw_b200.dbw import DifferentiableBlocksWorld, PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    cfg = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
           'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
           'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                          'decouple_rendering': True, 'opacity_noise': False},
           'loss': {'rgb_weight': 1, 'perceptual_weight': 0.1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1}}
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')                      # the lpips package is absent: the term starts dropped
        model = DifferentiableBlocksWorld((300, 400), **cfg).to(torch.device('cuda')).train()
    B = 4
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=1)
    g = torch.Generator().manual_seed(1)
    inp = {'imgs': torch.rand(B, 3, 300, 400, generator=g).cuda(), 'R': R.float().cuda(), 'T': T.float().cuda(),
           'K': K.float()[None].expand(B, -1, -1).cuda()}

    def one():
        model.zero_grad(set_to_none=True)
        model(inp)['total'].backward()
    res = {'shape': f'{B}x300x400'}
    t_with, t_without = [], []
    term = PerceptualTerm(LPIPS.from_state_dict(sd)).cuda()
    for _ in range(3):
        model.set_perceptual_loss(term)
        t_with.append(timed(one, repeat))
        model.set_perceptual_loss(None)
        t_without.append(timed(one, repeat))
    res.update(with_lpips_ms=round(min(t_with), 3), rgb_only_ms=round(min(t_without), 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true')
    ap.add_argument('--repeat', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lpips.py needs a GPU')
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    from oracle import lpips as OL
    sd = OL.random_state_dict(0)
    name, watts = card()
    out = dict(card=name, power_limit_w=watts, layers=layers(args.repeat))
    out['term'] = [term(4, 300, 400, max(3, args.repeat // 4), sd, args.check),
                   term(49, 400, 400, 3, sd, False)]
    out['step'] = step(max(3, args.repeat // 2), sd)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
