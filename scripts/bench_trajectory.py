"""What a trajectory video costs on the GPU: 240 supersampled frames of the scene model (10 blocks, the bench.py scene) along
get_circle_traj about one view, two ways, alternating in one process:

  pool    today's viz_purpose path: the hard render at 4H x 4W, F.avg_pool2d(., 4), then the uint8 conversion, in chunks of
          10 frames (the reference's B = 10)
  resolve Renderer.render_viz: the resolving kernel writes the uint8 frames directly, chunks sized by views.CHUNK_BYTES

Two shapes: 400x400 (DTU) and 576x768 (BlendedMVS).  Per shape and arm: frames/s (CUDA-synchronised wall clock, median of
--repeat) and the peak device memory above the (N,H,W,3) uint8 video both arms fill; the host time of encoding the 240
frames with OpenCV (mp4v) is reported separately.  --check asserts that both arms give the same float frames and the same uint8 frames, bit for bit.  Prints one JSON line with
the card's name and power limit.

    python scripts/bench_trajectory.py [--repeat 5] [--check]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from copy import deepcopy

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'dtu': (400, 400), 'bmvs': (576, 768)}
N_FRAMES = 240
CFG = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
       'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
       'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                      'decouple_rendering': True, 'opacity_noise': False},
       'loss': {'rgb_weight': 1}}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def to_u8(rgb):
    return (rgb * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8)


@torch.no_grad()
def pool_arm(renderer, mesh, R, T, frames, keep=None):
    """frames (N,H,W,3) uint8 receives the video; keep: a list that collects the float frames (--check)"""
    for k in range(0, len(R), 10):
        out = renderer(mesh, R[k:k + 10], T[k:k + 10], viz_purpose=True)
        frames[k:k + 10] = to_u8(out[:, :3])
        if keep is not None:
            keep.append(out)


@torch.no_grad()
def resolve_arm(renderer, mesh, R, T, frames, keep=None):
    from dbw_b200 import views as V
    for a, b in V._chunks(renderer, mesh, len(R), None):
        out = renderer.render_viz(mesh, R[a:b], T[a:b], frames_u8=True)
        frames[a:b] = out[1]
        if keep is not None:
            keep.append(out[0])


def timed(fn, *args):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def measure(shape, repeat, check):
    from dbw_b200 import views as V
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.synthetic import ring_cameras
    dev = torch.device('cuda')
    H, W = SHAPES[shape]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).eval()
    R0, T0, K = ring_cameras(1)
    model.renderer.update_cameras(device=dev, K=K[None].to(dev))
    mesh = model.build_scene(filter_transparent=True)
    R_traj = V.get_circle_traj(N_views=N_FRAMES)[0].to(dev)
    R, T = R0.to(dev) @ R_traj, T0.to(dev).expand(N_FRAMES, -1)
    arms = {'pool': pool_arm, 'resolve': resolve_arm}
    frames = {a: torch.empty(N_FRAMES, H, W, 3, dtype=torch.uint8, device=dev) for a in arms}
    res = {a: {'s': [], 'peak': 0} for a in arms}
    for a, fn in arms.items():                       # warm-up of every shape either arm launches
        fn(model.renderer, mesh, R, T, frames[a])
    for _ in range(repeat):
        for a, fn in arms.items():
            s, peak = timed(fn, model.renderer, mesh, R, T, frames[a])
            res[a]['s'].append(s)
            res[a]['peak'] = max(res[a]['peak'], peak)
    if check:
        kept = {a: [] for a in arms}
        for a, fn in arms.items():
            fn(model.renderer, mesh, R, T, frames[a], kept[a])
        assert torch.equal(torch.cat(kept['pool']), torch.cat(kept['resolve'])), 'float frames differ'
        assert torch.equal(frames['pool'], frames['resolve']), 'uint8 frames differ'
        del kept
    frames = frames['resolve'].cpu()
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        with V.VideoWriter(os.path.join(tmp, 'traj.mp4')) as vw:
            vw.write(frames)
        encode = time.perf_counter() - t0
    summary = {a: {'frames_per_s': round(N_FRAMES / statistics.median(r['s']), 1), 'median_s': round(statistics.median(r['s']), 4),
                   'peak_device_mib': round(r['peak'] / 2 ** 20, 1)} for a, r in res.items()}
    summary['host_encode_s'] = round(encode, 3)
    summary['speedup'] = round(statistics.median(res['pool']['s']) / statistics.median(res['resolve']['s']), 2)
    summary['bit_identical'] = bool(check) or None
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=5)
    ap.add_argument('--check', action='store_true', help='assert that both arms give the same bits')
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_trajectory.py needs a CUDA device')
    name, power = card()
    out = {'gpu': name, 'power_limit_w': power, 'frames': N_FRAMES}
    for shape in args.shapes.split(','):
        out[f'{shape}_{SHAPES[shape][0]}x{SHAPES[shape][1]}'] = measure(shape, args.repeat, args.check)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
