"""Times the k-NN kernels (csrc/dbw_knn.cu) on the two workloads of the reference's 3-D evaluation and prints one JSON
line of CUDA-event times, the card's name and power limit, and the registers / local memory of every k-NN kernel as
compiled into the library (cuobjdump -res-usage):

  ems_mbf   ems_eval.py / mbf_eval.py per scan: sample_points_from_meshes of 5e5 points on 10 level-1 superquadric
            blocks, then the chamfer-L1 legs, both 5e5 x 5e5 directions (acc: samples -> GT, comp: GT -> samples)
  icp       100 gradient_icp-shaped iterations at 1e5 x 1e5: both directions forward (K = 1) and their backward

--check adds scipy cKDTree on the host for the two 5e5 directions: its wall time and whether its nearest indices equal
the kernel's wherever the nearest distance is not tied (within fp32 rounding of the second nearest).

    python scripts/bench_chamfer.py [--check] [--repeat 3]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def blocks(seed=0, n_blocks=10):
    """10 superquadric blocks on the level-1 icosphere's angles, scaled, rotated and placed; (1, V, 3), (1, F, 3)"""
    from dbw_b200 import geometry as G
    iv, iff = G.ico_sphere(1)
    eta, omega = torch.asin(iv[:, 1].clamp(-1, 1)), torch.atan2(iv[:, 0], iv[:, 2])
    g = np.random.default_rng(seed)
    verts, faces = [], []
    for k in range(n_blocks):
        e1, e2 = (float(x) for x in g.uniform(0.2, 1.5, 2))
        p = G.superquadric_points(eta, omega, e1, e2) * torch.tensor(g.uniform(0.1, 0.4, 3), dtype=torch.float32)
        Q = torch.tensor(np.linalg.qr(g.normal(size=(3, 3)))[0], dtype=torch.float32)
        faces.append(iff + k * len(iv))
        verts.append(p @ Q + torch.tensor(g.uniform(-1, 1, 3), dtype=torch.float32))
    return torch.cat(verts)[None].float(), torch.cat(faces)[None]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def kernel_resources():
    """{kernel: {registers, local_bytes}} of the k-NN kernels in the built library, or None without cuobjdump"""
    from dbw_b200 import _lib
    exe = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    try:
        txt = subprocess.run([exe, '-res-usage', _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    except Exception:
        return None
    out, fn = {}, None
    for line in txt.splitlines():
        m = re.search(r'Function (\S+):', line)
        if m:
            fn = m.group(1)
        m = re.search(r'REG:(\d+).*?LOCAL:(\d+)', line)
        if m and fn and 'knn' in fn:
            name = re.sub(r'^_Z\d+', '', fn)
            out[name] = {'registers': int(m.group(1)), 'local_bytes': int(m.group(2))}
    return out


def timed(fn, repeat):
    """best of `repeat` CUDA-event timings (ms) of fn() after one warm-up call, and fn's last result"""
    res = fn()
    best = None
    for _ in range(repeat):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = fn()
        b.record()
        torch.cuda.synchronize()
        best = a.elapsed_time(b) if best is None else min(best, a.elapsed_time(b))
    return best, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true', help='also run scipy cKDTree on the host for the 5e5 directions')
    ap.add_argument('--repeat', type=int, default=3, help='timed runs after one warm-up run (the best is reported)')
    ap.add_argument('--points', type=int, default=500_000)
    ap.add_argument('--icp-points', type=int, default=100_000)
    ap.add_argument('--icp-iters', type=int, default=100)
    args = ap.parse_args()
    from dbw_b200.pointcloud import knn_points, sample_points_from_meshes
    from dbw_b200.structures import Meshes

    dev = torch.device('cuda:0')
    V, F = blocks()
    mesh = Meshes(V.to(dev), F.to(dev))
    S = args.points
    torch.manual_seed(0)
    gt = (sample_points_from_meshes(mesh, S) + 0.003 * torch.randn(1, S, 3, device=dev)).contiguous()

    def sample():
        torch.manual_seed(1)
        return sample_points_from_meshes(mesh, S)
    t_sample, pts = timed(sample, args.repeat)
    t_acc, acc_nn = timed(lambda: knn_points(pts, gt), args.repeat)
    t_comp, comp_nn = timed(lambda: knn_points(gt, pts), args.repeat)
    acc, comp = acc_nn.dists[0, :, 0].sqrt().mean().item(), comp_nn.dists[0, :, 0].sqrt().mean().item()

    n = args.icp_points
    g = torch.Generator(device=dev).manual_seed(2)
    pc_gt = torch.randn(1, n, 3, device=dev, generator=g) * torch.tensor([1.5, 1.0, 0.6], device=dev)
    pc_pred = (pc_gt.flip(1) * 1.05 + 0.02).detach().requires_grad_(True)

    def icp():
        for _ in range(args.icp_iters):
            pc_pred.grad = None
            loss = knn_points(pc_pred, pc_gt).dists.mean() + knn_points(pc_gt, pc_pred).dists.mean()
            loss.backward()
        return loss
    t_icp, _ = timed(icp, 1)

    name, plimit = card()
    pairs = float(S) * S
    out = {'metric': 'chamfer_knn_ms', 'card': name, 'power_limit_w': plimit,
           'ms': {'ems_mbf_sample': round(t_sample, 3), 'ems_mbf_acc': round(t_acc, 3), 'ems_mbf_comp': round(t_comp, 3),
                  'ems_mbf_total': round(t_sample + t_acc + t_comp, 3),
                  f'icp_{args.icp_iters}_iters': round(t_icp, 3)},
           'pairs_per_s': {'ems_mbf_directions': 2 * pairs / ((t_acc + t_comp) * 1e-3)},
           'points': {'ems_mbf': S, 'icp': n}, 'acc': acc, 'comp': comp, 'kernels': kernel_resources()}
    if args.check:
        from scipy.spatial import cKDTree
        p, q = pts[0].cpu().numpy().astype(np.float64), gt[0].cpu().numpy().astype(np.float64)
        t0 = time.perf_counter()
        da, ia = cKDTree(q).query(p, k=2, workers=-1)
        dc, ic = cKDTree(p).query(q, k=2, workers=-1)
        out['ckdtree_s'] = round(time.perf_counter() - t0, 2)
        match = []
        for (d, i), nn in (((da, ia), acc_nn), ((dc, ic), comp_nn)):
            untied = d[:, 1] ** 2 - d[:, 0] ** 2 > 1e-6 * d[:, 1] ** 2
            got = nn.idx[0, :, 0].cpu().numpy()
            match.append(bool(np.array_equal(got[untied], i[untied, 0])))
            out.setdefault('untied_fraction', []).append(float(untied.mean()))
        out['indices_match_ckdtree'] = match
        out['check'] = all(match)
    print(json.dumps(out))
    if args.check and not out['check']:
        sys.exit(1)


if __name__ == '__main__':
    main()
