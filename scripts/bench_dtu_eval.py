"""Times the GPU DTU chamfer evaluation (dbw_b200.dtu_eval) on a DBW-sized synthetic scene in millimetres and prints
one JSON line: CUDA-event times per stage (sample, shuffle, downsample + its round count, mask, d2s, s2d, total), the
card's name and power limit, and with --check the CPU restatement's (oracle/mesh_eval.py) wall time and scores on the
same inputs and shuffle.

The scene: 10 level-1 icospheres with radii of 30-90 mm (about 1e7 lattice samples) and a 2 M-point "STL" cloud of noisy
samples of their surfaces, an observation mask over the scene's box at 2 mm and a ground plane under it.

    python scripts/bench_dtu_eval.py [--check] [--repeat 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = ['sample', 'shuffle', 'downsample', 'mask', 'd2s', 's2d']


def scene(seed=0, n_spheres=10, n_stl=2_000_000):
    from dbw_b200 import geometry
    iv, iff = (t.numpy() for t in geometry.ico_sphere(1))
    iv = iv.astype(np.float64)
    g = np.random.default_rng(seed)
    verts, faces, centers, radii = [], [], [], []
    for k in range(n_spheres):
        c, r = g.uniform([-150, -150, 400], [150, 150, 700]), g.uniform(30, 90)
        Q = np.linalg.qr(g.normal(size=(3, 3)))[0]
        faces.append(iff + len(verts) * len(iv))
        verts.append(iv @ Q * r + c)
        centers.append(c), radii.append(r)
    V = np.concatenate(verts).astype(np.float32)
    F = np.concatenate(faces).astype(np.int64)
    k = g.integers(0, n_spheres, n_stl)
    d = g.normal(size=(n_stl, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    stl = (np.asarray(centers)[k] + d * (np.asarray(radii)[k, None] * 0.97 + g.normal(0, 0.3, (n_stl, 1))))
    stl = stl.astype(np.float32).astype(np.float64)
    lo, hi = V.min(0) - 10, V.max(0) + 10
    BB = np.stack([lo, hi]).astype(np.float64)
    res = 2.0
    obs = g.uniform(size=tuple(int(x) for x in np.ceil((hi - lo) / res) + 1)) < 0.9
    plane = np.array([[0.02], [-0.01], [-1.0], [float(hi[2]) - 20]])           # the top 20 mm are "below" the plane
    return V, F, stl, obs, BB, np.array([[res]]), plane


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true', help='also run the CPU restatement on the same inputs')
    ap.add_argument('--repeat', type=int, default=3, help='timed runs after one warm-up run (the best is reported)')
    ap.add_argument('--spheres', type=int, default=10)
    ap.add_argument('--stl', type=int, default=2_000_000)
    args = ap.parse_args()
    from dbw_b200.dtu_eval import evaluate_arrays
    from oracle import mesh_eval as M

    V, F, stl, obs, BB, Res, P = scene(n_spheres=args.spheres, n_stl=args.stl)
    dev = torch.device('cuda:0')
    n_pcd = None
    best = None
    for it in range(args.repeat + 1):
        events = []

        def timer(stage):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            events.append((stage, e))
        torch.cuda.synchronize()
        start = torch.cuda.Event(enable_timing=True)
        start.record()
        if n_pcd is None:
            r = evaluate_arrays(V, F, stl, obs, BB, Res, P, seed=0, device=dev, timer=timer)
            n_pcd = r['data_pcd'].shape[0]
            order = np.random.default_rng(1).permutation(n_pcd)
            continue                                             # warm-up (and the cloud size for the fixed order)
        r = evaluate_arrays(V, F, stl, obs, BB, Res, P, order=order, device=dev, timer=timer)
        torch.cuda.synchronize()
        t, prev = {}, start
        for stage, e in events:
            t[stage] = prev.elapsed_time(e)
            prev = e
        t['total'] = start.elapsed_time(events[-1][1])
        if best is None or t['total'] < best[0]['total']:
            best = (t, r)
    t, r = best
    name, plimit = card()
    out = {'metric': 'dtu_eval_ms', 'card': name, 'power_limit_w': plimit,
           'points': {'data_pcd': int(n_pcd), 'data_down': int(r['data_down'].shape[0]), 'data_in_obs': int(r['data_in_obs'].shape[0]),
                      'stl': int(len(stl)), 'stl_above': int(r['stl_above'].shape[0])},
           'ms': {k: round(v, 3) for k, v in t.items()}, 'downsample_rounds': r['rounds'],
           'scores': {'acc': float(r['acc']), 'comp': float(r['comp']), 'avg': float(r['avg'])}}
    if args.check:
        t0 = time.perf_counter()
        o = M.evaluate(V, F, order, obs, BB, Res, P, stl)
        out['cpu_oracle_s'] = round(time.perf_counter() - t0, 2)
        out['cpu_scores'] = {'acc': float(o['acc']), 'comp': float(o['comp']), 'avg': float(o['avg'])}
        rel = max(abs(float(r[k]) - float(o[k])) / abs(float(o[k])) for k in ('acc', 'comp', 'avg'))
        out['max_rel_diff'] = rel
        out['check'] = bool(rel <= 1e-9 and r['data_in'].shape[0] == len(o['data_in']))
    print(json.dumps(out))
    if args.check and not out['check']:
        sys.exit(1)


if __name__ == '__main__':
    main()
