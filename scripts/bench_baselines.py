"""What the CUDA RANSAC ground filter (dbw_b200.baselines) buys over the reference's, and what one scan of the baseline
tooling costs, on one GPU:
  ransac       the reference's Ransac.fit + filter (src/utils/ransac.py, dtu_3d_process.py:36-41) as torch ops on the
               device (restated below: each round builds (10, N) intermediates and reads its best count back) against
               dbw_ransac_fit / count / select / filter, on a 2.5e6-point cloud, 100 hypotheses
  preprocess   one scan's DTU3DPreprocess.run (shuffle, ground filter, scale back, EMS standardisation, the two files), with
               the reference's RANSAC and with the kernels
  ems_eval     one scan's EMSEvaluator.run (50 superquadrics, 5e5 samples against 5e5 ground-truth points, then the DTU
               evaluation); the reference's own evaluation (Open3D / scikit-learn on the CPU) is not restated here
--check confirms that both RANSACs choose the same hypothesis, and reports whether they keep the same cloud bit for bit and,
where they do not, how many points they disagree on and how close those lie to the threshold.  Prints one JSON line with
the card's name and power limit.

    python scripts/bench_baselines.py [--check] [--points 2500000] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from golden.make_baselines_golden import cloud  # noqa: E402


def reference_ransac(pc, n_points=3, n_iter=100, batch_size=10, thresh=0.001):
    """Ransac().fit(pc[:, :2], pc[:, 2:3]) and the filter, as the reference runs them on the device"""
    X, y = pc[:, :2], pc[:, 2:3]
    N, P, B = X.size(0), n_points, batch_size
    best_n, best = 0, None

    def predict(params, Xb):
        return torch.cat([torch.ones_like(Xb)[..., 0:1], Xb], dim=-1) @ params

    for k in range(n_iter // B):
        idxs = torch.randint(0, N, (B * P,))
        Xs = torch.cat([torch.ones_like(X[idxs].view(B, P, -1))[..., 0:1], X[idxs].view(B, P, -1)], dim=-1)
        Xt = Xs.transpose(-2, -1)
        params = (Xt @ Xs).inverse() @ Xt @ y[idxs].view(B, P, -1)
        diff = (y[None].expand(B, -1, -1) - predict(params, X[None].expand(B, -1, -1))).flatten(1)
        n_inliers = (diff.pow(2) < thresh).sum(1)
        best_idx = torch.argmax(n_inliers)
        n = n_inliers[best_idx].item()
        if n > best_n:
            best_n, best = n, (k * B + int(best_idx), params[best_idx].clone())
    is_inlier = (predict(best[1], pc[:, :2]) - pc[:, 2:]).pow(2) < thresh
    return pc[~is_inlier[:, 0]], best[0], best_n, is_inlier[:, 0]


def timed(fn, repeats):
    torch.cuda.synchronize()
    ts, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, ts


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        limit = 'unknown'
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true')
    ap.add_argument('--points', type=int, default=2500000)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_baselines.py needs a GPU')
    from dbw_b200 import _lib
    from dbw_b200.baselines import DTU3DPreprocess, EMSEvaluator, ransac_filter
    from dbw_b200 import baselines as B
    dev = torch.device('cuda:0')
    name, limit = card()
    res = dict(gpu=name, power_limit=limit, points=args.points, hypotheses=100)
    pc_np = cloud(args.points, 7)
    pc = torch.from_numpy(pc_np).to(dev)

    # ------------------------------------------------------------------ RANSAC
    torch.manual_seed(0)
    reference_ransac(pc)                                            # warm-up (cuBLAS / cuSOLVER handles, allocator)
    torch.manual_seed(0)
    ransac_filter(pc)
    torch.manual_seed(0)
    (ref_kept, ref_h, ref_n, _), t_ref = timed(lambda: reference_ransac(pc), args.repeats)
    torch.manual_seed(0)
    (kept, model, n_in), t_new = timed(lambda: ransac_filter(pc), args.repeats)
    res['ransac_reference_ms'] = 1e3 * float(np.median(t_ref))
    res['ransac_cuda_ms'] = 1e3 * float(np.median(t_new))
    # kernel time alone (the draws and their copy excluded), CUDA events over repeated launches
    torch.manual_seed(0)
    fit = B._ransac(pc, 3, 100, 10, 1e-3)
    L, st = _lib.lib(), B._stream(dev)
    counts = torch.empty(100, dtype=torch.int64, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        _lib.check(L.dbw_ransac_count(pc.shape[0], B._vp(pc), 100, B._vp(fit['params']), 1e-3, B._vp(counts), B._vp(fit['ws']),
                                      fit['ws'].numel(), st), 'dbw_ransac_count')
    e1.record()
    torch.cuda.synchronize()
    res['count_kernel_ms'] = e0.elapsed_time(e1) / 20
    res['count_kernel_GBps'] = pc.numel() * 4 / (res['count_kernel_ms'] * 1e-3) / 1e9
    if args.check:
        from dbw_b200.baselines import ransac_ground_mask
        torch.manual_seed(0)
        ref_kept, ref_h, ref_n, ref_in = reference_ransac(pc)
        torch.manual_seed(0)
        fit = B._ransac(pc, 3, 100, 10, 1e-3)
        torch.manual_seed(0)
        kept, model, n_in = ransac_filter(pc)
        torch.manual_seed(0)
        mine_in = ransac_ground_mask(pc)[0]
        res['check_same_hypothesis'] = ref_h == fit['hypothesis']
        res['check_same_cloud'] = ref_kept.cpu().numpy().tobytes() == kept.cpu().numpy().tobytes()
        res['inliers_reference'], res['inliers_cuda'] = ref_n, n_in
        # the reference inverts in float32, so a point whose squared residual lies within rounding of the threshold may
        # fall on either side: the points the two filters disagree on, and how far from the threshold they lie (float64)
        a, b, c = model
        p64 = pc.double()
        r2 = (p64[:, 2] - ((a + b * p64[:, 0]) + c * p64[:, 1])) ** 2
        differ = ref_in != mine_in
        res['check_points_disagreeing'] = int(differ.sum())
        res['check_max_abs_r2_minus_thresh_where_disagreeing'] = float((r2[differ] - 1e-3).abs().max()) if differ.any() else 0.0

    # ------------------------------------------------------------------ one scan's preprocess
    scale_mat = torch.tensor([[212.5, 0, 0, -11.25], [0, 212.5, 0, 37.5], [0, 0, 212.5, 640.0], [0, 0, 0, 1]])
    ds = types.SimpleNamespace(pc_gt=torch.from_numpy(pc_np), scale_mat=scale_mat)
    with tempfile.TemporaryDirectory() as tmp:
        pre = DTU3DPreprocess(tmp, 'ems', filter_ground=True, device=dev)
        pre.run({'scan24': ds}, seed=1234)
        _, t_pre = timed(lambda: pre.run({'scan24': ds}, seed=1234), 3)
        saved = B.ransac_filter
        B.ransac_filter = lambda p: reference_ransac(p)[:3]
        try:
            _, t_pre_ref = timed(lambda: pre.run({'scan24': ds}, seed=1234), 3)
        finally:
            B.ransac_filter = saved
        res['preprocess_reference_ransac_ms'] = 1e3 * float(np.median(t_pre_ref))
        res['preprocess_cuda_ms'] = 1e3 * float(np.median(t_pre))

        # -------------------------------------------------------------- one scan's EMS evaluation
        from tests.test_dtu_eval_gpu import _dtu_dir
        g = np.random.default_rng(3)
        n = 50
        spq = np.c_[g.uniform(0.2, 1.5, (n, 2)), g.uniform(0.3, 1.0, (n, 3)), g.uniform(-np.pi, np.pi, (n, 3)),
                    g.uniform(-6, 6, (n, 3))]
        ems = os.path.join(tmp, 'ems')
        os.makedirs(ems)
        np.save(os.path.join(ems, 'scan24_spq.npy'), spq)
        np.save(os.path.join(ems, 'scan24_scale.npy'), np.array([-11.25, 37.5, 640.0, 10 / 212.5], np.float32))
        stl = (pc_np[:2000000].astype(np.float64) * 212.5 + [-11.25, 37.5, 640.0])
        lo, hi = stl.min(0) - 5, stl.max(0) + 5
        obs = np.ones(tuple(int(x) for x in np.ceil((hi - lo) / 2.0) + 1), bool)
        _dtu_dir(os.path.join(tmp, 'DTU'), 24, stl, obs, np.stack([lo, hi]), np.array([[2.0]]),
                 np.array([[0.], [0.], [1.], [-(lo[2] + 3)]]))
        ev = EMSEvaluator(os.path.join(tmp, 'run'), ems, device=dev)
        ev.run({'scan24': ds}, os.path.join(tmp, 'DTU'), seed=1, dtu_seed=1)
        scores, t_ems = timed(lambda: ev.run({'scan24': ds}, os.path.join(tmp, 'DTU'), seed=1, dtu_seed=1), 2)
        res['ems_eval_ms'] = 1e3 * float(np.median(t_ems))
        res['ems_scores'] = scores['scan24']
    print(json.dumps(res))


if __name__ == '__main__':
    main()
