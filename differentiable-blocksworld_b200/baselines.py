"""The paper's comparison with the EMS (superquadrics) and MBF (MonteBoxFinder, boxes) baselines on DTU: the reference's
src/dtu_3d_process.py, src/ems_eval.py, src/mbf_eval.py and src/utils/ransac.py, on the GPU.

  ransac_ground_mask / ransac_filter   Ransac(n_points=3, n_iter=100, batch_size=10, thresh=0.001) with LSLinearRegressor,
                                       in the sm_90a kernels of csrc/dbw_ransac.cu
  DTU3DPreprocess                      the ground-truth clouds the baselines are fitted to: {tag}_scale.npy and {tag}.ply
  EMSEvaluator / MBFEvaluator          chamfer-L1 ({tag}_scores.tsv) and the official DTU scores (dtu_scores_{tag}.tsv) of
                                       the fitted superquadrics / boxes

The RANSAC draws are the reference's: one torch.randint(0, N, (batch_size n_points,)) per round on the CPU generator, so a
run seeded as the reference's `run(seed=...)` picks the same samples.  Each hypothesis is solved in float64 and stored as
float32; the reference inverts in float32, so the two agree to float32 rounding times the conditioning of the sample, and
counts can differ on points within that rounding of the threshold.  A sample whose X^T X is singular (a repeated index,
collinear points) gives a rounding-noise plane in both, with few inliers.  The choice keeps the reference's rule.

Datasets are passed in: a mapping tag -> an object with `pc_gt` (N, 3) and `scale_mat` (4, 4), as the reference's
DTUDataset has (take that class, or any stand-in).  The mesh point samples are drawn on the CPU, where the reference draws
them, so that a seeded run samples the reference's points; the nearest-neighbour searches behind both scores run on the GPU.
"""
import ctypes
import json
import random
import shutil
from collections import OrderedDict
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import torch

from . import _lib
from ._lib import DbwError, DbwRansacResult, check
from . import geometry as G
from .dtu_eval import evaluate_mesh, write_ply
from .pointcloud import knn_points, sample_points_from_meshes
from .structures import Meshes, join_meshes_as_scene

N_POINTS_EMS_FIT = 5000
N_POINTS_MBF_FIT = 200000
N_POINTS_EVAL = int(5e5)
CHAMFER_FACTOR = 10


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


@contextmanager
def _seeded(seed):
    """the reference's use_seed: seed random, numpy and torch when `seed` is given, and restore their states after"""
    if seed is None:
        yield
        return
    states = random.getstate(), np.random.get_state(), torch.get_rng_state()
    random.seed(seed), np.random.seed(seed), torch.manual_seed(seed)
    try:
        yield
    finally:
        random.setstate(states[0]), np.random.set_state(states[1]), torch.set_rng_state(states[2])


# ------------------------------------------------------------------------------------------------ RANSAC
def _cloud(pc):
    if not torch.is_tensor(pc) or not pc.is_cuda:
        raise DbwError('ransac: expected a CUDA tensor (there is no CPU fallback)')
    if pc.dim() != 2 or pc.shape[1] != 3 or pc.dtype != torch.float32:
        raise DbwError(f'ransac: expected float32 (N, 3) points, got {pc.dtype} {tuple(pc.shape)}')
    if not 1 <= pc.shape[0] <= 2 ** 31 - 1:
        raise DbwError('ransac: the cloud must have between 1 and 2^31 - 1 points')
    return pc.contiguous()


def _ransac(pc, n_points, n_iter, batch_size, thresh):
    """fit, count and select on the device; returns (params, counts, result, workspace, chosen (a, b, c), n_inliers)"""
    N, dev = pc.shape[0], pc.device
    n_batch = n_iter // batch_size
    H = n_batch * batch_size
    if H < 1 or H > _lib.RANSAC_MAX_HYPOTHESES or not 3 <= n_points <= _lib.RANSAC_MAX_SAMPLE:
        raise DbwError(f'ransac: {H} hypotheses of {n_points} points (1..{_lib.RANSAC_MAX_HYPOTHESES}, 3..{_lib.RANSAC_MAX_SAMPLE})')
    # Ransac.fit's draws, round by round on the CPU generator, sent to the device once
    idx = torch.cat([torch.randint(0, N, (batch_size * n_points,)) for _ in range(n_batch)]).to(dev)
    L, st = _lib.lib(), _stream(dev)
    nbytes = ctypes.c_size_t(0)
    check(L.dbw_ransac_workspace_bytes(N, H, ctypes.byref(nbytes)), 'dbw_ransac_workspace_bytes')
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    params = torch.empty(H, 3, dtype=torch.float32, device=dev)
    counts = torch.empty(H, dtype=torch.int64, device=dev)
    result = torch.empty(ctypes.sizeof(DbwRansacResult), dtype=torch.uint8, device=dev)
    check(L.dbw_ransac_fit(N, _vp(pc), H, n_points, _vp(idx), _vp(params), st), 'dbw_ransac_fit')
    check(L.dbw_ransac_count(N, _vp(pc), H, _vp(params), float(thresh), _vp(counts), _vp(ws), nbytes.value, st), 'dbw_ransac_count')
    check(L.dbw_ransac_select(H, batch_size, _vp(counts), _vp(params), _vp(result), st), 'dbw_ransac_select')
    r = DbwRansacResult.from_buffer_copy(result.cpu().numpy().tobytes())          # the one read of the whole fit
    if r.hypothesis < 0:
        raise DbwError('ransac: no hypothesis has an inlier (the reference has no model to filter with)')
    return dict(idx=idx, params=params, counts=counts, result=result, ws=ws, hypothesis=r.hypothesis,
                model=tuple(float(v) for v in r.params), n_inliers=int(r.n_inliers), n_models=r.n_improvements)


def _filter(pc, fit, thresh, kept=None, inlier=None):
    n_kept = torch.empty(1, dtype=torch.int64, device=pc.device)
    ws = fit['ws']
    check(_lib.lib().dbw_ransac_filter(pc.shape[0], _vp(pc), _vp(fit['result']), float(thresh),
                                       _vp(kept) if kept is not None else None, _vp(inlier) if inlier is not None else None,
                                       _vp(n_kept), _vp(ws), ws.numel(), _stream(pc.device)), 'dbw_ransac_filter')
    return n_kept


def ransac_ground_mask(pc, n_points=3, n_iter=100, batch_size=10, thresh=1e-3):
    """(inlier mask (N,) bool, (a, b, c), n_inliers) of the plane z = a + b x + c y that Ransac(...).fit(pc[:, :2], pc[:, 2:3])
    chooses (best_models[-1]) for the CUDA float32 cloud pc (N, 3); the mask is that model's predicate on every point.
    Draws from torch's CPU generator as the reference does.  Raises when no hypothesis has an inlier."""
    pc = _cloud(pc)
    fit = _ransac(pc, n_points, n_iter, batch_size, thresh)
    inlier = torch.empty(pc.shape[0], dtype=torch.uint8, device=pc.device)
    _filter(pc, fit, thresh, inlier=inlier)
    return inlier.bool(), fit['model'], fit['n_inliers']


def ransac_filter(pc, n_points=3, n_iter=100, batch_size=10, thresh=1e-3):
    """(pc[~inlier] in input order, (a, b, c), n_inliers): dtu_3d_process.py's ground filter, the kept points compacted
    on the device"""
    pc = _cloud(pc)
    fit = _ransac(pc, n_points, n_iter, batch_size, thresh)
    kept = torch.empty_like(pc)
    _filter(pc, fit, thresh, kept=kept)
    return kept[:pc.shape[0] - fit['n_inliers']], fit['model'], fit['n_inliers']


# ------------------------------------------------------------------------------------------------ preprocessing
class DTU3DPreprocess:
    """src/dtu_3d_process.py: per scan, the ground-truth cloud shuffled (torch.randperm), optionally without its RANSAC
    ground plane, mapped back to the original space by scale_mat and standardised as the baseline expects: centred, then
    scaled by 10 / max for EMS (5 000 points kept) or 5 / max for MBF (200 000).  Writes {tag}_scale.npy (mean x y z,
    scale) and {tag}.ply, the first points of the cloud.  The PLY holds double x y z (dtu_eval.write_ply); its bytes are not
    pinned to PyTorch3D's save_ply, which the reference calls and which is not available here: read back, it gives the
    same points."""

    def __init__(self, run_dir, model_name, filter_ground=False, device=None):
        if model_name not in ('ems', 'mbf'):
            raise NotImplementedError(model_name)
        self.run_dir = Path(run_dir)
        self.run_dir.mkdir(parents=True, exist_ok=True)
        self.model_name, self.filter_ground = model_name, filter_ground
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())

    def run(self, datasets, seed=None):
        """`datasets`: tag -> an object with pc_gt and scale_mat.  Returns tag -> (the standardised cloud, mean, scale)."""
        out = {}
        with _seeded(seed):
            for tag, ds in datasets.items():
                pc = ds.pc_gt[torch.randperm(len(ds.pc_gt))].to(self.device)
                scale_mat = ds.scale_mat.to(self.device)
                if self.filter_ground:
                    pc = ransac_filter(pc)[0]
                pc = pc @ scale_mat[:3, :3] + scale_mat[:3, 3]
                n_points, extent = (N_POINTS_EMS_FIT, 10) if self.model_name == 'ems' else (N_POINTS_MBF_FIT, 5)
                mean = pc.mean(0)
                pc = pc - mean
                scale = extent / pc.max()
                pc = pc * scale
                np.save(self.run_dir / f'{tag}_scale.npy', torch.cat([mean, scale.expand(1)]).cpu().numpy())
                write_ply(self.run_dir / f'{tag}.ply', pc[:n_points].cpu().numpy())
                out[tag] = (pc, mean, scale)
        return out


# ------------------------------------------------------------------------------------------------ evaluation
def create_sq_meshes(eps1, eps2, scale):
    """src/utils/superquadric.py:create_sq_meshes: the level-1 icosphere (the reference ignores its `level` argument) mapped
    to each superquadric, eps1 / eps2 (N, 1), scale (N, 3)"""
    verts, faces = G.ico_sphere(1)
    verts, faces = verts.to(eps1.device), faces.to(eps1.device)
    N = len(eps1)
    eta, omega = torch.asin(verts[..., 1]), torch.atan2(verts[..., 0], verts[..., 2])
    eta, omega = eta[None].expand(N, -1), omega[None].expand(N, -1)
    return Meshes(G.superquadric_points(eta, omega, eps1, eps2) * scale[:, None], faces[None].expand(N, -1, -1))


def box_hull_faces(corners):
    """(12, 3) int64 outward-facing triangles of the convex hull of a box's eight corners (8, 3).  The face order is Qhull's,
    not trimesh's, so the points sample_points_from_meshes draws on the hull differ from the reference's."""
    from scipy.spatial import ConvexHull
    c = np.asarray(corners, np.float64)
    tri = ConvexHull(c, qhull_options='QbB Pp Qt').simplices.astype(np.int64)
    if len(tri) != 12:
        raise DbwError(f'box_hull_faces: the hull of the eight corners has {len(tri)} triangles, not a box\'s 12')
    a, b, d = c[tri[:, 0]], c[tri[:, 1]], c[tri[:, 2]]
    outward = (np.cross(b - a, d - a) * ((a + b + d) / 3 - c.mean(0))).sum(1) > 0
    tri[~outward] = tri[~outward][:, [0, 2, 1]]
    return tri


def chamfer_l1(x, y):
    """the reference's chamfer_distance(x, y, return_L1=True, direction_reduction='none')[0] for one pair of clouds
    x (1, P1, 3), y (1, P2, 3): the mean nearest-neighbour distance each way"""
    lx = torch.full((1,), x.shape[1], dtype=torch.int64, device=x.device)
    ly = torch.full((1,), y.shape[1], dtype=torch.int64, device=y.device)
    cx = knn_points(x, y, K=1).dists[..., 0].sqrt().sum(1) / lx
    cy = knn_points(y, x, K=1).dists[..., 0].sqrt().sum(1) / ly
    return cx.sum() / 1, cy.sum() / 1


class _Evaluator:
    name = ''

    def __init__(self, run_dir, baseline_dir=None, device=None):
        self.run_dir = Path(run_dir)
        self.run_dir.mkdir(parents=True, exist_ok=True)
        if baseline_dir is not None:
            if not Path(baseline_dir).exists():
                raise FileNotFoundError(f'{Path(baseline_dir).absolute()} does not exist')
            shutil.copytree(str(baseline_dir), str(self.run_dir), dirs_exist_ok=True)
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())

    def scene(self, tag):
        raise NotImplementedError

    def run(self, datasets, dtu_dir, seed=None, dtu_seed=None):
        """`datasets`: tag -> an object with pc_gt and scale_mat (tags scan<id>); `dtu_dir` holds ObsMask/ and Points/stl/.
        `dtu_seed` seeds the shuffle of the DTU evaluation (unseeded by default, as in the reference).  Returns
        tag -> scores (n_blocks, chL1_acc, chL1_comp, and the DTU acc, comp, avg)."""
        out = {}
        with _seeded(seed):
            for tag, ds in datasets.items():
                gt = ds.pc_gt[torch.randperm(len(ds.pc_gt))][:N_POINTS_EVAL]
                mean, scale = torch.from_numpy(np.load(self.run_dir / f'{tag}_scale.npy')).split([3, 1])
                scene, n = self.scene(tag, mean, scale)
                points = sample_points_from_meshes(scene, num_samples=N_POINTS_EVAL).to(self.device)
                scale_inv = ds.scale_mat.inverse().to(self.device)
                points = points @ scale_inv[:3, :3] + scale_inv[:3, 3]
                acc, comp = chamfer_l1(points, gt[None].to(self.device))
                scores = OrderedDict([('n_blocks', n), ('chL1_acc', CHAMFER_FACTOR * acc.item()),
                                      ('chL1_comp', CHAMFER_FACTOR * comp.item())])
                with open(self.run_dir / f'{tag}_scores.tsv', mode='w') as f:
                    f.write('\t'.join(scores.keys()) + '\n')
                    f.write('\t'.join(map('{:.5f}'.format, scores.values())) + '\n')
                dtu = evaluate_mesh(scene, int(tag.replace('scan', '')), dtu_dir, self.run_dir, suffix=f'_{tag}',
                                    save_viz=False, seed=dtu_seed, device=self.device)
                scores.update(dtu)
                out[tag] = dict(scores)
        return out


class EMSEvaluator(_Evaluator):
    """src/ems_eval.py: the superquadrics of {tag}_spq.npy (N, 11: eps1, eps2, S (3), ZYX Euler angles (3), T (3)) in the
    EMS-standardised space, meshed by create_sq_meshes, rotated, translated and mapped back by {tag}_scale.npy"""

    def scene(self, tag, mean, scale):
        from scipy.spatial.transform import Rotation
        params = torch.from_numpy(np.load(self.run_dir / f'{tag}_spq.npy')).float()
        eps1, eps2, S, T = params[:, 0:1], params[:, 1:2], params[:, 2:5], params[:, 8:11]
        R = torch.from_numpy(Rotation.from_euler('ZYX', params[:, 5:8]).as_matrix()).float()
        meshes = create_sq_meshes(eps1, eps2, S)
        verts = (R @ meshes.verts_padded().permute(0, 2, 1) + T[:, :, None]).permute(0, 2, 1)
        verts = verts / scale + mean
        return join_meshes_as_scene(Meshes(verts, meshes.faces_padded())), len(params)


class MBFEvaluator(_Evaluator):
    """src/mbf_eval.py: the boxes of {tag}/UH.json's `bbox` (N, 8, 3) in the MBF-standardised space, mapped back by
    {tag}_scale.npy, each meshed as the convex hull of its corners (box_hull_faces)"""

    def scene(self, tag, mean, scale):
        with open(self.run_dir / tag / 'UH.json', mode='r') as f:
            metrics = json.load(f)
        verts = torch.Tensor(metrics['bbox']).float()
        verts = verts / scale + mean
        faces = torch.stack([torch.from_numpy(box_hull_faces(v.numpy())) for v in verts])
        return join_meshes_as_scene(Meshes(verts, faces)), len(verts)
