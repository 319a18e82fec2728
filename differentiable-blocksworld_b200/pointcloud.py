"""Point-cloud ops of PyTorch3D 0.7.1 that the reference's 3-D evaluation calls: `knn_points`, `knn_gather`, the chamfer
helpers `_validate_chamfer_reduction_inputs` / `_handle_pointcloud_input`, PyTorch3D's own `chamfer_distance` and
`sample_points_from_meshes`.  `compat.install()` registers them under their pytorch3d names, so that the reference's
`utils/chamfer.py` (ChamferLoss), `utils/icp.py:gradient_icp` and the chamfer legs of `ems_eval.py` / `mbf_eval.py` run
on the GPU.

PyTorch3D is not installed here; the semantics below are its published behaviour as recalled (arguments, masking,
padding, the order of the random draws), not its code.  The search is the sm_90a kernel pair of csrc/dbw_knn.cu (exact
brute force, fp32, ties to the lower index); there is no CPU fallback: `knn_points` raises on CPU tensors.  The rest is
torch plumbing around it."""
import ctypes
import sys
from collections import namedtuple

import torch
from torch.nn import functional as F

from . import _lib
from ._lib import DbwError, check

_KNN = namedtuple('KNN', 'dists idx knn')
MAX_K = 32                     # DBW_KNN_MAX_K


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _lengths(lengths, N, P, dev):
    if lengths is None:
        return torch.full((N,), P, dtype=torch.int64, device=dev)
    return lengths.to(device=dev, dtype=torch.int64).contiguous()


class _KnnPoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p1, p2, lengths1, lengths2, K):
        N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
        dists = torch.empty(N, P1, K, dtype=torch.float32, device=p1.device)
        idx = torch.empty(N, P1, K, dtype=torch.int64, device=p1.device)
        check(_lib.lib().dbw_knn_forward(_vp(p1), _vp(p2), _vp(lengths1), _vp(lengths2), N, P1, P2, K, _vp(dists), _vp(idx),
                                         _stream(p1.device)), 'dbw_knn_forward')
        ctx.save_for_backward(p1, p2, lengths1, lengths2, idx)
        ctx.mark_non_differentiable(idx)
        return dists, idx

    @staticmethod
    def backward(ctx, grad_dists, grad_idx):
        p1, p2, lengths1, lengths2, idx = ctx.saved_tensors
        N, P1, P2, K = p1.shape[0], p1.shape[1], p2.shape[1], idx.shape[2]
        g = grad_dists.to(torch.float32).contiguous()
        grad_p1, grad_p2 = torch.zeros_like(p1), torch.zeros_like(p2)
        check(_lib.lib().dbw_knn_backward(_vp(p1), _vp(p2), _vp(lengths1), _vp(lengths2), _vp(idx), _vp(g), N, P1, P2, K,
                                          _vp(grad_p1), _vp(grad_p2), _stream(p1.device)), 'dbw_knn_backward')
        return grad_p1, grad_p2, None, None, None


def knn_points(p1, p2, lengths1=None, lengths2=None, norm=2, K=1, version=-1, return_nn=False, return_sorted=True):
    """pytorch3d.ops.knn_points (0.7.1, as recalled): the K nearest points of p2 (N,P2,3) to each point of p1 (N,P1,3)
    in squared L2, as `KNN(dists (N,P1,K), idx (N,P1,K), knn (N,P1,K,3) or None)`, differentiable in p1 and p2.
    `lengths1` / `lengths2` (N,) give the valid points per cloud; padded rows and slots beyond lengths2 are 0 in dists
    and idx, as in PyTorch3D.  The result is always sorted ascending (ties to the lower index), so `return_sorted` and
    `version` change nothing.  Here: CUDA float32 tensors, D = 3, norm = 2 and K <= 32; anything else raises."""
    if p1.shape[0] != p2.shape[0]:
        raise ValueError('pts1 and pts2 must have the same batch dimension.')
    if p1.shape[2] != p2.shape[2]:
        raise ValueError('pts1 and pts2 must have the same point dimension.')
    if norm == 1:
        raise NotImplementedError('knn_points: norm=1 is not implemented (only the squared L2 the reference uses)')
    if norm != 2:
        raise ValueError('Support for 1 or 2 norm.')
    if p1.shape[2] != 3:
        raise NotImplementedError(f'knn_points: D = {p1.shape[2]} is not implemented (D = 3 only)')
    if not (p1.is_cuda and p2.is_cuda):
        raise DbwError('knn_points: expected CUDA tensors (there is no CPU fallback)')
    if p1.dtype != torch.float32 or p2.dtype != torch.float32:
        raise DbwError(f'knn_points: expected float32 points, got {p1.dtype} / {p2.dtype}')
    if not 1 <= int(K) <= MAX_K:
        raise DbwError(f'knn_points: K = {K} is outside [1, {MAX_K}]')
    p1, p2 = p1.contiguous(), p2.contiguous()
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    lengths1 = _lengths(lengths1, N, P1, p1.device)
    lengths2 = _lengths(lengths2, N, P2, p1.device)
    dists, idx = _KnnPoints.apply(p1, p2, lengths1, lengths2, int(K))
    return _KNN(dists=dists, idx=idx, knn=knn_gather(p2, idx, lengths2) if return_nn else None)


def knn_gather(x, idx, lengths=None):
    """pytorch3d.ops.knn_gather: x (N,M,U) gathered at idx (N,L,K) -> (N,L,K,U); slots k >= lengths[n] are zeroed."""
    N, M, U = x.shape
    _N, L, K = idx.shape
    if N != _N:
        raise ValueError('x and idx must have same batch dimension.')
    if lengths is None:
        lengths = torch.full((N,), M, dtype=torch.int64, device=x.device)
    out = x[:, :, None].expand(-1, -1, K, -1).gather(1, idx[..., None].expand(-1, -1, -1, U))
    if lengths.min() < K:
        empty = lengths[:, None] <= torch.arange(K, device=x.device)[None]              # (N, K)
        out[empty[:, None, :, None].expand(-1, L, -1, U)] = 0.0
    return out


# ------------------------------------------------------------------------------------------------ chamfer
def _validate_chamfer_reduction_inputs(batch_reduction, point_reduction):
    """pytorch3d.loss.chamfer._validate_chamfer_reduction_inputs"""
    if batch_reduction is not None and batch_reduction not in ['mean', 'sum']:
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction not in ['mean', 'sum']:
        raise ValueError('point_reduction must be one of ["mean", "sum"]')


def _handle_pointcloud_input(points, lengths, normals):
    """pytorch3d.loss.chamfer._handle_pointcloud_input for tensors: (points, lengths or a full (N,) tensor, normals) after
    PyTorch3D's shape checks.  A `Pointclouds` stays a placeholder here and raises."""
    if not torch.is_tensor(points):
        if type(points).__name__ == 'Pointclouds':
            raise NotImplementedError('chamfer inputs: Pointclouds is not provided by dbw_b200 (pass (N, P, 3) tensors)')
        raise ValueError('The input pointclouds should be either Pointclouds objects or torch.Tensor of shape '
                         '(minibatch, num_points, 3).')
    if points.ndim != 3:
        raise ValueError('Expected points to be of shape (N, P, D)')
    if lengths is not None:
        if lengths.ndim != 1 or lengths.shape[0] != points.shape[0]:
            raise ValueError('Expected lengths to be of shape (N,)')
        if lengths.max() > points.shape[1]:
            raise ValueError('A length value was too long')
    else:
        lengths = torch.full((points.shape[0],), points.shape[1], dtype=torch.int64, device=points.device)
    if normals is not None and normals.ndim != 3:
        raise ValueError('Expected normals to be of shape (N, P, 3')
    return points, lengths, normals


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction='mean', point_reduction='mean', norm=2):
    """pytorch3d.loss.chamfer_distance (0.7.1, as recalled): (squared-L2 chamfer distance, normal cosine term or None)
    between x (N,P1,3) and y (N,P2,3), summed over the two directions, reduced over points ('mean' divides by the
    lengths clamped to 1, or 'sum') and over the batch ('mean' divides by the weight sum or N, 'sum', or None)."""
    _validate_chamfer_reduction_inputs(batch_reduction, point_reduction)
    if norm not in (1, 2):
        raise ValueError('Support for 1 or 2 norm.')
    x, x_lengths, x_normals = _handle_pointcloud_input(x, x_lengths, x_normals)
    y, y_lengths, y_normals = _handle_pointcloud_input(y, y_lengths, y_normals)
    N, P1, D = x.shape
    P2 = y.shape[1]
    if y.shape[0] != N or y.shape[2] != D:
        raise ValueError('y does not have the correct shape.')
    with_normals = x_normals is not None and y_normals is not None
    if weights is not None:
        if weights.size(0) != N:
            raise ValueError('weights must be of shape (N,).')
        if not (weights >= 0).all():
            raise ValueError('weights cannot be negative.')
        if weights.sum() == 0.0:
            z = x.sum((1, 2)) * weights.view(N, 1)
            return (z.sum() * 0.0, z.sum() * 0.0) if batch_reduction in ['mean', 'sum'] else (z * 0.0, z * 0.0)

    terms, norm_terms = [], []
    for a, b, la, lb, na, nb, P in ((x, y, x_lengths, y_lengths, x_normals, y_normals, P1),
                                    (y, x, y_lengths, x_lengths, y_normals, x_normals, P2)):
        nn = knn_points(a, b, lengths1=la, lengths2=lb, norm=norm, K=1)
        pad = torch.arange(P, device=a.device)[None] >= la[:, None]
        hetero = bool((la != P).any())
        d = nn.dists[..., 0]
        if hetero:
            d[pad] = 0.0
        if weights is not None:
            d *= weights.view(N, 1)
        terms.append(d.sum(1))
        if with_normals:
            near = knn_gather(nb, nn.idx, lb)[..., 0, :]
            c = 1 - torch.abs(F.cosine_similarity(na, near, dim=2, eps=1e-6))
            if hetero:
                c[pad] = 0.0
            if weights is not None:
                c *= weights.view(N, 1)
            norm_terms.append(c.sum(1))
    lens = (x_lengths.clamp(min=1), y_lengths.clamp(min=1))

    def reduce(t):
        if point_reduction == 'mean':
            t = [t[0] / lens[0], t[1] / lens[1]]
        if batch_reduction is not None:
            t = [v.sum() for v in t]
            if batch_reduction == 'mean':
                div = weights.sum() if weights is not None else max(N, 1)
                t = [v / div for v in t]
        return t[0] + t[1]
    return reduce(terms), (reduce(norm_terms) if with_normals else None)


# ------------------------------------------------------------------------------------------------ sampling
def _rand_barycentric_coords(n, s, dtype, device):
    """PyTorch3D's draw: one torch.rand(2, n, s), w = (1 - sqrt(u), sqrt(u) (1 - v), sqrt(u) v)"""
    u, v = torch.rand(2, n, s, dtype=dtype, device=device)
    su = u.sqrt()
    return 1.0 - su, su * (1.0 - v), su * v


def sample_points_from_meshes(meshes, num_samples=10000, return_normals=False, return_textures=False):
    """pytorch3d.ops.sample_points_from_meshes (0.7.1, as recalled) on dbw_b200's `Meshes`: `num_samples` points per
    mesh (N, S, 3), uniform over its surface, and with `return_normals` the unit normal (v1 - v0) x (v2 - v1) of each
    sample's face.  The random draws are PyTorch3D's, in its order: face areas -> areas.multinomial(S, replacement=True)
    -> torch.rand(2, N, S) -> barycentric weights; a seeded run draws the same numbers.  A mesh of zero total area has
    no distribution to sample and gives zeros, as an empty mesh does in PyTorch3D; no faces at all raise as there.
    Works on CPU and CUDA tensors alike (torch ops: the cost of the reference's evaluation is in the search)."""
    if return_textures:
        raise NotImplementedError('sample_points_from_meshes: return_textures is not provided by dbw_b200')
    verts, faces = meshes.verts_padded(), meshes.faces_padded()
    if len(meshes) == 0 or faces.shape[1] == 0:
        raise ValueError('Meshes are empty.')
    if not torch.isfinite(verts).all():
        raise ValueError('Meshes contain nan or inf.')
    N, dev = verts.shape[0], verts.device
    fv = verts.gather(1, faces.reshape(N, -1, 1).expand(-1, -1, 3)).reshape(N, -1, 3, 3)     # (N, F, 3, 3)
    v0, v1, v2 = fv[:, :, 0], fv[:, :, 1], fv[:, :, 2]
    samples = torch.zeros(N, num_samples, 3, device=dev)
    normals = torch.zeros(N, num_samples, 3, device=dev)
    with torch.no_grad():
        areas = 0.5 * torch.linalg.cross(v1 - v0, v2 - v0, dim=-1).norm(dim=-1)                # (N, F)
        valid = areas.sum(1) > 0
        face = areas[valid].multinomial(num_samples, replacement=True)                    # (n_valid, S)
    w0, w1, w2 = _rand_barycentric_coords(face.shape[0], num_samples, verts.dtype, dev)

    def pick(t):                                                                          # (n_valid, S, 3)
        return t[valid].gather(1, face[..., None].expand(-1, -1, 3))
    samples[valid] = w0[..., None] * pick(v0) + w1[..., None] * pick(v1) + w2[..., None] * pick(v2)
    if not return_normals:
        return samples
    n = torch.linalg.cross(v1 - v0, v2 - v1, dim=-1)
    normals[valid] = pick(n / n.norm(dim=-1, keepdim=True).clamp(min=sys.float_info.epsilon))
    return samples, normals
