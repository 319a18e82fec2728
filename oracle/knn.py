"""oracle/knn.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the k-nearest-neighbour contract of csrc/dbw_knn.cu (include/dbw_render.h, "k-nearest neighbours")
and of the two reference functions that sit on it, written from their documented semantics:

  knn_f32        numpy float32, the kernel's exact arithmetic: d = (dx*dx + dy*dy) + dz*dz with dx = p1.x - p2.x, each
                 operation rounded to float32 (numpy never contracts), so dists and idx are the kernel's bit for bit
  knn_f64        the same selection on float64 distances (the reference for generic inputs and for cKDTree)
  knn_backward_f64   closed form: d dist / d p1 = 2 (p1 - p2[idx]), the negative into p2, masked as the kernel masks
  knn_points     torch autograd wrapper of knn_f32 / knn_backward_f64 on CPU tensors (the golden generator's k-NN)
  chamfer_distance, gradient_icp   the reference's src/utils/chamfer.py and src/utils/icp.py (non-batched path), restated
                 on top of any knn_points with PyTorch3D's signature

Selection rule (both variants): per query row i < lengths1[n], the K smallest (distance, index) pairs of the targets
j < lengths2[n] whose distance is below +inf.  Padding, as PyTorch3D 0.7.1 is recalled to leave it (its knn_points
zero-initialises both outputs and writes only the neighbours it found): rows i >= lengths1[n] and slots beyond the
neighbours found are distance 0, index 0.  The reference masks both itself, so none of its results depend on this.

Only tests/ and scripts/bench_chamfer.py --check import this module.
"""
import numpy as np
import torch

CHUNK = 1 << 22                # query x target pairs per numpy block


def _lengths(lengths, N, P):
    if lengths is None:
        return np.full(N, P, np.int64)
    return np.clip(np.asarray(lengths, np.int64), 0, P)


def _select(d, K, out_d, out_i):
    """the K smallest (d, index) pairs of each row of d (finite entries only) into out_d / out_i (pre-zeroed)"""
    rows, M = d.shape
    if M == 0:
        return
    d = np.where(d < np.inf, d, np.inf)                      # NaN never selected: treat as +inf
    if K >= M:
        cand = np.broadcast_to(np.arange(M), d.shape)
    else:
        kth = np.partition(d, K - 1, axis=1)[:, K - 1:K]     # every pair of the top K has d <= the K-th value
        cand = None
    for r in range(rows):
        c = np.arange(M) if cand is not None else np.nonzero(d[r] <= kth[r])[0]
        o = c[np.argsort(d[r, c], kind='stable')][:K]        # stable on ascending indices: ties to the lower index
        o = o[d[r, o] < np.inf]
        out_d[r, :len(o)] = d[r, o]
        out_i[r, :len(o)] = o


def _select_k1(d, out_d, out_i):
    if d.shape[1] == 0:
        return
    d = np.where(d < np.inf, d, np.inf)
    j = np.argmin(d, axis=1)                                 # first minimum: ties to the lower index
    v = d[np.arange(len(d)), j]
    ok = v < np.inf
    out_d[ok, 0], out_i[ok, 0] = v[ok], j[ok]


def _knn(p1, p2, lengths1, lengths2, K, dtype):
    p1, p2 = np.asarray(p1, dtype), np.asarray(p2, dtype)
    N, P1, _ = p1.shape
    P2 = p2.shape[1]
    l1, l2 = _lengths(lengths1, N, P1), _lengths(lengths2, N, P2)
    dists, idx = np.zeros((N, P1, K), dtype), np.zeros((N, P1, K), np.int64)
    with np.errstate(over='ignore', invalid='ignore'):
        for n in range(N):
            t = p2[n, :l2[n]]
            step = max(1, CHUNK // max(len(t), 1))
            for a in range(0, l1[n], step):
                q = p1[n, a:min(a + step, l1[n])]
                dx, dy, dz = (q[:, None, c] - t[None, :, c] for c in range(3))
                d = (dx * dx + dy * dy) + dz * dz
                if K == 1:
                    _select_k1(d, dists[n, a:a + len(q)], idx[n, a:a + len(q)])
                else:
                    _select(d, K, dists[n, a:a + len(q)], idx[n, a:a + len(q)])
    return dists, idx


def knn_f32(p1, p2, lengths1=None, lengths2=None, K=1):
    """(dists (N,P1,K) float32, idx (N,P1,K) int64): the kernel's result bit for bit"""
    return _knn(p1, p2, lengths1, lengths2, K, np.float32)


def knn_f64(p1, p2, lengths1=None, lengths2=None, K=1):
    return _knn(p1, p2, lengths1, lengths2, K, np.float64)


def knn_backward_f64(p1, p2, lengths1, lengths2, idx, grad_dists):
    """(grad_p1, grad_p2) float64 of sum(grad_dists * dists) through the selected pairs"""
    p1, p2, g = np.asarray(p1, np.float64), np.asarray(p2, np.float64), np.asarray(grad_dists, np.float64)
    N, P1, K = idx.shape
    P2 = p2.shape[1]
    l1, l2 = _lengths(lengths1, N, P1), _lengths(lengths2, N, P2)
    g1, g2 = np.zeros_like(p1), np.zeros_like(p2)
    for n in range(N):
        i = np.arange(l1[n])
        for k in range(min(K, l2[n])):
            j = idx[n, i, k]
            ok = (j >= 0) & (j < l2[n])
            diff = 2.0 * g[n, i[ok], k, None] * (p1[n, i[ok]] - p2[n, j[ok]])
            g1[n, i[ok]] += diff
            np.add.at(g2[n], j[ok], -diff)
    return g1, g2


class _KnnOracle(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p1, p2, lengths1, lengths2, K):
        d, i = knn_f32(p1.detach().numpy(), p2.detach().numpy(), lengths1.numpy(), lengths2.numpy(), K)
        idx = torch.from_numpy(i)
        ctx.save_for_backward(p1, p2, lengths1, lengths2, idx)
        ctx.mark_non_differentiable(idx)
        return torch.from_numpy(d), idx

    @staticmethod
    def backward(ctx, gd, gi):
        p1, p2, l1, l2, idx = ctx.saved_tensors
        g1, g2 = knn_backward_f64(p1.detach().numpy(), p2.detach().numpy(), l1.numpy(), l2.numpy(), idx.numpy(), gd.numpy())
        return torch.from_numpy(g1).to(p1.dtype), torch.from_numpy(g2).to(p2.dtype), None, None, None


def knn_points(p1, p2, lengths1=None, lengths2=None, norm=2, K=1, version=-1, return_nn=False, return_sorted=True):
    """PyTorch3D's knn_points signature on CPU float32 tensors: KNN(dists, idx, knn=None); squared L2 only"""
    from collections import namedtuple
    assert norm == 2 and not return_nn and p1.shape[2] == 3
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    l1 = torch.full((N,), P1, dtype=torch.int64) if lengths1 is None else lengths1.to(torch.int64)
    l2 = torch.full((N,), P2, dtype=torch.int64) if lengths2 is None else lengths2.to(torch.int64)
    d, i = _KnnOracle.apply(p1.float().contiguous(), p2.float().contiguous(), l1, l2, K)
    return namedtuple('KNN', 'dists idx knn')(d, i, None)


# ------------------------------------------------------------------------------------------------ the reference's chamfer
def _gather1(x, idx):
    """x (N,M,D) at idx (N,L) -> (N,L,D)"""
    return x.gather(1, idx[..., None].expand(-1, -1, x.shape[2]))


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction='mean', point_reduction='mean', direction_reduction='sum', return_L1=False,
                     knn_points=knn_points):
    """The reference's chamfer (src/utils/chamfer.py): PyTorch3D's chamfer_distance with `return_L1` (square roots of the
    nearest squared distances) and `direction_reduction` ('sum', 'mean', or None / 'none' for the pair (x -> y, y -> x)).
    Point means divide by the lengths (not clamped), batch means by the weight sum or N.  Tensor inputs only."""
    if batch_reduction not in (None, 'mean', 'sum'):
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction not in ('mean', 'sum'):
        raise ValueError('point_reduction must be one of ["mean", "sum"]')
    N, P1, D = x.shape
    P2 = y.shape[1]
    lx = torch.full((N,), P1, dtype=torch.int64, device=x.device) if x_lengths is None else x_lengths
    ly = torch.full((y.shape[0],), P2, dtype=torch.int64, device=y.device) if y_lengths is None else y_lengths
    if y.shape[0] != N or y.shape[2] != D:
        raise ValueError('y does not have the correct shape.')
    if weights is not None:
        if weights.size(0) != N:
            raise ValueError('weights must be of shape (N,).')
        if not (weights >= 0).all():
            raise ValueError('weights cannot be negative.')
        if weights.sum() == 0.0:
            z = x.sum((1, 2)) * weights.view(N, 1) * 0.0
            return (z.sum(), z.sum()) if batch_reduction in ('mean', 'sum') else (z, z)
    with_normals = x_normals is not None and y_normals is not None
    dist, cos = [], []
    for a, b, la, lb, na, nb in ((x, y, lx, ly, x_normals, y_normals), (y, x, ly, lx, y_normals, x_normals)):
        nn = knn_points(a, b, lengths1=la, lengths2=lb, K=1)
        keep = (torch.arange(a.shape[1], device=a.device)[None] < la[:, None]).to(a.dtype)
        w = keep if weights is None else keep * weights.view(N, 1)
        d = nn.dists[..., 0]
        d = d.sqrt() if return_L1 else d
        dist.append((d * w).sum(1))
        if with_normals:
            # knn_gather's mask zeroes the slot only when the other cloud is empty: then the cosine is 0
            near = _gather1(nb, nn.idx[..., 0]) * (lb > 0).to(nb.dtype)[:, None, None]
            c = 1 - torch.abs(torch.nn.functional.cosine_similarity(na, near, dim=2, eps=1e-6))
            cos.append((c * w).sum(1))

    def reduce(pair):
        if point_reduction == 'mean':
            pair = [pair[0] / lx, pair[1] / ly]
        if batch_reduction is not None:
            div = (weights.sum() if weights is not None else N) if batch_reduction == 'mean' else 1
            pair = [v.sum() / div for v in pair]
        if direction_reduction is None or direction_reduction == 'none':
            return tuple(pair)
        return (pair[0] + pair[1]) * (0.5 if direction_reduction == 'mean' else 1.0)
    return reduce(dist), (reduce(cos) if with_normals else None)


def gradient_icp(pc_pred, pc_gt, estimate_scale=True, anisotropic_scale=False, lr=0.01, n_iter=300, knn_points=knn_points,
                 losses=None):
    """The reference's gradient_icp (src/utils/icp.py, one parameter set per batch element, no mini-batches): Adam over
    (R_6d, T[, s]) minimising chamfer_distance(s * pc_pred @ R + T, pc_gt) with the default reductions.  Every 10th
    iteration (from 0) the mean loss since the last check is compared with the best so far; when lower, the rotation of
    that moment is kept.  T and s are returned as they are at the end: the reference keeps detached views of the live
    parameters, which the optimiser keeps updating.  Returns (s * pc_pred @ R_best + T, [R_best, T, s]); the loss of each
    iteration is appended to `losses` when given."""
    from dbw_b200.geometry import rotation_6d_to_matrix
    with torch.enable_grad():
        N, dev = len(pc_pred), pc_pred.device
        R_6d = torch.nn.Parameter(torch.tensor([[1., 0., 0., 0., 1., 0.]], device=dev).repeat(N, 1))
        T = torch.nn.Parameter(torch.zeros(N, 3, device=dev))
        s = torch.nn.Parameter(torch.ones(N, 3 if anisotropic_scale else 1, device=dev)) if estimate_scale \
            else torch.ones(N, 3, device=dev)
        opt = torch.optim.Adam([R_6d, T, s] if estimate_scale else [R_6d, T], lr=lr)
        best, R_best, acc, cnt = 1e6, rotation_6d_to_matrix(R_6d).detach(), 0.0, 0
        for it in range(n_iter):
            opt.zero_grad()
            loss = chamfer_distance(s[:, None] * pc_pred @ rotation_6d_to_matrix(R_6d) + T[:, None], pc_gt,
                                    knn_points=knn_points)[0]
            loss.backward()
            opt.step()
            acc, cnt = acc + loss.item() * N, cnt + N
            if losses is not None:
                losses.append(loss.item())
            if it % 10 == 0:
                if acc / cnt < best:
                    best, R_best = acc / cnt, rotation_6d_to_matrix(R_6d).detach()
                acc, cnt = 0.0, 0
        T, s = T.detach(), s.detach()
        return s[:, None] * pc_pred @ R_best + T[:, None], [R_best, T, s]
