"""CPU restatement (numpy + scipy.spatial.cKDTree) of the DTU chamfer evaluation of the reference
(src/utils/dtu_eval.py: evaluate_mesh, after DTUeval-python), written from its documented semantics:

  1. the mesh (float32 -> fp64 exactly, unreferenced vertices dropped) is sampled per triangle on the lattice
     c0 = (i + 0.5) / max(n1, 1e-7), c1 = (j + 0.5) / max(n2, 1e-7), c0 + c1 < 1, q = (v1 c0 + v2 c1) + t0, with
     n = floor(l / thr), thr = 0.2 sqrt(l1 l2 / area2); zero-area triangles are dropped; data_pcd = [vertices; samples];
  2. data_pcd is shuffled and greedily downsampled: in order, a point that is still alive removes every other point within
     0.2 (inclusive);
  3. points inside [BB0 - 60, BB1 + 120) (bounds in float32) are `data_in`; those whose rounded grid index
     rint((p - BB0) / Res) lies in the ObsMask grid and is set there are `data_in_obs`;
  4. acc = mean 1-NN distance data_in_obs -> STL over distances < 20; comp = the same for the STL points above the plane
     (P . [x, y, z, 1] > 0) -> data_in; avg = their mean.

Used by the CPU tests (against golden vectors produced by the reference's own code) and by
scripts/bench_dtu_eval.py --check.  No scikit-learn, no Open3D."""
import numpy as np
from scipy.spatial import cKDTree

MAX_DIST = 20
PATCH = 60
DOWNSAMPLE_DENSITY = 0.2


def remove_unreferenced(vertices, triangles):
    used = np.zeros(len(vertices), bool)
    used[triangles.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return vertices[used], remap[triangles]


def _norm(v):
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])


def triangle_lattice(tri_vert):
    """per triangle (F,3,3) fp64: v1, v2, n1, n2 and the keep mask (area2 > 0)"""
    v1 = tri_vert[:, 1] - tri_vert[:, 0]
    v2 = tri_vert[:, 2] - tri_vert[:, 0]
    cr = np.stack([v1[:, 1] * v2[:, 2] - v1[:, 2] * v2[:, 1],
                   v1[:, 2] * v2[:, 0] - v1[:, 0] * v2[:, 2],
                   v1[:, 0] * v2[:, 1] - v1[:, 1] * v2[:, 0]], -1)
    l1, l2, area2 = _norm(v1), _norm(v2), _norm(cr)
    ok = area2 > 0
    with np.errstate(divide='ignore', invalid='ignore'):
        thr = DOWNSAMPLE_DENSITY * np.sqrt(l1 * l2 / area2)
        n1, n2 = np.floor(l1 / thr), np.floor(l2 / thr)
    return v1, v2, n1, n2, ok


def sample_triangle(t0, v1, v2, n1, n2):
    """the lattice samples of one triangle, row-major over (i, j)"""
    c0 = (np.arange(int(n1) + 1, dtype=np.float64) + 0.5) / max(n1, 1e-7)
    c1 = (np.arange(int(n2) + 1, dtype=np.float64) + 0.5) / max(n2, 1e-7)
    C0, C1 = np.broadcast_arrays(c0[:, None], c1[None, :])
    inside = C0 + C1 < 1
    a, b = C0[inside][:, None], C1[inside][:, None]
    return (v1[None] * a + v2[None] * b) + t0[None]


def sample_mesh(vertices, triangles):
    """samples (S,3) of the triangles of an fp64 mesh (after remove_unreferenced), in the reference's order"""
    if len(triangles) == 0:
        return np.zeros((0, 3))
    tri_vert = vertices[triangles]
    v1, v2, n1, n2, ok = triangle_lattice(tri_vert)
    pts = [sample_triangle(tri_vert[f, 0], v1[f], v2[f], n1[f], n2[f]) for f in np.nonzero(ok)[0]]
    return np.concatenate(pts, 0) if pts else np.zeros((0, 3))


def data_pcd(vertices32, triangles):
    v, t = remove_unreferenced(np.asarray(vertices32).astype(np.float64), np.asarray(triangles, np.int64))
    return np.concatenate([v, sample_mesh(v, t)], 0)


def greedy_downsample(points, radius=DOWNSAMPLE_DENSITY):
    """keep mask of the sequential loop over `points` in order: a kept point removes all later points within radius"""
    n = len(points)
    keep = np.ones(n, bool)
    if n == 0:
        return keep
    pairs = cKDTree(points).query_pairs(radius, output_type='ndarray')     # i < j, dist <= radius
    if len(pairs) == 0:
        return keep
    pairs = pairs[np.argsort(pairs[:, 0], kind='stable')]
    starts = np.searchsorted(pairs[:, 0], np.arange(n + 1))
    later = pairs[:, 1]
    for i in np.unique(pairs[:, 0]):
        if keep[i]:
            keep[later[starts[i]:starts[i + 1]]] = False
    return keep


def nn_distance(queries, targets, max_dist=MAX_DIST):
    """1-NN distance of each query; +inf where it is not < max_dist (the reference averages only distances < max_dist)"""
    out = np.full(len(queries), np.inf)
    if len(queries) == 0 or len(targets) == 0:
        return out
    d, _ = cKDTree(targets).query(queries, k=1)
    out[d < max_dist] = d[d < max_dist]
    return out


def observation_mask(data_down, ObsMask, BB, Res):
    """(inbound, grid_inbound, in_obs) masks of the reference's masking step"""
    BB = np.asarray(BB).astype(np.float32)
    lo, hi = BB[:1] - PATCH, BB[1:] + PATCH * 2                  # float32
    inbound = ((data_down >= lo) & (data_down < hi)).sum(axis=-1) == 3
    data_in = data_down[inbound]
    grid = np.rint((data_in - BB[:1]) / Res).astype(np.int32)
    grid_inbound = ((grid >= 0) & (grid < np.asarray(ObsMask.shape)[None])).sum(axis=-1) == 3
    g = grid[grid_inbound]
    in_obs = ObsMask[g[:, 0], g[:, 1], g[:, 2]].astype(bool)
    return inbound, grid_inbound, in_obs


def above_plane(stl, P):
    P = np.asarray(P, np.float64).reshape(4)
    return ((stl[:, 0] * P[0] + stl[:, 1] * P[1]) + stl[:, 2] * P[2]) + P[3] * 1.0 > 0


def masked_mean(d, max_dist=MAX_DIST):
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.float64(d[d < max_dist].mean()) if np.any(d < max_dist) else np.float64(np.nan)


def evaluate(vertices32, triangles, order, ObsMask, BB, Res, P, stl):
    """all intermediate arrays and the scores of one evaluation under the shuffle `order` (shuffled = data_pcd[order])"""
    pcd = data_pcd(vertices32, triangles)
    shuffled = pcd[np.asarray(order)]
    keep = greedy_downsample(shuffled)
    data_down = shuffled[keep]
    inbound, grid_inbound, in_obs = observation_mask(data_down, ObsMask, BB, Res)
    data_in = data_down[inbound]
    data_in_obs = data_in[grid_inbound][in_obs]
    d2s = nn_distance(data_in_obs, stl)
    above = above_plane(stl, P)
    stl_above = stl[above]
    s2d = nn_distance(stl_above, data_in)
    acc, comp = masked_mean(d2s), masked_mean(s2d)
    return dict(data_pcd=pcd, shuffled=shuffled, keep=keep, data_down=data_down, data_in=data_in, data_in_obs=data_in_obs,
                stl_above=stl_above, d2s=d2s, s2d=s2d, acc=acc, comp=comp, avg=(acc + comp) / 2)


def scores_tsv(acc, comp, avg):
    """dtu_scores.tsv as the reference writes it (header line, one unterminated value line)"""
    return f'acc\tcomp\tavg\n{acc}\t{comp}\t{avg}'
