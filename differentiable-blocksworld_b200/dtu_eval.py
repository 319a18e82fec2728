"""DTU chamfer evaluation on the GPU: a drop-in for the reference's utils/dtu_eval.evaluate_mesh (after DTUeval-python),
which Trainer.evaluate() calls at the end of a DTU run on the filtered blocks scaled to millimetres.

The reference's version is an Open3D + scikit-learn CPU pipeline (a process pool of per-triangle numpy calls, a kd-tree
and a Python loop over every sampled point).  Here the per-point work runs in the sm_90a kernels of csrc/dbw_eval.cu,
in fp64 and without FMA contraction, so that the numbers are the reference's:
  sample_mesh_points   the triangle lattice samples, bit for bit numpy's, in the reference's order
  radius_downsample    the greedy 0.2 mm downsample over the shuffled cloud, exactly (as parallel rounds)
  nearest_distances    exact 1-NN distances within MAX_DIST (+inf beyond: the reference averages only distances < 20)
Scans, sorts, masking and file I/O are torch / numpy plumbing around them.  There is no CPU fallback: the point
functions take CUDA tensors and raise otherwise.

    import trainer
    trainer.evaluate_mesh = dbw_b200.dtu_eval.evaluate_mesh
"""
import ctypes
import logging
import time
from pathlib import Path

import numpy as np
import torch

from . import _lib
from ._lib import DbwError, DbwEvalGrid, check

MAX_DIST = 20
PATCH = 60
DOWNSAMPLE_DENSITY = 0.2
NN_BLOCK = 4                 # 4x4x4 cells per block of the 1-NN grid (the coarse occupancy level)
NN_MAX_CELLS = 1 << 25
MAX_ROUNDS = 10000           # rounds of the parallel downsample (a random order needs a few tens)


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _points(x, name):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise DbwError(f'{name}: expected a CUDA tensor (there is no CPU fallback)')
    if x.dim() != 2 or x.shape[1] != 3:
        raise DbwError(f'{name}: expected shape (N, 3), got {tuple(x.shape)}')
    return x.to(torch.float64).contiguous()


def _grid(lo, hi, cell, block):
    dims = [max(int(np.floor((h - l) / cell)) + 1, 1) for l, h in zip(lo, hi)]
    dims = [(d + block - 1) // block * block for d in dims]
    g = DbwEvalGrid()
    g.origin[:] = [float(x) for x in lo]
    g.cell, g.block = float(cell), block
    g.dims[:] = dims
    return g


def _cell_keys(points, grid):
    keys = torch.empty(points.shape[0], dtype=torch.int64, device=points.device)
    check(_lib.lib().dbw_eval_cell_keys(_vp(points), points.shape[0], ctypes.byref(grid), _vp(keys), _stream(points.device)),
          'dbw_eval_cell_keys')
    return keys


# ------------------------------------------------------------------------------------------------ the three stages
def sample_mesh_points(verts, faces):
    """Lattice samples (S, 3) fp64 of the triangles `faces` (F, 3) of `verts` (V, 3), in the reference's order: triangle
    order, then row-major over (i, j).  Zero-area triangles give none.  The reference's data_pcd is
    torch.cat([verts, samples]) after its unreferenced vertices are dropped."""
    v = _points(verts, 'verts')
    dev = v.device
    f = faces.to(device=dev, dtype=torch.int64).contiguous()
    if f.dim() != 2 or f.shape[1] != 3:
        raise DbwError(f'faces: expected shape (F, 3), got {tuple(f.shape)}')
    F = f.shape[0]
    empty = torch.zeros(0, 3, dtype=torch.float64, device=dev)
    if F == 0:
        return empty
    if int(f.min()) < 0 or int(f.max()) >= v.shape[0]:
        raise DbwError('faces: vertex index out of range')
    L, st = _lib.lib(), _stream(dev)
    tri = torch.empty(F, 12, dtype=torch.float64, device=dev)
    rows = torch.empty(F, dtype=torch.int64, device=dev)
    check(L.dbw_eval_sample_setup(_vp(v), _vp(f), F, _vp(tri), _vp(rows), st), 'dbw_eval_sample_setup')
    row_begin = torch.zeros(F + 1, dtype=torch.int64, device=dev)
    torch.cumsum(rows, 0, out=row_begin[1:])
    R = int(row_begin[-1])
    if R == 0:
        return empty
    row_count = torch.empty(R, dtype=torch.int64, device=dev)
    check(L.dbw_eval_sample_count(_vp(tri), _vp(row_begin), F, R, _vp(row_count), st), 'dbw_eval_sample_count')
    sample_begin = torch.zeros(R + 1, dtype=torch.int64, device=dev)
    torch.cumsum(row_count, 0, out=sample_begin[1:])
    S = int(sample_begin[-1])
    out = torch.empty(S, 3, dtype=torch.float64, device=dev)
    if S:
        check(L.dbw_eval_sample_write(_vp(tri), _vp(row_begin), F, R, _vp(row_count), _vp(sample_begin), _vp(out), st),
              'dbw_eval_sample_write')
    return out


def radius_downsample(points, radius=DOWNSAMPLE_DENSITY, max_rounds=MAX_ROUNDS):
    """(keep (N,) bool, rounds) of the reference's greedy loop over `points` in their order: a point still alive removes
    every other point within `radius` (inclusive).  Exact, computed in parallel rounds; more than `max_rounds` raises."""
    p = _points(points, 'points')
    dev, n = p.device, p.shape[0]
    if n == 0:
        return torch.zeros(0, dtype=torch.bool, device=dev), 0
    if n > 2 ** 31 - 1:
        raise DbwError('radius_downsample: more than 2^31 - 1 points')
    lo, hi = p.min(0).values.tolist(), p.max(0).values.tolist()
    if not all(np.isfinite(lo + hi)):
        raise DbwError('radius_downsample: non-finite coordinates')
    # cells no smaller than the radius: every neighbour lies in the 3x3x3 cells around a point
    cell = max(radius * (1 + 1e-6), max(h - l for l, h in zip(lo, hi)) / (1 << 20), 1e-300)
    grid = _grid(lo, hi, cell, 1)
    keys, perm = torch.sort(_cell_keys(p, grid), stable=True)
    ps = p[perm].contiguous()
    ukeys, counts = torch.unique_consecutive(keys, return_counts=True)
    C = ukeys.shape[0]
    cbegin = torch.zeros(C + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=cbegin[1:])
    cell_of = torch.repeat_interleave(torch.arange(C, dtype=torch.int32, device=dev), counts)
    nb = torch.empty(C, 9, dtype=torch.int32, device=dev)
    ne = torch.empty(C, 9, dtype=torch.int32, device=dev)
    L, st = _lib.lib(), _stream(dev)
    check(L.dbw_eval_cell_ranges(_vp(ukeys), _vp(cbegin), C, ctypes.byref(grid), _vp(nb), _vp(ne), st), 'dbw_eval_cell_ranges')
    nbytes = ctypes.c_size_t(0)
    check(L.dbw_eval_downsample_workspace_bytes(n, ctypes.byref(nbytes)), 'dbw_eval_downsample_workspace_bytes')
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    rounds = ctypes.c_int32(0)
    check(L.dbw_eval_radius_downsample(_vp(ps), _vp(perm), _vp(cell_of), _vp(nb), _vp(ne), n, float(radius), int(max_rounds),
                                       _vp(keep), ctypes.byref(rounds), _vp(ws), nbytes.value, st), 'dbw_eval_radius_downsample')
    return keep.bool(), rounds.value


def nearest_distances(queries, targets, max_dist=MAX_DIST):
    """(Nq,) fp64 distance from each query to its nearest target when that is < max_dist, +inf otherwise (no target
    within max_dist, or no target at all).  Exact: sqrt((dx^2 + dy^2) + dz^2) of the nearest point."""
    q, t = _points(queries, 'queries'), _points(targets, 'targets')
    dev, nq, nt = q.device, q.shape[0], t.shape[0]
    out = torch.full((nq,), float('inf'), dtype=torch.float64, device=dev)
    if nq == 0 or nt == 0:
        return out
    if nt > 2 ** 31 - 1:
        raise DbwError('nearest_distances: more than 2^31 - 1 targets')
    lo, hi = t.min(0).values.tolist(), t.max(0).values.tolist()
    if not all(np.isfinite(lo + hi)):
        raise DbwError('nearest_distances: non-finite target coordinates')
    # about 8 cells per target over the bounding box, at most NN_MAX_CELLS cells, and blocks no smaller than max_dist / 8
    # (a query walks at most ~10 rings of blocks before the cutoff ends its search, whatever the cloud's extent)
    ext = [max(h - l, 1e-9 * (1 + abs(l) + abs(h))) for l, h in zip(lo, hi)]
    cell = max((ext[0] * ext[1] * ext[2] / (8 * nt)) ** (1 / 3), max_dist / (8 * NN_BLOCK))
    while True:
        grid = _grid(lo, hi, cell, NN_BLOCK)
        if grid.dims[0] * grid.dims[1] * grid.dims[2] <= NN_MAX_CELLS:
            break
        cell *= 1.25
    n_cells = grid.dims[0] * grid.dims[1] * grid.dims[2]
    keys, perm = torch.sort(_cell_keys(t, grid))
    ts = t[perm].contiguous()
    cell_start = torch.zeros(n_cells + 1, dtype=torch.int32, device=dev)
    torch.cumsum(torch.bincount(keys, minlength=n_cells), 0, out=cell_start[1:])
    qperm = torch.sort(_cell_keys(q, grid)).indices        # coherent warps: neighbouring queries search the same cells
    qs = q[qperm].contiguous()
    d = torch.empty(nq, dtype=torch.float64, device=dev)
    check(_lib.lib().dbw_eval_nn_distance(_vp(qs), nq, _vp(ts), _vp(cell_start), ctypes.byref(grid), float(max_dist), _vp(d),
                                          _stream(dev)), 'dbw_eval_nn_distance')
    out[qperm] = d
    return out


# ------------------------------------------------------------------------------------------------ PLY (vertex element)
_PLY_TYPES = {'char': 'i1', 'int8': 'i1', 'uchar': 'u1', 'uint8': 'u1', 'short': 'i2', 'int16': 'i2', 'ushort': 'u2',
              'uint16': 'u2', 'int': 'i4', 'int32': 'i4', 'uint': 'u4', 'uint32': 'u4', 'float': 'f4', 'float32': 'f4',
              'double': 'f8', 'float64': 'f8'}


def read_ply(path):
    """(N, 3) fp64 x y z of the vertex element of a PLY file (ascii or binary_little_endian; other properties skipped;
    the vertex element must come first or after elements without list properties)."""
    with open(path, 'rb') as fh:
        if fh.readline().strip() != b'ply':
            raise ValueError(f'{path}: not a PLY file')
        fmt, elements = None, []
        while True:
            line = fh.readline()
            if not line:
                raise ValueError(f'{path}: no end_header')
            tok = line.decode('ascii', 'replace').split()
            if not tok or tok[0] in ('comment', 'obj_info'):
                continue
            if tok[0] == 'end_header':
                break
            if tok[0] == 'format':
                fmt = tok[1]
            elif tok[0] == 'element':
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == 'property':
                if tok[1] == 'list':
                    elements[-1][2].append((tok[4], None))
                else:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
        if fmt not in ('ascii', 'binary_little_endian'):
            raise ValueError(f'{path}: unsupported PLY format {fmt}')
        body = fh.read()
    offset = 0
    for name, count, props in elements:
        if name == 'vertex':
            names = [p for p, _ in props]
            if any(t is None for _, t in props) or not {'x', 'y', 'z'} <= set(names):
                raise ValueError(f'{path}: vertex element needs scalar x y z properties')
            if fmt == 'ascii':
                lines = body.decode('ascii').splitlines()[offset:offset + count]
                vals = np.array([[float(x) for x in l.split()[:len(names)]] for l in lines], np.float64).reshape(count, len(names))
                return vals[:, [names.index('x'), names.index('y'), names.index('z')]].copy()
            dt = np.dtype([(p, '<' + t) for p, t in props])
            arr = np.frombuffer(body, dt, count=count, offset=offset)
            return np.stack([arr['x'], arr['y'], arr['z']], 1).astype(np.float64)
        if any(t is None for _, t in props):
            raise ValueError(f'{path}: element {name} with list properties before the vertex element')
        offset += count if fmt == 'ascii' else count * np.dtype([(p, '<' + t) for p, t in props]).itemsize
    raise ValueError(f'{path}: no vertex element')


def write_ply(path, points, colors=None, binary=True):
    """points (N, 3) as double x y z, colors (N, 3) in [0, 1] as uchar red green blue (round(255 c), as Open3D writes them)."""
    points = np.asarray(points, np.float64).reshape(-1, 3)
    fields = [('x', '<f8'), ('y', '<f8'), ('z', '<f8')]
    if colors is not None:
        fields += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
    arr = np.empty(len(points), np.dtype(fields))
    arr['x'], arr['y'], arr['z'] = points.T
    if colors is not None:
        c = np.floor(np.clip(np.asarray(colors, np.float64).reshape(-1, 3), 0, 1) * 255 + 0.5).astype(np.uint8)
        arr['red'], arr['green'], arr['blue'] = c.T
    head = ['ply', f'format {"binary_little_endian" if binary else "ascii"} 1.0', f'element vertex {len(points)}',
            'property double x', 'property double y', 'property double z']
    if colors is not None:
        head += ['property uchar red', 'property uchar green', 'property uchar blue']
    head.append('end_header')
    with open(path, 'wb') as fh:
        fh.write(('\n'.join(head) + '\n').encode('ascii'))
        if binary:
            fh.write(arr.tobytes())
        else:
            for row in arr:
                fh.write((' '.join(repr(float(v)) if i < 3 else str(int(v)) for i, v in enumerate(row)) + '\n').encode('ascii'))


# ------------------------------------------------------------------------------------------------ the evaluation
def _remove_unreferenced(verts, faces):
    used = torch.zeros(verts.shape[0], dtype=torch.bool, device=verts.device)
    used[faces.reshape(-1)] = True
    remap = torch.cumsum(used.to(torch.int64), 0) - 1
    return verts[used], remap[faces]


def _masked_mean(d):
    d = d.cpu().numpy()
    return d[d < MAX_DIST].mean()         # numpy's pairwise sum in the reference's order; NaN (and a warning) when empty


def evaluate_arrays(verts, faces, stl, obs_mask, bb, res, plane, *, order=None, seed=None, device=None, timer=None):
    """The evaluation on arrays: verts (V, 3) float32 (converted exactly to fp64), faces (F, 3), stl (M, 3), ObsMask, BB,
    Res and the plane P as loaded from the DTU .mat files.  The shuffle is `order` (shuffled = data_pcd[order]) when
    given, else a random permutation (seeded by `seed` when given).  `timer(stage)` is called after each stage.
    Returns the scores and the intermediate clouds (CUDA tensors)."""
    dev = torch.device(device) if device is not None else (verts.device if torch.is_tensor(verts) and verts.is_cuda
                                                          else torch.device('cuda', torch.cuda.current_device()))
    tick = timer or (lambda stage: None)
    v = torch.as_tensor(verts).detach().to(dev).to(torch.float64)
    f = torch.as_tensor(faces).detach().to(device=dev, dtype=torch.int64)
    if f.numel():
        v, f = _remove_unreferenced(v, f)
    else:
        v = v[:0]
    data_pcd = torch.cat([v, sample_mesh_points(v, f.reshape(-1, 3))])
    tick('sample')
    n = data_pcd.shape[0]
    if order is not None:
        perm = torch.as_tensor(np.asarray(order) if not torch.is_tensor(order) else order).to(device=dev, dtype=torch.int64)
        if perm.shape != (n,):
            raise DbwError(f'order: expected a permutation of {n} points, got shape {tuple(perm.shape)}')
    else:
        gen = torch.Generator(device=dev)
        if seed is not None:
            gen.manual_seed(int(seed))
        else:
            gen.seed()
        perm = torch.randperm(n, generator=gen, device=dev)
    shuffled = data_pcd[perm]
    tick('shuffle')
    keep, rounds = radius_downsample(shuffled)
    data_down = shuffled[keep]
    tick('downsample')
    # the mask bounds are formed in float32 (the reference casts BB), then compared with the fp64 points
    bb32 = torch.from_numpy(np.ascontiguousarray(np.asarray(bb).astype(np.float32)))
    lo, hi = (bb32[:1] - PATCH).double().to(dev), (bb32[1:] + PATCH * 2).double().to(dev)
    inbound = ((data_down >= lo) & (data_down < hi)).all(1)
    data_in = data_down[inbound]
    res_t = torch.from_numpy(np.asarray(res, np.float64)).to(dev)
    obs = torch.from_numpy(np.ascontiguousarray(np.asarray(obs_mask).astype(bool))).to(dev)
    grid = torch.round((data_in - bb32[:1].double().to(dev)) / res_t).to(torch.int32)      # half to even, as np.around
    shape = torch.tensor(obs.shape, dtype=torch.int32, device=dev)
    grid_inbound = ((grid >= 0) & (grid < shape)).all(1)
    g = grid[grid_inbound].long()
    in_obs = obs[g[:, 0], g[:, 1], g[:, 2]]
    data_in_obs = data_in[grid_inbound][in_obs]
    tick('mask')
    stl_t = torch.as_tensor(stl).to(device=dev, dtype=torch.float64)
    d2s = nearest_distances(data_in_obs, stl_t)
    tick('d2s')
    P = np.asarray(plane, np.float64).reshape(4)
    above = ((stl_t[:, 0] * P[0] + stl_t[:, 1] * P[1]) + stl_t[:, 2] * P[2]) + P[3] * 1.0 > 0
    stl_above = stl_t[above]
    s2d = nearest_distances(stl_above, data_in)
    tick('s2d')
    acc, comp = _masked_mean(d2s), _masked_mean(s2d)
    return dict(acc=acc, comp=comp, avg=(acc + comp) / 2, rounds=rounds, data_pcd=data_pcd, shuffled=shuffled, keep=keep,
                data_down=data_down, inbound=inbound, grid_inbound=grid_inbound, in_obs=in_obs, data_in=data_in,
                data_in_obs=data_in_obs, above=above, stl_above=stl_above, d2s=d2s, s2d=s2d, stl=stl_t)


def _vis_colors(n, idx, dist):
    """the reference's colouring: blue, points with a distance red -> white by distance (1 mm = red), green beyond MAX_DIST"""
    color = np.tile(np.array([[0., 0., 1.]]), (n, 1))
    alpha = np.clip(dist, None, 1)[:, None]
    color[idx] = np.array([[1., 0., 0.]]) * alpha + np.array([[1., 1., 1.]]) * (1 - alpha)
    color[idx[dist >= MAX_DIST]] = np.array([0., 1., 0.])
    return color


def _print_log(msg):
    print(f'[{time.strftime("%Y-%m-%d %H:%M:%S")}] {msg}')
    logging.getLogger('trainer').info(msg)


def evaluate_mesh(inp, scan_id, dataset_dir, eval_dir, suffix='', save_viz=True, *, order=None, seed=None, device=None):
    """The reference's evaluate_mesh(inp, scan_id, dataset_dir, eval_dir, suffix='', save_viz=True): `inp` is a Meshes
    (its first mesh) or the path of an .obj; reads {dataset_dir}/ObsMask/ObsMask{scan}_10.mat, ObsMask/Plane{scan}.mat and
    Points/stl/stl{scan:03}_total.ply; writes {eval_dir}/dtu_scores{suffix}.tsv (and, with save_viz, the coloured clouds
    vis_{scan:03}_d2s{suffix}.ply / vis_{scan:03}_s2d{suffix}.ply).  Keyword-only: `order` (explicit shuffle permutation),
    `seed`, `device`.  Returns {'acc', 'comp', 'avg'}."""
    from scipy.io import loadmat
    from .geometry import load_obj
    if isinstance(inp, (str, Path)):
        verts, faces = load_obj(str(inp))
    elif hasattr(inp, 'get_mesh_verts_faces'):
        verts, faces = inp.get_mesh_verts_faces(0)
    else:
        raise TypeError(f'evaluate_mesh: expected a Meshes or a path, got {type(inp).__name__}')
    m = loadmat(f'{dataset_dir}/ObsMask/ObsMask{scan_id}_10.mat')
    P = loadmat(f'{dataset_dir}/ObsMask/Plane{scan_id}.mat')['P']
    stl = read_ply(f'{dataset_dir}/Points/stl/stl{scan_id:03}_total.ply')
    r = evaluate_arrays(verts, faces, stl, m['ObsMask'], m['BB'], m['Res'], P, order=order, seed=seed, device=device)
    acc, comp, avg = r['acc'], r['comp'], r['avg']
    if save_viz:
        down = r['data_down'].cpu().numpy()
        idx = torch.nonzero(r['inbound']).reshape(-1)[r['grid_inbound']][r['in_obs']].cpu().numpy()
        write_ply(f'{eval_dir}/vis_{scan_id:03}_d2s{suffix}.ply', down, _vis_colors(len(down), idx, r['d2s'].cpu().numpy()))
        idx = torch.nonzero(r['above']).reshape(-1).cpu().numpy()
        write_ply(f'{eval_dir}/vis_{scan_id:03}_s2d{suffix}.ply', stl, _vis_colors(len(stl), idx, r['s2d'].cpu().numpy()))
    with open(f'{eval_dir}/dtu_scores{suffix}.tsv', 'w') as fh:
        fh.write('acc\tcomp\tavg\n')
        fh.write(f'{acc}\t{comp}\t{avg}')
    _print_log('dtu_scores{}: acc={:.5f}, comp={:.5f}, avg={:.5f}'.format(suffix, acc, comp, avg))
    return {'acc': float(acc), 'comp': float(comp), 'avg': float(avg)}
