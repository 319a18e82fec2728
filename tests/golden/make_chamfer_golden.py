"""Generates tests/golden/chamfer.npz: the reference's OWN chamfer_distance (src/utils/chamfer.py) and gradient_icp
(src/utils/icp.py) of a checkout of monniert/differentiable-blocksworld named by DBW_REFERENCE, extracted with `ast` by
tests/_refextract.py and run on the CPU on top of the oracle k-NN (oracle/knn.py: the kernel's float32 arithmetic and
the closed-form gradient) and dbw_b200.pointcloud's knn_gather / _validate_chamfer_reduction_inputs /
_handle_pointcloud_input.  It freezes, for a covering set of calls (every batch / point / direction reduction,
return_L1, normals, weights including all-zero weights, heterogeneous lengths, and the calls that raise), the inputs, the
outputs and the gradients of their sum; and 10 iterations of gradient_icp (isotropic and anisotropic scale): the loss of
every iteration, the returned cloud and the returned R, T, s.  Only data is stored.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_chamfer_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from _refextract import extract, have_reference  # noqa: E402

SEED = 77
ARRAYS = ('x', 'y', 'x_lengths', 'y_lengths', 'x_normals', 'y_normals', 'weights')


def clouds(seed=SEED):
    """two batches of float32 clouds with normals, lengths and weights; no exact duplicates between x and y (return_L1
    differentiates sqrt at the nearest distance)"""
    g = np.random.default_rng(seed)
    x = g.normal(0, 1, (2, 300, 3)).astype(np.float32)
    y = (g.normal(0, 1, (2, 257, 3)) * [1.3, 0.8, 1.0] + 0.2).astype(np.float32)
    nx = g.normal(0, 1, x.shape).astype(np.float32)
    ny = g.normal(0, 1, y.shape).astype(np.float32)
    return dict(x=x, y=y, x_normals=nx / np.linalg.norm(nx, axis=2, keepdims=True),
                y_normals=ny / np.linalg.norm(ny, axis=2, keepdims=True),
                x_lengths=np.array([300, 211], np.int64), y_lengths=np.array([190, 257], np.int64),
                weights=np.array([0.7, 1.9], np.float32))


def case_list():
    """(name, arrays used, keyword arguments) of every frozen call"""
    cases, i = [], 0
    for br in ('mean', 'sum', None):
        for pr in ('mean', 'sum'):
            for dr in ('sum', 'mean', 'none'):
                arrays = ['x', 'y'] + (['x_lengths', 'y_lengths'] if i % 3 == 0 else []) \
                    + (['x_normals', 'y_normals'] if i % 4 == 0 else []) + (['weights'] if i % 5 == 0 else [])
                cases.append((f'r{i:02d}', arrays, dict(batch_reduction=br, point_reduction=pr, direction_reduction=dr,
                                                        return_L1=i % 2 == 1)))
                i += 1
    full = ['x', 'y', 'x_lengths', 'y_lengths', 'x_normals', 'y_normals', 'weights']
    cases += [('all_l1', full, dict(return_L1=True)),
              ('all_none', full, dict(batch_reduction=None, direction_reduction=None)),
              ('zero_w_mean', ['x', 'y', 'weights0'], {}),
              ('zero_w_none', ['x', 'y', 'weights0'], dict(batch_reduction=None)),
              ('x_empty_row', ['x', 'y', 'x_lengths0', 'x_normals', 'y_normals'], dict(batch_reduction='sum', point_reduction='sum')),
              # the calls that raise (the message is frozen)
              ('bad_batch_red', ['x', 'y'], dict(batch_reduction='max')),
              ('bad_point_red', ['x', 'y'], dict(point_reduction=None)),
              ('x_2d', ['x2d', 'y'], {}),
              ('lengths_2d', ['x', 'y', 'x_lengths2d'], {}),
              ('length_too_long', ['x', 'y', 'x_lengths_long'], {}),
              ('normals_2d', ['x', 'y', 'x_normals2d', 'y_normals'], {}),
              ('y_batch', ['x', 'y1'], {}),
              ('y_dim', ['x', 'y2d'], {}),
              ('weights_size', ['x', 'y', 'weights3'], {}),
              ('weights_negative', ['x', 'y', 'weights_neg'], {})]
    return cases


def case_arrays(c):
    """the arrays of the derived cases: name -> (chamfer argument, value)"""
    return {'weights0': ('weights', np.zeros(2, np.float32)),
            'x_lengths0': ('x_lengths', np.array([300, 0], np.int64)),
            'x2d': ('x', c['x'][0]),
            'x_lengths2d': ('x_lengths', c['x_lengths'][None]),
            'x_lengths_long': ('x_lengths', np.array([300, 301], np.int64)),
            'x_normals2d': ('x_normals', c['x_normals'][0]),
            'y1': ('y', c['y'][:1]),
            'y2d': ('y', c['y'][..., :2].copy()),
            'weights3': ('weights', np.ones(3, np.float32)),
            'weights_neg': ('weights', np.array([1.0, -0.5], np.float32))}


def call_args(c, arrays):
    """chamfer keyword tensors of a case; x and y are leaves that require grad"""
    derived = case_arrays(c)
    out = {}
    for a in arrays:
        name, v = derived.get(a, (a, c.get(a)))
        t = torch.from_numpy(np.ascontiguousarray(v))
        out[name] = t.requires_grad_(True) if name in ('x', 'y') else t
    return out


def flatten(out):
    """chamfer's (dist, normals) with tuples / None inside -> list of arrays (None -> absent)"""
    res = []
    for o in out:
        if o is None:
            res.append(None)
        elif isinstance(o, tuple):
            res.append(list(o))
        else:
            res.append([o])
    return res


def icp_cases(seed=SEED):
    g = np.random.default_rng(seed + 1)
    gt = (g.normal(0, 1, (2, 2500, 3)) * [1.5, 1.0, 0.6]).astype(np.float32)
    a = 0.15
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    pred = ((gt[:, :2200] @ R.T) * [1.1, 0.95, 1.05] + [0.1, -0.05, 0.08] + g.normal(0, 0.01, (2, 2200, 3))).astype(np.float32)
    return [('iso', pred[:1], gt[:1], dict(estimate_scale=True, anisotropic_scale=False)),
            ('aniso', pred, gt, dict(estimate_scale=True, anisotropic_scale=True))]


def ref_chamfer_golden():
    assert have_reference()
    from oracle import knn as OK
    from dbw_b200 import pointcloud as PC
    from dbw_b200.geometry import rotation_6d_to_matrix
    ns = extract('src/utils/chamfer.py', ['chamfer_distance'],
                 {'knn_points': OK.knn_points, 'knn_gather': PC.knn_gather,
                  '_validate_chamfer_reduction_inputs': PC._validate_chamfer_reduction_inputs,
                  '_handle_pointcloud_input': PC._handle_pointcloud_input})
    chamfer = ns['chamfer_distance']
    c = clouds()
    data = {k: v for k, v in c.items()}
    meta = []
    for name, arrays, kw in case_list():
        args = call_args(c, arrays)
        entry = dict(name=name, arrays=arrays, kwargs=kw)
        try:
            out = chamfer(**args, **kw)
        except Exception as e:                          # noqa: BLE001 -- the exception is the frozen result
            entry['error'] = [type(e).__name__, str(e)]
            meta.append(entry)
            continue
        flat = flatten(out)
        entry['shape'] = [None if o is None else len(o) for o in flat]
        total = sum(t.sum() for o in flat if o is not None for t in o)
        for j, o in enumerate(flat):
            for k, t in enumerate(o or []):
                data[f'{name}__out{j}_{k}'] = t.detach().numpy()
        try:
            gx, gy = torch.autograd.grad(total, [args['x'], args['y']], allow_unused=True)
        except RuntimeError as e:
            # return_L1 with masking or weights: the reference writes in place into the output of sqrt, so its
            # backward raises; the values are still frozen
            entry['grad_error'] = str(e).split(':')[0]
        else:
            data[f'{name}__gx'] = np.zeros_like(args['x'].detach().numpy()) if gx is None else gx.numpy()
            data[f'{name}__gy'] = np.zeros_like(args['y'].detach().numpy()) if gy is None else gy.numpy()
            assert all(np.isfinite(data[f'{name}__g{a}']).all() for a in 'xy'), name
        meta.append(entry)

    losses = []

    def recorded(*a, **k):
        out = chamfer(*a, **k)
        losses.append(out[0].item())
        return out
    metrics = extract('src/utils/metrics.py', ['AverageMeter'])
    icp = extract('src/utils/icp.py', ['gradient_icp'],
                  {'nn': torch.nn, 'Adam': torch.optim.Adam, 'rotation_6d_to_matrix': rotation_6d_to_matrix,
                   'chamfer_distance': recorded, 'AverageMeter': metrics['AverageMeter']})['gradient_icp']
    icp_meta = []
    for name, pred, gt, kw in icp_cases():
        losses.clear()
        torch.manual_seed(0)
        upd, (R, T, s) = icp(torch.from_numpy(pred), torch.from_numpy(gt), lr=0.01, n_iter=10, **kw)
        data.update({f'icp_{name}__pred': pred, f'icp_{name}__gt': gt, f'icp_{name}__upd': upd.detach().numpy(),
                     f'icp_{name}__R': R.numpy(), f'icp_{name}__T': T.numpy(), f'icp_{name}__s': s.numpy(),
                     f'icp_{name}__losses': np.array(losses)})
        icp_meta.append(dict(name=name, kwargs=kw))
    data['meta'] = np.array(json.dumps(dict(cases=meta, icp=icp_meta, n_iter=10, lr=0.01)))
    return data


if __name__ == '__main__':
    if not have_reference():
        sys.exit('DBW_REFERENCE names no reference checkout')
    out = ref_chamfer_golden()
    path = os.path.join(HERE, 'chamfer.npz')
    np.savez_compressed(path, **out)
    print('wrote chamfer.npz', len(out), 'arrays,', os.path.getsize(path), 'bytes')
