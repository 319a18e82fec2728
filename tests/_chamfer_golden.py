"""Loads tests/golden/chamfer.npz (the reference's own chamfer_distance and gradient_icp, frozen by
tests/golden/make_chamfer_golden.py) and replays its calls through any chamfer_distance."""
import importlib.util
import json
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_chamfer_golden', os.path.join(HERE, 'golden', 'make_chamfer_golden.py'))
GEN = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GEN)


def load():
    d = dict(np.load(os.path.join(HERE, 'golden', 'chamfer.npz')))
    return d, json.loads(str(d['meta']))


def tensors(gold, arrays, device='cpu'):
    """the case's keyword tensors (x and y as leaves that require grad) on `device`"""
    args = GEN.call_args({k: gold[k] for k in GEN.ARRAYS}, arrays)
    return {k: (v.detach().to(device).requires_grad_(True) if k in ('x', 'y') else v.to(device)) for k, v in args.items()}


def outputs(out):
    return GEN.flatten(out)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30) if a.size else 0.0


def replay(gold, case, chamfer, device='cpu'):
    """run one non-raising golden case through `chamfer`; returns (max relative error of the outputs, of the gradients
    or None when the reference's backward raised)"""
    args = tensors(gold, case['arrays'], device)
    flat = outputs(chamfer(**args, **case['kwargs']))
    assert [None if o is None else len(o) for o in flat] == case['shape'], case['name']
    err = 0.0
    for j, o in enumerate(flat):
        for k, t in enumerate(o or []):
            err = max(err, rel(t.detach().cpu().numpy(), gold[f"{case['name']}__out{j}_{k}"]))
    if 'grad_error' in case:
        return err, None
    total = sum(t.sum() for o in flat if o is not None for t in o)
    gx, gy = torch.autograd.grad(total, [args['x'], args['y']], allow_unused=True)
    gerr = 0.0
    for g, t, a in ((gx, args['x'], 'x'), (gy, args['y'], 'y')):
        got = np.zeros(t.shape, np.float32) if g is None else g.cpu().numpy()
        want = gold[f"{case['name']}__g{a}"]
        gerr = max(gerr, np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))
    return err, gerr
