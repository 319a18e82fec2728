"""Seeded inputs shared by the golden-vector generator (make_golden.py) and the tests that compare against its vectors."""
import torch

from oracle import dbw_path as D


def regulariser_case():
    """4 crowded blocks (the overlap term is active), one of them killed: parameters and the state build_* leaves behind"""
    tpl = D.SceneTemplate(n_blocks=4, txt_size=16)
    p = D.init_params(4, 16, seed=2, boxy=True)
    p['alpha_logit'] = torch.tensor([3.0, 2.5, 2.0, -6.0])
    p['T'] = p['T'] * 0.02
    keep = torch.sigmoid(p['alpha_logit']) > 0.01                    # kill_blocks
    return tpl, p, keep
